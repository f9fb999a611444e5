"""Regenerates the Poseidon fixture from the reference tree (run in the build container only; the reference tree does not exist on
the GPU machines).  Only DATA is extracted — the expect-test snapshots of algorithms/src/crypto_hash/tests.rs — never source code.

    python tests/golden/make_poseidon_golden.py [path/to/snarkVM]

Writes poseidon_vectors.json:
  * grain_first_sample, grain_second_sample — test_grain_lfsr_consistency: PoseidonGrainLFSR::new(false, 253, 3, 8, 31), two
                              rejection-sampled Fr elements;
  * ark, mds                — bls12_377_fr_poseidon_default_parameters_test: Fr::default_poseidon_parameters::<RATE>() for
                              RATE = 2 … 8 (optimize_for_weights false), keyed by the rate;
  * absorb_squeeze          — test_poseidon_sponge_consistency: PoseidonSponge<Fr, 2, 1> after absorbing `absorb` copies of 1237812
                              and squeezing `squeeze` native elements, for absorb, squeeze in 0 … 9, keyed "absorb,squeeze".
Every value is a canonical decimal integer, as the snapshots print them.
"""
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
SNAP = os.path.join(REF, "algorithms/src/crypto_hash/resources/poseidon")
OUT = os.path.dirname(os.path.abspath(__file__))
PREFIX = "snarkvm_algorithms_crypto_hash_tests_"


def snapshot(name):
    """the snapshot's nested list of integers"""
    with open(os.path.join(SNAP, PREFIX + name + ".snap")) as f:
        text = f.read().strip()
    assert re.fullmatch(r"[\[\]\d,\s]*", text), name
    return json.loads(text)


golden = {
    "grain_first_sample": snapshot("first sample"),
    "grain_second_sample": snapshot("second sample"),
    "ark": {str(r): snapshot(f"Ark for rate {r} and optimize_for_weights false") for r in range(2, 9)},
    "mds": {str(r): snapshot(f"MDS for rate {r} and optimize_for_weights false") for r in range(2, 9)},
    "absorb_squeeze": {f"{a},{s}": snapshot(f"Absorb {a} and Squeeze {s}") for a in range(10) for s in range(10)},
}
with open(os.path.join(OUT, "poseidon_vectors.json"), "w") as f:
    json.dump(golden, f, indent=0)
    f.write("\n")
print("wrote", os.path.join(OUT, "poseidon_vectors.json"))
