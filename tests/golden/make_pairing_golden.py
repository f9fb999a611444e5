"""Regenerates the pairing fixtures from the reference tree (run in the build container only; the reference tree does not exist on
the GPU machines).  Only DATA is extracted — constants and SRS points — never source code.

    python tests/golden/make_pairing_golden.py [path/to/snarkVM]

Writes
  * pairing_constants.json — the Frobenius coefficients of curves/src/bls12_377/fq6.rs (FROBENIUS_COEFF_FP6_C1, _C2) and fq12.rs
                             (FROBENIUS_COEFF_FP12_C1) as Montgomery u64 limbs, [c0 limbs, c1 limbs] per Fq2;
  * beta_h.usrs            — parameters/src/mainnet/resources/beta-h.usrs, the mainnet β·H (192 B: x.c0, x.c1, y.c0, y.c1, 48 B LE
                             each, flags in the top bits of the last byte).
"""
import json
import os
import re
import shutil
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))


def read(p):
    with open(os.path.join(REF, p)) as f:
        return f.read()


def fq2_table(src, name):
    """the `[Fq2; n]` table `const NAME`: every BigInteger limb list in order, paired (c0, c1)"""
    m = re.search(r"const\s+" + name + r"\b[^=]*=\s*\[(.*?)\n    \];", src, re.S)
    assert m, name
    lists = []
    for lm in re.finditer(r"BigInteger(?:384)?\(\[([^\[\]]*?)\]\)", m.group(1), re.S):
        lists.append([int(t.strip().replace("_", "").replace("u64", ""), 0) for t in lm.group(1).split(",") if t.strip()])
    assert len(lists) % 2 == 0, name
    return [[lists[i], lists[i + 1]] for i in range(0, len(lists), 2)]


fq6 = read("curves/src/bls12_377/fq6.rs")
fq12 = read("curves/src/bls12_377/fq12.rs")
golden = {
    "source": "curves/src/bls12_377/fq6.rs (FROBENIUS_COEFF_FP6_C1, FROBENIUS_COEFF_FP6_C2), curves/src/bls12_377/fq12.rs "
              "(FROBENIUS_COEFF_FP12_C1); Montgomery u64 limbs, [c0, c1] per Fq2",
    "FROBENIUS_COEFF_FP6_C1": fq2_table(fq6, "FROBENIUS_COEFF_FP6_C1"),
    "FROBENIUS_COEFF_FP6_C2": fq2_table(fq6, "FROBENIUS_COEFF_FP6_C2"),
    "FROBENIUS_COEFF_FP12_C1": fq2_table(fq12, "FROBENIUS_COEFF_FP12_C1"),
}
assert [len(golden[k]) for k in ("FROBENIUS_COEFF_FP6_C1", "FROBENIUS_COEFF_FP6_C2", "FROBENIUS_COEFF_FP12_C1")] == [6, 6, 12]
with open(os.path.join(OUT, "pairing_constants.json"), "w") as f:
    json.dump(golden, f, indent=1)
shutil.copyfile(os.path.join(REF, "parameters/src/mainnet/resources/beta-h.usrs"), os.path.join(OUT, "beta_h.usrs"))
print("wrote pairing_constants.json, beta_h.usrs")
