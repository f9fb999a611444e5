"""Regenerates the byte-form fixtures from the reference tree (run where the reference is checked out; it is not needed to run
the tests).  Only DATA is copied, never source code.

    varuna_bytes/<program>.verifier, .metadata   parameters/src/mainnet/resources/*.verifier and their .metadata, whole: a version
                                                 byte, a 664-byte compressed CircuitVerifyingKey, in most files a u64
                                                 num_variables; the metadata's verifier_checksum is the file's SHA-256
    varuna_bytes/genesis_proof_<k>.bin           the 8 compressed Varuna proofs of parameters/src/mainnet/resources/block.genesis
                                                 (an execution and a fee proof per transaction), each cut from its first byte to
                                                 its last; the synthesizer's version byte 1 before each is not kept

The proofs are found by walking the proof layout (tests/varuna_bytes_oracle.py) at every offset after a version byte 1: a proof
is where the walk reads one circuit, a small batch, every point decodes and every Fr is below r.

    python tests/golden/make_bytes_golden.py [/root/reference]
"""
import glob
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]
import varuna_bytes_oracle as vb                                                 # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
RES = os.path.join(REF, "parameters/src/mainnet/resources")
OUT = os.path.join(HERE, "varuna_bytes")
os.makedirs(OUT, exist_ok=True)

names = sorted(os.path.basename(f)[:-len(".verifier")] for f in glob.glob(os.path.join(RES, "*.verifier")))
assert len(names) == 16, names
for n in names:
    for ext in (".verifier", ".metadata"):
        shutil.copyfile(os.path.join(RES, n + ext), os.path.join(OUT, n + ext))

with open(os.path.join(RES, "block.genesis"), "rb") as f:
    block = f.read()
found = []
for off in range(1, len(block) - 8):
    if block[off - 1] != 1 or block[off: off + 8] != b"\x01" + b"\x00" * 7:          # a version byte, then one circuit
        continue
    r = vb.Reader(block, off, compressed=True)
    try:
        p = vb.read_proof(r)
    except ValueError:
        continue
    if 1 <= sum(p["batch_sizes"]) <= 64:
        found.append((off, r.o))
assert len(found) == 8, found
for k, (a, b) in enumerate(found):
    with open(os.path.join(OUT, f"genesis_proof_{k}.bin"), "wb") as f:
        f.write(block[a:b])
print("proofs at", [a for a, _b in found], "sizes", sorted({b - a for a, b in found}))
print(f"wrote {len(names)} verifying keys and {len(found)} proofs to {OUT}")
