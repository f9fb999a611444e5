"""Regenerates the verifier's mainnet fixtures from the reference tree (run in the build container only; /root/reference does not
exist on the GPU box).  Only DATA is copied — SRS points — never source code.

    neg_powers_of_beta.usrs        parameters/src/mainnet/resources/neg-powers-of-beta.usrs, whole (β^{-(D − d)}·H for d = 2^k − 2)
    powers_of_beta_gamma.usrs      parameters/src/mainnet/resources/powers-of-beta-gamma.usrs, whole (γβ^i·G; key 0 is γ·G)
    shifted_powers_of_beta_top1024.usrs
                                   the last 1024 points of parameters/src/mainnet/resources/shifted-powers-of-beta-15.usrs (the top
                                   2^15 powers of the 2^28 SRS), under the same u64 count header: β^{D − 1023} … β^D·G, D = 2^28 − 1,
                                   every shift the tests' degree bounds (at most 1022) need

    python tests/golden/make_verifier_golden.py [/root/reference]
"""
import os
import shutil
import struct
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
RES = os.path.join(REF, "parameters/src/mainnet/resources")
TOP = 1024

for name in ("neg-powers-of-beta", "powers-of-beta-gamma"):
    shutil.copyfile(os.path.join(RES, f"{name}.usrs"), os.path.join(OUT, f"{name.replace('-', '_')}.usrs"))
with open(os.path.join(RES, "shifted-powers-of-beta-15.usrs"), "rb") as f:
    blob = f.read()
(n,) = struct.unpack_from("<Q", blob, 0)
assert len(blob) == 8 + 96 * n and n >= TOP
with open(os.path.join(OUT, f"shifted_powers_of_beta_top{TOP}.usrs"), "wb") as f:
    f.write(struct.pack("<Q", TOP) + blob[8 + 96 * (n - TOP):])
print("wrote neg_powers_of_beta.usrs, powers_of_beta_gamma.usrs, shifted_powers_of_beta_top1024.usrs")
