"""CPU: the instruction mix of the out-of-line Montgomery product and square (Fp::mul_call / Fp::sqr_call, csrc/ff.cuh) in the
built library, read with cuobjdump.

Every 32×32→64 product of the multiplier should be ONE IMAD.WIDE.U32(.X).  ptxas can instead issue a product as IMAD.X for the
low word plus IMAD.HI.U32.X for the high word, with the carry threaded through both: twice the fmaheavy instructions and a carry
chain twice as long.  It did so for every m·p product of the reduction rows until the reduction multiplier m = −x was written so
that ptxas no longer folds the negation into the products (ptx_neg).  A later edit or toolkit that splits the products again
fails here, without a GPU.

mul_call and sqr_call are called, and only they, by msm.cu's element-wise test kernel k_test_field_op<P> (FF_CALL_MUL), so they
are the two subroutines its SASS calls; the MSM kernels call the same functions.
"""
import collections
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "snarkvm_b200", "libsnarkvm_b200.so")


def _cuobjdump():
    found = shutil.which("cuobjdump")
    if found:
        return found
    for base in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if base and os.path.exists(os.path.join(base, "bin", "cuobjdump")):
            return os.path.join(base, "bin", "cuobjdump")
    return None


CUOBJDUMP = _cuobjdump()
pytestmark = pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump not found")

INS = re.compile(r"\s+/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)(.*?);")


def _mix(body):
    c = collections.Counter()
    for op in body:
        if op.startswith("IMAD.WIDE"):
            c["wide"] += 1
        elif op.startswith("IMAD.HI"):
            c["hi"] += 1
        elif op.startswith(("IMAD.MOV", "IMAD.SHL", "IMAD.IADD")):
            continue                                   # moves and shifts ptxas places on the IMAD pipe
        elif op.startswith("IMAD"):
            c["lo"] += 1
    c["family"] = c["wide"] + c["hi"] + c["lo"]
    return c


@pytest.fixture(scope="module")
def sass():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is not built")
    out = subprocess.run([CUOBJDUMP, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = INS.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2), m.group(3)))
    return funcs


def _mul_and_sqr(funcs, params):
    names = [f for f in funcs if "msm_cu" in f and f"k_test_field_opINS_8{params}" in f]
    assert len(names) == 1, names
    ins = funcs[names[0]]
    targets = sorted({int(re.search(r"0x([0-9a-f]+)", args).group(1), 16) for _, op, args in ins if op.startswith("CALL.REL")})
    assert len(targets) == 2, f"{names[0]} calls {len(targets)} subroutines, expected mul_call and sqr_call"
    bodies = []
    for t in targets:
        body = []
        for addr, op, _ in ins:
            if addr < t:
                continue
            body.append(op)
            if op.startswith("RET"):
                break
        bodies.append(_mix(body))
    bodies.sort(key=lambda c: c["family"])
    return bodies[1], bodies[0]                        # the product has more multiplications than the square


# N limbs; 32×32→64 products per call: mul = N² (a·b) + N(N−1) (m·p, p[0] = 1 needs none);
# sqr = N(N−1)/2 cross + N diagonal + N(N−1) (m·p)
FIELDS = {"FqParams": 12, "FrParams": 8}


@pytest.mark.parametrize("params", sorted(FIELDS))
def test_every_product_is_one_wide_multiply(sass, params):
    N = FIELDS[params]
    mul, sqr = _mul_and_sqr(sass, params)
    for what, c, products in (("mul_call", mul, 2 * N * N - N), ("sqr_call", sqr, N * (N - 1) // 2 + N + N * (N - 1))):
        assert c["hi"] <= N, f"{params} {what}: {c['hi']} IMAD.HI.U32 — products are split into IMAD + IMAD.HI again ({dict(c)})"
        assert c["wide"] >= 0.95 * products, f"{params} {what}: {c['wide']} IMAD.WIDE for {products} products ({dict(c)})"
        assert c["family"] <= 1.12 * products, f"{params} {what}: {c['family']} IMAD-family instructions for {products} products ({dict(c)})"
