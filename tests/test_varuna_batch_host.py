"""CPU: the argument checks of the many-circuit Varuna calls, which raise before anything reaches a device, and the ctypes images of
the C ABI's segment tables (include/snarkvm_b200.h) that carry every circuit's matrices and polynomials to the segmented kernels."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_empty_and_mismatched_batches_raise():
    from snarkvm_b200 import varuna as dv
    with pytest.raises(ValueError):
        dv.index_circuits([])
    with pytest.raises(ValueError):
        dv.batch_circuit_setup([], None, None)
    with pytest.raises(ValueError):
        dv.prove_vk_batch([], [], [])
    with pytest.raises(ValueError):
        dv.verify_vk_batch([], [], [], [], [])
    with pytest.raises(ValueError):                                      # one set of challenges per proving key
        dv.prove_vk_batch([object(), object()], [[0] * 12], [[1, 2]] * 2)
    with pytest.raises(ValueError):                                      # a certificate takes twelve challenges
        dv.prove_vk_batch([object()], [[0] * 11], [[1, 2]])
    with pytest.raises(ValueError):
        dv.verify_vk_batch([object()], [object()], [object()], [[0] * 12], [])


def _c_struct_fields(name: str) -> list:
    """the member declarations of `typedef struct { … } name;` in the public header, one (type, declarator) per member"""
    src = open(os.path.join(ROOT, "include", "snarkvm_b200.h")).read()
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", src).group(1)
    fields = []
    for decl in body.split(";"):
        decl = " ".join(decl.split())
        if not decl:
            continue
        m = re.match(r"(const void\*|void\*|uint64_t|uint32_t|uint8_t) (.*)", decl)
        for d in m.group(2).split(","):
            fields.append((m.group(1), d.strip().lstrip("*")))
    return fields


_C_SIZE = {"const void*": 8, "void*": 8, "uint64_t": 8, "uint32_t": 4, "uint8_t": 1}


@pytest.mark.parametrize("c_name, py_name", [("snarkvm_b200_csr_segment_t", "CsrSegment"),
                                             ("snarkvm_b200_lincomb_segment_t", "LincombSegment"),
                                             ("snarkvm_b200_evals_segment_t", "EvalsSegment")])
def test_segment_structs_match_the_header(c_name, py_name):
    """same members in the same order at the same offsets (natural alignment, as the C compiler lays them out)"""
    from snarkvm_b200 import _lib
    cls = getattr(_lib, py_name)
    fields = _c_struct_fields(c_name)
    assert [f for f, _ in cls._fields_] == [re.sub(r"\[.*", "", d) for _, d in fields]
    off = 0
    for (ctype, decl), (pname, _t) in zip(fields, cls._fields_):
        size = _C_SIZE[ctype]
        count = 1
        for dim in re.findall(r"\[(\d+)\]", decl):
            count *= int(dim)
        off = (off + size - 1) // size * size
        assert getattr(cls, pname).offset == off, (c_name, pname)
        assert getattr(cls, pname).size == size * count, (c_name, pname)
        off += size * count
    assert ctypes.sizeof(cls) == (off + 7) // 8 * 8
