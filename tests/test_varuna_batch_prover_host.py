"""CPU: the ctypes images of the batched prover's segment tables (include/snarkvm_b200.h) and the argument checks of
varuna.BatchProver that raise before anything reaches a device."""
import pytest

from test_varuna_batch_host import _c_struct_fields, _C_SIZE


@pytest.mark.parametrize("c_name, py_name", [("snarkvm_b200_lincomb_term_t", "LincombTerm"),
                                             ("snarkvm_b200_lincomb_output_t", "LincombOutput"),
                                             ("snarkvm_b200_spmv_segment_t", "SpmvSegment"),
                                             ("snarkvm_b200_polymul_job_t", "PolymulJob"),
                                             ("snarkvm_b200_round4_segment_t", "Round4Segment")])
def test_prover_structs_match_the_header(c_name, py_name):
    """same members in the same order at the same offsets (natural alignment, as the C compiler lays them out)"""
    import ctypes
    import re
    from snarkvm_b200 import _lib
    cls = getattr(_lib, py_name)
    fields = _c_struct_fields(c_name)
    assert [f for f, _ in cls._fields_] == [re.sub(r"\[.*", "", d) for _, d in fields]
    off = 0
    for (ctype, decl), (pname, _t) in zip(fields, cls._fields_):
        size, count = _C_SIZE[ctype], 1
        for dim in re.findall(r"\[(\d+)\]", decl):
            count *= int(dim)
        off = (off + size - 1) // size * size
        assert getattr(cls, pname).offset == off, (c_name, pname)
        assert getattr(cls, pname).size == size * count, (c_name, pname)
        off += size * count
    assert ctypes.sizeof(cls) == (off + 7) // 8 * 8


class _Stub:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def test_batch_prover_argument_errors():
    from snarkvm_b200 import varuna as dv
    with pytest.raises(ValueError, match="no circuits"):
        dv.BatchProver([])
    circuit = _Stub(num_variables=8)
    with pytest.raises(ValueError, match="circuit 1: instance does not match the index"):
        dv.BatchProver([(circuit, [_Stub(shape=(8, 4))]), (circuit, [_Stub(shape=(8, 4)), _Stub(shape=(7, 4))])])
    with pytest.raises(ValueError, match="circuit 0: no instances"):
        dv.BatchProver([(circuit, [])])
    p = dv.BatchProver.__new__(dv.BatchProver)                            # a prover of two circuits with 1 and 2 instances
    p.circuits, p.batch = [circuit, circuit], [1, 2]
    with pytest.raises(ValueError, match="batch combiners"):
        p.second_round([(1, [1])])
    with pytest.raises(ValueError, match="instance combiners"):
        p.third_round(2, 3, 4, [(1, [1]), (1, [1])])
    with pytest.raises(ValueError, match="δ"):
        p.fifth_round([[1, 2, 3]])
    with pytest.raises(ValueError, match="δ"):
        p.fifth_round([[1, 2, 3], [1, 2]])
