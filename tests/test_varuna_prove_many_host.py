"""CPU: the ctypes images of the segment tables varuna.prove_batch_many adds (include/snarkvm_b200.h), and its argument checks that
raise before anything reaches a device."""
import ctypes
import re

import pytest

from test_varuna_batch_host import _C_SIZE, _c_struct_fields


@pytest.mark.parametrize("c_name, py_name", [("snarkvm_b200_round4_batch_segment_t", "Round4BatchSegment"),
                                             ("snarkvm_b200_poly_eval_segment_t", "PolyEvalSegment"),
                                             ("snarkvm_b200_poly_divide_segment_t", "PolyDivideSegment")])
def test_structs_match_the_header(c_name, py_name):
    """same members in the same order at the same offsets (natural alignment, as the C compiler lays them out)"""
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


def test_prove_batch_many_argument_errors():
    from snarkvm_b200 import varuna as dv
    with pytest.raises(ValueError, match="EmptyBatch: no jobs"):
        dv.prove_batch_many([])
    import torch
    d = _Stub(size=1)
    pk = _Stub(circuit=_Stub(num_variables=8, a=_Stub(row_ptr=torch.zeros(1)), constraint_domain=d, variable_domain=d,
                             max_non_zero_domain=d), committer_key=None)      # a one-circuit job that passes the host checks
    z = torch.zeros((8, 4), dtype=torch.int64)
    with pytest.raises(ValueError, match="job 0: EmptyBatch: no circuits"):
        dv.prove_batch_many([[]])
    with pytest.raises(ValueError, match="job 1: circuit 0: no instances"):
        dv.prove_batch_many([[(pk, [z])], [(pk, [])], [(pk, [])]])
    with pytest.raises(ValueError, match="job 2: circuit 0: instance does not match the index"):
        dv.prove_batch_many([[(pk, [z])]] * 2 + [[(pk, [z[:7]])]])
    with pytest.raises(ValueError, match="1 rngs for 2 jobs"):
        dv.prove_batch_many([[(pk, [z])]] * 2, True, [object()])
    with pytest.raises(ValueError, match="job 0: EmptyBatch"):
        dv.prove_batch([])
