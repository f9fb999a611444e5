"""GPU: resumable Poseidon transcripts (snarkvm_b200_poseidon_transcripts_resume_device).  Random operation lists over Fq and Fr cut
into chains of resume calls give word for word the outputs and final state of one call (and of the oracle); a fresh record equals the
entry point without state; a malformed record is refused and nothing is written."""
import random

import numpy as np
import pytest

from oracle import poseidon as op
from snarkvm_b200 import poseidon

pytestmark = pytest.mark.gpu
OPS = (poseidon.OP_ABSORB, poseidon.OP_SQUEEZE, poseidon.OP_SQUEEZE_NONNATIVE, poseidon.OP_SQUEEZE_SHORT_NONNATIVE)


def _lists(rng, field, T):
    """per transcript: a list of (kind, n), with values to absorb; directions change often, lengths cross the rate.  Every list starts
    with absorb 3 (which ends mid-rate, at index 1), squeeze 1 (a change of direction that ends at index 1 of the squeezing mode)
    and absorb 1, so that cuts at 1 and 2 store a record mid-rate and right after a change of direction."""
    p = poseidon.FIELDS[field][0]
    out = []
    for _ in range(T):
        ops = [(poseidon.OP_ABSORB, 3, [rng.randrange(p) for _ in range(3)]), (rng.choice(OPS[1:]), 1, None),
               (poseidon.OP_ABSORB, 1, [rng.randrange(p)])]
        for _k in range(rng.randrange(1, 12)):
            kind = rng.choice(OPS)
            n = rng.choice([0, 1, 1, 2, 3, 5])
            ops.append((kind, n, [rng.randrange(p) for _ in range(n)] if kind == poseidon.OP_ABSORB else None))
        out.append(ops)
    return out


def _run(field, lists, cuts, states):
    """run segment [cuts[t][s], cuts[t][s+1]) of every transcript in call s, resuming from `states` → (native, fr) per transcript"""
    import torch
    from snarkvm_b200 import device
    limbs = poseidon.FIELDS[field][2]
    T = len(lists)
    results = [([], []) for _ in range(T)]
    for s in range(max(len(c) for c in cuts) - 1):
        ops, start, ins, nout, nfr, spans = [], [0], [], 0, 0, []
        for t in range(T):
            c = cuts[t]
            seg = lists[t][c[s]: c[s + 1]] if s + 1 < len(c) else []
            for kind, n, vals in seg:
                if kind == poseidon.OP_ABSORB:
                    ops.append((kind, n, len(ins))); ins += vals
                elif kind == poseidon.OP_SQUEEZE:
                    ops.append((kind, n, nout)); spans.append((t, 0, nout, n)); nout += n
                else:
                    ops.append((kind, n, nfr)); spans.append((t, 1, nfr, n)); nfr += n
            start.append(len(ops))
        words = poseidon.to_mont_words(field, ins) if ins else np.zeros((0, limbs), dtype=np.uint32)
        out, fr = device.poseidon_transcripts(field, torch.tensor(ops, dtype=torch.int32).reshape(-1, 3).cuda(),
                                              torch.tensor(start, dtype=torch.int32).cuda(), torch.from_numpy(words.view(np.int64)).cuda(),
                                              nout, nfr, states)
        out, fr = out.cpu().numpy().view(np.uint32), fr.cpu().numpy().view(np.uint32)
        for t, which, off, n in spans:
            results[t][which].append((out if which == 0 else fr)[off: off + n].copy())
    return [tuple(np.concatenate(x) if x else None for x in r) for r in results]


def _oracle_state(field, ops):
    p, bits, _n = poseidon.FIELDS[field]
    s = op.Sponge(p, bits, poseidon.parameters(field))
    for kind, n, vals in ops:
        if kind == poseidon.OP_ABSORB:
            s.absorb_native_field_elements(vals)
        elif kind == poseidon.OP_SQUEEZE:
            s.squeeze_native_field_elements(n)
        else:
            s.get_fe(n, kind == poseidon.OP_SQUEEZE_SHORT_NONNATIVE)
    return s


@pytest.mark.parametrize("field", [poseidon.FIELD_FQ, poseidon.FIELD_FR])
def test_chains_of_resume_calls_equal_one_call(field):
    import torch
    rng = random.Random(field + 11)
    T = 96
    lists = _lists(rng, field, T)
    whole = [[0, len(ops)] for ops in lists]
    chained = []
    for ops in lists:
        # random cuts; the fixed ones mid-rate (1) and right after a change of direction (2); and right after the first later
        # operation of non-zero length that changes direction
        cut = {0, 1, 2, len(ops)} | {rng.randrange(len(ops) + 1) for _ in range(rng.randrange(4))}
        turns = [k for k in range(3, len(ops)) if ops[k][1] and (ops[k][0] == poseidon.OP_ABSORB) != (ops[k - 1][0] == poseidon.OP_ABSORB)]
        if turns:
            cut.add(turns[0] + 1)
        chained.append(sorted(cut))
    one_state = poseidon.fresh_states(field, T, "cuda")
    chain_state = poseidon.fresh_states(field, T, "cuda")
    a = _run(field, lists, whole, one_state)
    b = _run(field, lists, chained, chain_state)
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert (u is None and v is None) or (u == v).all()
    assert torch.equal(one_state, chain_state)
    # the final state is the oracle's: state elements, mode, index
    limbs = poseidon.FIELDS[field][2]
    host = one_state.cpu().numpy().view(np.uint32)
    for t, ops in enumerate(lists):
        s = _oracle_state(field, ops)
        assert poseidon.from_mont_words(field, host[t, : 3 * limbs].reshape(3, limbs)) == s.state, t
        assert list(host[t, 3 * limbs:]) == [int(s.mode[0] == "squeezing"), s.mode[1], 0, 0], t


@pytest.mark.parametrize("field", [poseidon.FIELD_FQ, poseidon.FIELD_FR])
def test_fresh_record_equals_the_stateless_entry_point(field):
    rng = random.Random(field + 21)
    lists = _lists(rng, field, 64)
    whole = [[0, len(ops)] for ops in lists]
    a = _run(field, lists, whole, None)
    b = _run(field, lists, whole, poseidon.fresh_states(field, 64, "cuda"))
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert (u is None and v is None) or (u == v).all()


@pytest.mark.parametrize("field", [poseidon.FIELD_FQ, poseidon.FIELD_FR])
@pytest.mark.parametrize("defect", ["element", "mode", "index"])
def test_malformed_record_is_refused(field, defect):
    import torch
    from snarkvm_b200 import CudaError, device
    p, _bits, limbs = poseidon.FIELDS[field]
    T = 8
    states = poseidon.fresh_states(field, T, "cuda")
    _run(field, [[(poseidon.OP_ABSORB, 3, [5, 6, 7])]] * T, [[0, 1]] * T, states)
    host = states.cpu().numpy().view(np.uint32).copy()
    for t in (3, 6):
        if defect == "element":
            host[t, limbs: 2 * limbs] = np.frombuffer(p.to_bytes(4 * limbs, "little"), dtype=np.uint32)
        elif defect == "mode":
            host[t, 3 * limbs] = 2
        else:
            host[t, 3 * limbs + 1] = poseidon.RATE + 1
    bad = torch.from_numpy(host.view(np.int64)).cuda()
    before = bad.clone()
    ops = torch.tensor([[poseidon.OP_SQUEEZE, 2, 2 * t] for t in range(T)], dtype=torch.int32).cuda()
    with pytest.raises(CudaError) as ei:
        device.poseidon_transcripts(field, ops, torch.arange(T + 1, dtype=torch.int32).cuda(),
                                    torch.zeros((0, limbs // 2), dtype=torch.int64).cuda(), 2 * T, 0, bad)
    assert ei.value.transcript == 3
    assert torch.equal(bad, before)
