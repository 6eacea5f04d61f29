"""The structured-output kernels (csrc/structured.cu) against their numpy / torch restatement (tests/structured_double.py):
cts_struct_mask_build bit-identical on a synthetic vocabulary of random 1-8-byte tokens plus stop ids, for DFAs of 1, 37 and 4096 states;
cts_struct_mask_apply bitwise equal to torch.where on bf16 and fp16 rows with NaN / inf logits and a row stride, rows with state -1
untouched; cts_struct_advance equal to a walk on the host; the argument errors."""
import numpy as np
import pytest
import torch

from tests.gpu_util import ctx
from tests.structured_double import mask_build_reference, unpack_bits, walk

pytestmark = pytest.mark.gpu
ALPHA = np.frombuffer(b"abcdefgh01234567", dtype=np.uint8)


def _vocab(V, seed, n_empty=50):
    """Random 1-8-byte tokens over a 16-byte alphabet (so walks go deep), a few ids without bytes."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 9, size=V)
    lens[rng.choice(V, size=min(n_empty, V // 4), replace=False)] = 0
    offsets = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    data = ALPHA[rng.integers(0, len(ALPHA), size=max(int(offsets[-1]), 1))]
    return offsets, data


def _dfa(S, seed, per_state):
    """Random DFA: each state has transitions on `per_state` alphabet bytes (and one byte outside it) to random states."""
    rng = np.random.default_rng(seed)
    trans = np.full((S, 256), -1, dtype=np.int32)
    for s in range(S):
        for b in rng.choice(ALPHA, size=per_state, replace=False):
            trans[s, b] = rng.integers(0, S)
        trans[s, 200 + s % 50] = rng.integers(0, S)
    accept = rng.random(S) < 0.3
    accept[0] = S == 1 or accept[0]
    return trans, accept


def _dev(trans, accept, offsets, data, stops):
    c = torch.device("cuda")
    return (torch.from_numpy(trans).to(c), torch.from_numpy(accept.astype(np.uint8)).to(c), torch.from_numpy(offsets).to(c),
            torch.from_numpy(data).to(c), torch.tensor(stops, dtype=torch.int32, device=c))


@pytest.mark.parametrize("S,per_state", [(1, 16), (37, 12), (4096, 3)])
@pytest.mark.parametrize("V", [1000, 1003, 152064])
def test_mask_build_bit_identical(S, per_state, V):
    if S == 4096 and V != 152064:
        pytest.skip("the 4096-state automaton runs at the full vocabulary only")
    offsets, data = _vocab(V, seed=V + S)
    trans, accept = _dfa(S, seed=S, per_state=per_state)
    stops = [V - 1, 5, V // 2] if V > 10 else []
    t, a, o, d, st = _dev(trans, accept, offsets, data, stops)
    allowed = torch.full((S, (V + 31) // 32), -7, dtype=torch.int32, device="cuda")
    ctx().struct_mask_build(t, a, o, d, st, allowed)
    torch.cuda.synchronize()
    ref = mask_build_reference(trans, accept, offsets, data, stops)
    got = allowed.cpu().numpy()
    assert np.array_equal(got, ref), int((got != ref).sum())
    bits = unpack_bits(got, V)
    assert bits.any() and not bits.all()
    assert (bits[:, stops[0]] == accept).all() if stops else True
    # repeatable: the same words on a second launch
    ctx().struct_mask_build(t, a, o, d, st, allowed)
    assert np.array_equal(allowed.cpu().numpy(), got)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V,ld", [(1000, 1000), (1003, 1024), (152064, 152064)])
def test_mask_apply_matches_torch_where(dt, V, ld):
    rng = np.random.default_rng(V)
    S, B = 5, 7
    bits = rng.random((S, V)) < 0.4
    from tests.structured_double import pack_bits
    allowed = torch.from_numpy(pack_bits(bits)).cuda()
    base = torch.randn(B, ld, generator=torch.Generator().manual_seed(1)).to(dt)
    base[0, :50] = float("nan")
    base[1, 10:20] = float("inf")
    base[2, 30:40] = float("-inf")
    base[3, ::7] = float("nan")
    state = torch.tensor([0, 4, -1, 2, 3, -1, 1], dtype=torch.int32)
    logits = base.cuda()
    ctx().struct_mask_apply(logits[:, :V] if ld != V else logits, B, state.cuda(), allowed, vocab=V)
    torch.cuda.synchronize()
    got = logits.cpu()
    ref = base.clone()
    for b in range(B):
        s = int(state[b])
        if s >= 0:
            keep = torch.from_numpy(bits[s])
            ref[b, :V] = torch.where(keep, base[b, :V], torch.tensor(float("-inf"), dtype=dt))
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))              # bitwise, NaN included
    assert torch.equal(got[:, V:].view(torch.int16), base[:, V:].view(torch.int16))  # past the vocabulary: untouched


def test_struct_advance_matches_host_walk():
    V = 3000
    offsets, data = _vocab(V, seed=3)
    trans, accept = _dfa(37, seed=4, per_state=14)
    stops = [7, 2999]
    t, a, o, d, st = _dev(trans, accept, offsets, data, stops)
    rng = np.random.default_rng(5)
    B = 300
    state = rng.integers(-1, 37, size=B).astype(np.int32)
    cur = rng.integers(0, V, size=B).astype(np.int32)
    cur[:10] = 7
    cur[10:20] = 2999
    cur[20] = V + 5                                                       # outside the vocabulary: state unchanged
    s_dev = torch.from_numpy(state).cuda()
    for _ in range(3):                                                    # three steps, new tokens each time
        ctx().struct_advance(torch.from_numpy(cur).cuda(), B, s_dev, t, o, d, st)
        for b in range(B):
            s, tok = int(state[b]), int(cur[b])
            if s < 0 or tok >= V or tok in stops:
                continue
            n = walk(trans, s, data[offsets[tok]:offsets[tok + 1]])
            if n >= 0:
                state[b] = n
        assert np.array_equal(s_dev.cpu().numpy(), state)
        cur = rng.integers(0, V, size=B).astype(np.int32)


def test_argument_errors():
    from chatts_b200._cabi import CtsError
    c = ctx()
    trans, accept = _dfa(3, 0, 4)
    offsets, data = _vocab(100, 0)
    t, a, o, d, st = _dev(trans, accept, offsets, data, [1])
    with pytest.raises(CtsError):
        c.struct_mask_build(t, a, o, d, st, torch.zeros(3, 3, dtype=torch.int32, device="cuda"))          # words != ceil(V / 32)
    with pytest.raises(CtsError):
        c.struct_mask_build(t, a, o, d, torch.zeros(65, dtype=torch.int32, device="cuda"), torch.zeros(3, 4, dtype=torch.int32, device="cuda"))
    with pytest.raises(CtsError):
        c.struct_mask_apply(torch.zeros(2, 100, dtype=torch.float32, device="cuda"), 2, torch.zeros(2, dtype=torch.int32, device="cuda"),
                            torch.zeros(3, 4, dtype=torch.int32, device="cuda"))
    with pytest.raises(CtsError):
        c.struct_mask_apply(torch.zeros(2, 100, dtype=torch.bfloat16, device="cuda"), 2, torch.zeros(2, dtype=torch.int32, device="cuda"),
                            torch.zeros(3, 2, dtype=torch.int32, device="cuda"))                        # too few words
