"""cts_logprobs (csrc/sampling.cu) against log_softmax of the same 16-bit logits, computed in float64 and rounded to fp32
(tests/logprobs_double.py; torch's fp32 log_softmax on the CPU is itself up to ~2e-5 off at V = 152k): logprobs within 1e-5,
ranks and top-k ids exact under the tie rule (value descending, then the smaller id)."""
import pytest
import torch

from tests.gpu_util import ctx
from tests.logprobs_double import logprobs_reference

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _run(c, logits, chosen, k, vocab=None, out_ld=1, step_ptr=None):
    R = logits.shape[0]
    vocab = logits.shape[-1] if vocab is None else vocab
    lp = torch.full((R, out_ld), -7.0, dtype=torch.float32, device="cuda")
    rank = torch.full((R, out_ld), -7, dtype=torch.int32, device="cuda")
    ids = torch.full((R, out_ld, max(k, 1)), -7, dtype=torch.int32, device="cuda")
    vals = torch.full((R, out_ld, max(k, 1)), -7.0, dtype=torch.float32, device="cuda")
    ws = torch.empty(max(c.logprobs_workspace_floats(R, vocab, k), 2), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(R, dtype=torch.int32, device="cuda")
    c.logprobs(logits, R, chosen, k, lp, rank, ids, vals, ws, cnt, step_ptr=step_ptr, vocab=vocab)
    torch.cuda.synchronize()
    assert int(cnt.abs().sum()) == 0, "arrival counters not reset"
    return lp.cpu(), rank.cpu(), ids[:, :, :k].cpu(), vals[:, :, :k].cpu()


def _maxabs(d):
    return float(d.abs().max()) if d.numel() else 0.0


def _check(got, ref):
    lp, rank, ids, vals = got
    rlp, rrank, rids, rvals = ref
    assert torch.equal(torch.isnan(lp), torch.isnan(rlp))
    ok = ~torch.isnan(rlp)
    assert _maxabs(lp[ok] - rlp[ok]) <= TOL
    assert torch.equal(rank, rrank)
    assert torch.equal(ids, rids)
    fin = torch.isfinite(rvals)
    assert torch.equal(fin, torch.isfinite(vals)) and torch.equal(torch.isnan(vals), torch.isnan(rvals))
    assert _maxabs(vals[fin] - rvals[fin]) <= TOL
    return _maxabs(lp[ok] - rlp[ok])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("k", [0, 1, 5, 20])
@pytest.mark.parametrize("rows", [1, 5, 33, 128])
@pytest.mark.parametrize("vocab", [1000, 1003, 151936, 152064])
def test_logprobs_match_log_softmax(vocab, rows, k, dtype):
    c = ctx()
    g = torch.Generator().manual_seed(vocab * 131 + rows * 7 + k)
    logits = (torch.randn(rows, vocab, generator=g) * 4).to(dtype)
    chosen = torch.randint(0, vocab, (rows, 1), generator=g, dtype=torch.int32)
    chosen[0, 0] = int(logits[0].float().argmax())
    got = _run(c, logits.cuda(), chosen.cuda(), k)
    ref = logprobs_reference(logits, chosen[:, 0], k)
    _check(tuple(t[:, 0] for t in got), ref)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("vocab,pad", [(1000, 13), (152064, 64), (151936, 1)])
def test_logprobs_row_stride(vocab, pad, dtype):
    """ld > vocab (odd strides take the scalar loads); the columns past vocab hold values that would win if read."""
    c = ctx()
    g = torch.Generator().manual_seed(vocab + pad)
    full = (torch.randn(7, vocab + pad, generator=g) * 3).to(dtype)
    full[:, vocab:] = 100.0
    chosen = torch.randint(0, vocab, (7, 1), generator=g, dtype=torch.int32)
    got = _run(c, full.cuda(), chosen.cuda(), 20, vocab=vocab)
    _check(tuple(t[:, 0] for t in got), logprobs_reference(full[:, :vocab], chosen[:, 0], 20))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("vocab", [1003, 152064])
def test_logprobs_ties_and_non_finite(vocab, dtype):
    """Many equal values (ids break the ties, across slice boundaries), -0 next to +0, -inf entries, NaN entries, a row that is -inf
    except one entry, a row of NaN except two, a NaN chosen logit and an out-of-range chosen id."""
    c = ctx()
    g = torch.Generator().manual_seed(vocab)
    R = 8
    x = torch.randint(-3, 4, (R, vocab), generator=g).float()
    x[1, ::7] = float("-inf")
    x[2, ::5] = float("nan")
    x[3] = float("-inf")
    x[3, vocab // 2] = 1.5
    x[4] = float("nan")
    x[4, 3], x[4, vocab - 1] = 2.0, 2.0
    x[5, :: 3] = -0.0
    x[5, 1:: 3] = 0.0
    x[6, 100:] = float("nan")
    logits = x.to(dtype)
    chosen = torch.randint(0, vocab, (R, 1), generator=g, dtype=torch.int32)
    chosen[2, 0] = 10                     # NaN chosen logit
    chosen[3, 0] = vocab // 2
    chosen[4, 0] = vocab - 1
    chosen[6, 0] = vocab + 5              # outside the row
    chosen[7, 0] = 0
    got = tuple(t[:, 0] for t in _run(c, logits.cuda(), chosen.cuda(), 20))
    ref = logprobs_reference(logits, chosen[:, 0], 20)
    _check(got, ref)
    assert torch.isnan(got[0][2]) and torch.isnan(got[0][6]) and int(got[1][2]) == 0
    assert float(got[0][3]) == 0.0 and int(got[1][3]) == 1
    assert got[2][4, :2].tolist() == [3, vocab - 1] and (got[2][4, 2:] == -1).all() and torch.isnan(got[3][4, 2:]).all()


@pytest.mark.parametrize("vocab", [1000, 152064])
def test_logprobs_column_mode(vocab):
    """With step_ptr, the chosen id and the outputs sit at column step_ptr[0] - 1; every other column is untouched."""
    c = ctx()
    g = torch.Generator().manual_seed(5)
    R, ld, k = 5, 6, 5
    logits = (torch.randn(R, vocab, generator=g) * 3).bfloat16()
    chosen = torch.randint(0, vocab, (R, ld), generator=g, dtype=torch.int32)
    step_ptr = torch.tensor([3, 0], dtype=torch.int32, device="cuda")
    lp, rank, ids, vals = _run(c, logits.cuda(), chosen.cuda(), k, out_ld=ld, step_ptr=step_ptr)
    _check((lp[:, 2], rank[:, 2], ids[:, 2], vals[:, 2]), logprobs_reference(logits, chosen[:, 2], k))
    others = [j for j in range(ld) if j != 2]
    assert (lp[:, others] == -7.0).all() and (rank[:, others] == -7).all() and (ids[:, others] == -7).all()
    assert step_ptr.cpu().tolist() == [3, 0]


def test_logprobs_repeatable_and_graph_replay():
    """Two eager launches give the same bits, and so do the replays of a captured launch (the arrival counters reset themselves)."""
    c = ctx()
    g = torch.Generator().manual_seed(9)
    R, V, k = 8, 152064, 20
    logits = (torch.randn(R, V, generator=g) * 4).bfloat16().cuda()
    chosen = torch.randint(0, V, (R, 1), generator=g, dtype=torch.int32).cuda()
    a = _run(c, logits, chosen, k)
    b = _run(c, logits, chosen, k)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    lp = torch.zeros(R, 1, device="cuda"); rank = torch.zeros(R, 1, dtype=torch.int32, device="cuda")
    ids = torch.zeros(R, 1, k, dtype=torch.int32, device="cuda"); vals = torch.zeros(R, 1, k, device="cuda")
    ws = torch.empty(c.logprobs_workspace_floats(R, V, k), device="cuda")
    cnt = torch.zeros(R, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c.logprobs(logits, R, chosen, k, lp, rank, ids, vals, ws, cnt)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.logprobs(logits, R, chosen, k, lp, rank, ids, vals, ws, cnt)
    for _ in range(3):
        lp.zero_(); ids.zero_()
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip((lp.cpu(), rank.cpu(), ids.cpu(), vals.cpu()), a):
            assert torch.equal(x, y)
    assert int(cnt.abs().sum()) == 0


def test_logprobs_argument_errors():
    from chatts_b200._cabi import CtsError
    c = ctx()
    logits = torch.zeros(2, 64, dtype=torch.bfloat16, device="cuda")
    ch = torch.zeros(2, 1, dtype=torch.int32, device="cuda")
    lp = torch.zeros(2, 1, device="cuda"); rank = torch.zeros(2, 1, dtype=torch.int32, device="cuda")
    ids = torch.zeros(2, 1, 21, dtype=torch.int32, device="cuda"); vals = torch.zeros(2, 1, 21, device="cuda")
    ws = torch.zeros(c.logprobs_workspace_floats(2, 64, 21) + 2, device="cuda")
    cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    for k in (21, -1):
        with pytest.raises(CtsError):
            c.logprobs(logits, 2, ch, k, lp, rank, ids, vals, ws, cnt)
    with pytest.raises(CtsError):                       # vocab past the row stride
        c.logprobs(logits, 2, ch, 1, lp, rank, ids, vals, ws, cnt, vocab=65)
    with pytest.raises(CtsError):                       # chosen outputs without chosen ids
        c.logprobs(logits, 2, None, 1, lp, rank, ids, vals, ws, cnt)
    with pytest.raises(CtsError):
        c.logprobs(logits.float(), 2, ch, 1, lp, rank, ids, vals, ws, cnt)
    with pytest.raises(CtsError):
        c.logprobs(logits, 2, ch, 1, lp, rank, ids, vals, None, cnt)
    with pytest.raises(CtsError):
        c.logprobs(logits, 2, ch, 1, lp, rank, ids, vals, ws, None)
    assert c.logprobs_workspace_floats(0, 64, 1) == 0
