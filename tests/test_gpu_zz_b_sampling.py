"""cts_sample_advance (csrc/sampling.cu) against its CPU statement (tests/cabi_double.py ``sample_reference``, itself checked
against transformers' logits warpers in tests/test_host_sampling.py)."""
import numpy as np
import pytest
import torch

from tests.cabi_double import TorchDouble
from tests.gpu_util import ctx, record

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("vocab,dtype", [(1000, torch.bfloat16), (151936, torch.bfloat16), (1003, torch.bfloat16), (4096, torch.float16)])
@pytest.mark.parametrize("top_k,top_p,temp", [(0, 0.9, 0.7), (20, 1.0, 1.0), (50, 0.8, 0.2), (0, 1.0, 1.3)])
def test_sample_advance_matches_reference(vocab, dtype, top_k, top_p, temp):
    c = ctx()
    B, page, max_pages = 5, 16, 8
    g = torch.Generator().manual_seed(vocab + top_k)
    logits = (torch.randn(B, vocab, generator=g) * 3).to(dtype)
    out = torch.full((B, 8), -1, dtype=torch.int32, device="cuda")
    step_ptr = torch.tensor([2, 0], dtype=torch.int32, device="cuda")
    cur = torch.zeros(B, dtype=torch.int32, device="cuda")
    pos = torch.tensor([3, 15, 16, 31, 40], dtype=torch.int32, device="cuda")
    sl = pos + 1
    slot = torch.zeros(B, dtype=torch.int32, device="cuda")
    pt = torch.arange(B * max_pages, dtype=torch.int32).view(B, max_pages).cuda()
    c.sample_advance(logits.cuda(), B, temp, top_k, top_p, 1234, out, step_ptr, cur, pos, sl, slot, pt, page)
    torch.cuda.synchronize()
    toks = out[:, 2].cpu().tolist()
    exact, near = 0, 0
    for b in range(B):
        ref, cdf, target, kept = TorchDouble.sample_reference(logits[b], temp, top_k, top_p, 1234, 2, b)
        assert 0 <= toks[b] < vocab and kept[toks[b]], (b, toks[b])
        if toks[b] == ref:
            exact += 1
        else:       # fp32 vs fp64 prefix sums: allowed only when the target sits on a CDF boundary of the chosen token
            lo = cdf[toks[b] - 1] if toks[b] > 0 else 0.0
            assert min(abs(target - lo), abs(target - cdf[toks[b]])) < 1e-4 * cdf[-1], (b, toks[b], ref)
            near += 1
    record("sample_advance", vocab=vocab, top_k=top_k, top_p=top_p, temp=temp, exact=exact, boundary=near)
    assert exact >= B - 1
    assert step_ptr.cpu().tolist() == [3, 0] and cur.cpu().tolist() == toks
    p2 = (pos.cpu() % page).tolist()
    assert pos.cpu().tolist() == [4, 16, 17, 32, 41] and sl.cpu().tolist() == [5, 17, 18, 33, 42]
    assert slot.cpu().tolist() == [int(pt[b, pos.cpu()[b] // page]) * page + p2[b] for b in range(B)]


def test_sample_advance_is_reproducible_and_distributed_right():
    c = ctx()
    vocab, B = 1000, 32
    g = torch.Generator().manual_seed(0)
    row = (torch.randn(vocab, generator=g) * 2).to(torch.bfloat16)
    logits = row[None].repeat(B, 1).cuda()
    draws = []
    for step in range(40):
        out = torch.zeros(B, 64, dtype=torch.int32, device="cuda")
        sp = torch.tensor([step, 0], dtype=torch.int32, device="cuda")
        c.sample_advance(logits, B, 1.0, 0, 0.95, 99, out, sp, None, None, None, None, None, 16)
        draws.append(out[:, step].cpu())
    out2 = torch.zeros(B, 64, dtype=torch.int32, device="cuda")
    c.sample_advance(logits, B, 1.0, 0, 0.95, 99, out2, torch.tensor([39, 0], dtype=torch.int32, device="cuda"), None, None, None, None, None, 16)
    assert torch.equal(out2[:, 39].cpu(), draws[-1])
    d = torch.cat(draws).numpy()
    _, cdf, _, kept = TorchDouble.sample_reference(row, 1.0, 0, 0.95, 99, 0, 0)
    assert kept[d].all()
    p = np.diff(np.concatenate([[0.0], cdf])) / cdf[-1]
    top = int(np.argmax(p))
    n = d.shape[0]
    assert abs((d == top).mean() - p[top]) < 4 * np.sqrt(p[top] * (1 - p[top]) / n) + 0.01


@pytest.mark.parametrize("vocab,dtype", [(1000, torch.bfloat16), (151936, torch.float16), (1003, torch.bfloat16)])
def test_repetition_penalty_kernels_match_the_statement(vocab, dtype):
    """cts_rep_penalty_mark / _apply against tests/cabi_double.py (itself equal to transformers' RepetitionPenaltyLogitsProcessor,
    tests/test_host_sampling.py): bit-exact logits, repeated tokens penalised once, rows independent."""
    c, dbl = ctx(), TorchDouble()
    g = torch.Generator().manual_seed(vocab)
    B, W = 4, (vocab + 31) // 32
    logits = (torch.randn(B, vocab, generator=g) * 4).to(dtype)
    toks = torch.randint(0, vocab, (B * 40,), generator=g).to(torch.int32)
    toks[:5] = toks[5]                                            # repeats
    toks[7] = vocab - 1
    rows = torch.arange(B).repeat_interleave(40).to(torch.int32)
    seen_ref = torch.zeros(B, W, dtype=torch.int32)
    dbl.rep_penalty_mark(toks, rows, seen_ref, vocab)
    new = torch.randint(0, vocab, (B,), generator=g).to(torch.int32)
    dbl.rep_penalty_mark(new, None, seen_ref, vocab)
    want = logits.clone()
    dbl.rep_penalty_apply(want, B, seen_ref, 1.25)
    seen = torch.zeros(B, W, dtype=torch.int32, device="cuda")
    c.rep_penalty_mark(toks.cuda(), rows.cuda(), seen, vocab)
    c.rep_penalty_mark(new.cuda(), None, seen, vocab)
    got = logits.clone().cuda()
    c.rep_penalty_apply(got, B, seen, 1.25)
    torch.cuda.synchronize()
    assert torch.equal(seen.cpu(), seen_ref) and torch.equal(got.cpu(), want)
