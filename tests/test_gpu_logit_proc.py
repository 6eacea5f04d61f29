"""The logits-processor kernels (csrc/logit_proc.cu) against their torch statement (tests/logit_proc_double.py): cts_logit_proc_apply bit
for bit (NaN as NaN) at V = 1000, 1003 and 152 064, batch 1, 5 and 32, bf16 and fp16, with a row stride, NaN / +-inf logits, neutral and
active rows mixed, a shared and a per-row bias row, allowed-id masks, min_tokens stop ids, uint16 counts above 32 767; with only the
repetition penalty set, bit-identical to cts_rep_penalty_apply; cts_logit_proc_update over 200 steps equal to bincount; argument
errors."""
import pytest
import torch

from tests.gpu_util import ctx
from tests.logit_proc_double import apply_reference, unpack_seen, update_reference

pytestmark = pytest.mark.gpu


def _same(a, b):
    """Bitwise equal, except that a NaN only has to be a NaN (torch and CUDA write different NaN patterns)."""
    na, nb = a.isnan(), b.isnan()
    return torch.equal(na, nb) and torch.equal(a.view(torch.int16)[~na], b.view(torch.int16)[~nb])


def _case(B, V, dt, seed, ld=None, neutral_every=3):
    g = torch.Generator().manual_seed(seed)
    ld = V if ld is None else ld
    lg = (torch.randn(B, ld, generator=g) * 5).to(dt)
    for b in range(B):
        lg[b, torch.randint(0, V, (3,), generator=g)] = float("nan")
        lg[b, torch.randint(0, V, (3,), generator=g)] = float("inf")
        lg[b, torch.randint(0, V, (3,), generator=g)] = float("-inf")
    lg[:, 0] = -0.0
    rep = torch.tensor([[1.0, 1.3, 0.7, 2.0][b % 4] for b in range(B)])
    pres = torch.tensor([[0.0, 0.5, -1.5, 2.0, 0.0][b % 5] for b in range(B)])
    freq = torch.tensor([[0.0, 0.25, 0.0, -2.0, 1.0, 0.3][b % 6] for b in range(B)])
    seen = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, (V + 31) // 32), generator=g, dtype=torch.int64).to(torch.int32)
    counts = torch.randint(0, 4, (B, V), generator=g, dtype=torch.int32)
    counts[:, :64] = torch.randint(0, 65536, (B, 64), generator=g, dtype=torch.int32)
    counts = counts.to(torch.int16)
    bias = torch.zeros(1 + B, V)
    bias[0, torch.randint(0, V, (20,), generator=g)] = torch.randn(20, generator=g) * 10
    for b in range(B):
        bias[1 + b, torch.randint(0, V, (10,), generator=g)] = torch.randn(10, generator=g) * 10
        if b % 2:
            off = torch.rand(V, generator=g) < 0.7                          # allowed_token_ids: 30 % of the vocabulary
            bias[1 + b, off] = float("-inf")
    bias_row = torch.tensor([[-1, 0, 1 + b, 0][b % 4] for b in range(B)], dtype=torch.int32)
    n_gen = torch.randint(0, 6, (B,), generator=g, dtype=torch.int32)
    min_tok = torch.tensor([[0, 3, 10, 4, 0][b % 5] for b in range(B)], dtype=torch.int32)
    stops = torch.full((B, 5), -1, dtype=torch.int32)
    for b in range(B):
        k = b % 4 + 1
        stops[b, :k] = torch.randint(0, V, (k,), generator=g)
    stops[0, 0] = V - 1
    for b in range(0, B, neutral_every):                                    # neutral rows
        rep[b], pres[b], freq[b], bias_row[b], min_tok[b] = 1.0, 0.0, 0.0, -1, 0
    cuda = lambda *ts: [t.cuda() for t in ts]
    return cuda(lg, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("B", [1, 5, 32])
@pytest.mark.parametrize("V", [1000, 1003, 152064])
def test_apply_matches_statement(V, B, dt):
    lg, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops = _case(B, V, dt, V + B)
    orig, want = lg.clone(), lg.clone()
    apply_reference(want, B, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops, V)
    ctx().logit_proc_apply(lg, B, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops, vocab=V)
    torch.cuda.synchronize()
    assert _same(lg.cpu(), want.cpu())
    assert torch.equal(lg[0].view(torch.int16), orig[0].view(torch.int16))                     # a neutral row is not written
    if B > 1:
        assert not torch.equal(lg[1].view(torch.int16), orig[1].view(torch.int16))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V,ld", [(1000, 1024), (1003, 1011), (1003, 1003)])
def test_row_stride_and_optional_tables(V, ld, dt):
    """ld > V leaves the columns past V alone; no counts, no bias table and no stop ids are valid arguments."""
    B = 5
    lg, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops = _case(B, V, dt, 7, ld=ld, neutral_every=2)
    for cnt, bs, st in ((counts, bias, stops), (None, None, None), (None, bias[:1], stops[:, :1].contiguous())):
        x, want = lg.clone(), lg.clone()
        br = bias_row.clamp(max=0) if bs is not None and bs.shape[0] == 1 else bias_row
        apply_reference(want, B, rep, pres, freq, seen, cnt, bs, br, n_gen, min_tok, st, V)
        ctx().logit_proc_apply(x, B, rep, pres, freq, seen, cnt, bs, br, n_gen, min_tok, st, vocab=V)
        torch.cuda.synchronize()
        assert _same(x.cpu(), want.cpu()) and torch.equal(x[:, V:].view(torch.int16), lg[:, V:].view(torch.int16))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [1000, 1003, 152064])
def test_rep_only_equals_rep_penalty_apply(V, dt):
    B = 5
    lg, _, _, _, seen, *_ = _case(B, V, dt, 3)
    c = ctx()
    z = torch.zeros(B, device="cuda")
    neg = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    zi = torch.zeros(B, dtype=torch.int32, device="cuda")
    for p in (1.3, 0.6):
        a, b = lg.clone(), lg.clone()
        c.rep_penalty_apply(a, B, seen, p)
        c.logit_proc_apply(b, B, torch.full((B,), p, device="cuda"), z, z, seen, None, None, neg, zi, zi, None)
        torch.cuda.synchronize()
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("V", [1000, 1003, 152064])
def test_update_over_200_steps_equals_bincount(V):
    B = 5
    g = torch.Generator().manual_seed(V)
    ids = torch.randint(0, 40, (200, B), generator=g, dtype=torch.int32)
    ids[::7, 1] = -1
    ids[::5, 2] = V
    ids[:, 3] = V - 1
    seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32, device="cuda")
    counts = torch.zeros(B, V, dtype=torch.int16, device="cuda")
    n_gen = torch.zeros(B, dtype=torch.int32, device="cuda")
    seen_r, counts_r, n_r = seen.clone().cpu(), counts.clone().cpu(), n_gen.clone().cpu()
    for s in range(200):
        cur = ids[s].cuda()
        ctx().logit_proc_update(cur, B, seen, counts, n_gen, V)
        update_reference(ids[s], B, seen_r, counts_r, n_r, V)
    torch.cuda.synchronize()
    for b in range(B):
        ok = ids[:, b][(ids[:, b] >= 0) & (ids[:, b] < V)].long()
        assert torch.equal(counts[b].cpu().long(), torch.bincount(ok, minlength=V))
        assert torch.equal(unpack_seen(seen[b:b + 1].cpu(), V)[0], torch.bincount(ok, minlength=V) > 0)
        assert int(n_gen[b]) == len(ok)
    assert torch.equal(seen.cpu(), seen_r) and torch.equal(counts.cpu(), counts_r) and torch.equal(n_gen.cpu(), n_r)
    ctx().logit_proc_update(ids[0].cuda(), B, seen, None, n_gen, V)          # without counts
    torch.cuda.synchronize()


def test_argument_errors():
    from chatts_b200._cabi import CtsError
    c = ctx()
    B, V = 2, 100
    lg, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops = _case(B, V, torch.bfloat16, 1)
    with pytest.raises(CtsError):
        c.logit_proc_apply(lg.float(), B, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops)
    with pytest.raises(CtsError):
        c.logit_proc_apply(lg, B, rep, pres, freq, seen[:, :3], counts, bias, bias_row, n_gen, min_tok, stops)      # too few words
    with pytest.raises(CtsError):
        c.logit_proc_apply(lg, B, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok,
                           torch.full((B, 65), -1, dtype=torch.int32, device="cuda"))                                  # > 64 stop ids
    with pytest.raises(CtsError):
        c.logit_proc_apply(lg, B, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops, vocab=V + 1)  # ld < vocab
    with pytest.raises(CtsError):
        c.logit_proc_update(torch.zeros(B, dtype=torch.int32, device="cuda"), B, seen[:, :3], counts, n_gen, V)
    for kw in (dict(bias_row=bias_row.long()), dict(rep=rep.double()), dict(counts=counts.int()), dict(stops=stops[:, :2]),
               dict(bias=torch.zeros(3, V + 8, device="cuda")), dict(counts=torch.zeros(B, V + 8, dtype=torch.int16, device="cuda")),
               dict(n_gen=n_gen[:1])):                  # wrong dtype, non-contiguous, rows wider than vocab, too few rows
        a = {**dict(rep=rep, bias_row=bias_row, counts=counts, stops=stops, bias=bias, n_gen=n_gen), **kw}
        with pytest.raises(CtsError):
            c.logit_proc_apply(lg, B, a["rep"], pres, freq, seen, a["counts"], a["bias"], a["bias_row"], a["n_gen"], min_tok, a["stops"])
    with pytest.raises(CtsError):
        c.logit_proc_update(torch.zeros(B, dtype=torch.int64, device="cuda"), B, seen, counts, n_gen, V)
    c.logit_proc_apply(lg, 0, rep, pres, freq, seen, counts, bias, bias_row, n_gen, min_tok, stops)                   # batch 0: no-op
    torch.cuda.synchronize()
