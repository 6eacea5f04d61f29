"""cts_peer_greedy_advance and cts_peer_allreduce_residual_rmsnorm (csrc/allreduce.cu) on ONE GPU: the W "ranks" are W streams of this
process and their symmetric tables W plain allocations (the technique of test_gpu_zz_f_peer_ll.py -- to the kernels a peer is only a
pointer), so the pushes, flags, epochs and merges run as they do over NVLink, minus the link.

The W grids of a call spin on each other and therefore must be co-resident: greedy W x batch <= 128 CTAs of 1024 threads, all-reduce
W x C x T <= 128 CTAs of 128 threads (C: the cluster width the entry point picks from h).  Every call launches all W ranks and then
synchronizes the device before the next call: the candidate table of the greedy kernel is not double-buffered, and in the model the
all-reduces of the next step are what order two greedy calls across ranks.

Expected values.  Greedy: cts_greedy_advance on the concatenated row with its own copy of the decode state (bit-identical state on
every rank), and the rule stated here from the fp32 row: the smallest index holding the maximum over the non-NaN entries, token 0 when
no entry is greater than -inf.  All-reduce: the step-by-step sum of test_gpu_zz_f_peer_ll.py (splits in split order, ranks in rank
order, h = dtype(resid + dtype(sum))) bit for bit, cts_peer_allreduce_ll on the same inputs bit for bit, and norm_out within 2 ulps
of the model dtype of the fp64 RMSNorm of h."""
import contextlib

import pytest
import torch

from tests.gpu_util import ctx, record
from tests.test_gpu_zz_f_peer_ll import _expected
from tests.test_gpu_zz_f_peer_ll import _Ranks as _LLRanks

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]
WORLDS = [1, 2, 4, 8]
W_IDS = [f"W{w}" for w in WORLDS]


def _on(streams, r):
    """Rank r's stream (a single rank runs on the current one)."""
    return torch.cuda.stream(streams[r]) if streams else contextlib.nullcontext()


# ---------------------------------------------------------------------------------------------------------------------------------
# cts_peer_greedy_advance
# ---------------------------------------------------------------------------------------------------------------------------------
PAGE, MAX_PAGES, OUT_LD = 2, 3, 4
STATE = ("out_tokens", "step_ptr", "cur_ids", "positions", "seq_lens", "slot_map", "page_table")


class _GreedyRanks:
    """W ranks of the vocab-parallel greedy step, laid out as tp.PeerBuffers does: per rank a candidate table float2 [W][max_b] and a
    flag table int32 [W][max_b] (zeroed), the int64 pointer arrays every rank passes, and the rank's own state int32[2] and stream."""

    def __init__(self, c, W, max_b):
        self.c, self.W, self.max_b = c, W, max_b
        self.cand = [torch.zeros(W, max_b, 2, dtype=torch.float32, device="cuda") for _ in range(W)]
        self.flags = [torch.zeros(W, max_b, dtype=torch.int32, device="cuda") for _ in range(W)]
        self.cand_ptrs = torch.tensor([t.data_ptr() for t in self.cand], dtype=torch.int64, device="cuda")
        self.flag_ptrs = torch.tensor([t.data_ptr() for t in self.flags], dtype=torch.int64, device="cuda")
        self.state = [torch.zeros(2, dtype=torch.int32, device="cuda") for _ in range(W)]
        self.streams = [torch.cuda.Stream() for _ in range(W)] if W > 1 else None

    def call(self, shards, batch, dec):
        """shards[r]: rank r's logits [batch, vshard]; dec[r]: rank r's decode state (advanced in place)."""
        torch.cuda.synchronize()
        for r in range(self.W):
            d = dec[r]
            with _on(self.streams, r):
                self.c.peer_greedy_advance(shards[r], batch, r, self.W, self.cand_ptrs, self.flag_ptrs, self.state[r], self.max_b,
                                           d["out_tokens"], d["step_ptr"], d["cur_ids"], d["positions"], d["seq_lens"], d["slot_map"],
                                           d["page_table"], PAGE)
        torch.cuda.synchronize()


def _decode_state(max_b, g):
    """Initial decode state of max_b rows.  Row 0 sits one position before the last page: its three steps cross into page 2, stay
    there, then pass the last page (slot -1)."""
    pos = torch.randint(0, PAGE * MAX_PAGES - 1, (max_b,), generator=g, dtype=torch.int32)
    pos[0] = PAGE * (MAX_PAGES - 1) - 1
    return dict(out_tokens=torch.full((max_b, OUT_LD), -1, dtype=torch.int32), step_ptr=torch.zeros(2, dtype=torch.int32),
                cur_ids=torch.full((max_b,), -2, dtype=torch.int32), positions=pos, seq_lens=pos + 1,
                slot_map=torch.full((max_b,), -3, dtype=torch.int32),
                page_table=torch.randperm(max_b * MAX_PAGES, generator=g).to(torch.int32).view(max_b, MAX_PAGES))


def _on_device(state):
    return {k: v.clone().cuda() for k, v in state.items()}


def _rule(x):
    """Greedy token of every row of the fp32 logits x [B, V]: the smallest index holding the maximum over the non-NaN entries; 0 when
    no entry is greater than -inf."""
    y = torch.where(torch.isnan(x), torch.full_like(x, float("-inf")), x)
    m = y.max(dim=1, keepdim=True).values
    out = []
    for b in range(x.shape[0]):
        hit = torch.nonzero((y[b] == m[b]) & (m[b] > float("-inf")))
        out.append(int(hit[0]) if hit.numel() else 0)
    return out


# rows whose maximum sits where a vocab-parallel argmax goes wrong; every one has an entry greater than -inf
PLANTED = ["random", "tie_across_ranks", "max_last_of_last_rank", "max_first_of_other_rank", "tie_inside_shard", "signed_zero_max",
           "inf_in_two_shards", "nan_before_max", "nan_shard", "neg_inf_shard", "one_finite_entry"]
# rows with no entry greater than -inf: the single-GPU step emits token 0
NO_CANDIDATE = ["all_neg_inf", "all_nan", "neg_inf_and_nan"]


def _plant(x, kind, W, vs, g):
    """Writes row kind `kind` into the fp32 row x of W shards of vs entries (x holds random values in about [-12, 12])."""
    V, top, last = W * vs, 16.0, (W - 1) * vs            # last: first index of the last rank
    nan, inf = float("nan"), float("inf")
    if kind == "tie_across_ranks":                        # the last entry of one rank and the first of the next: the lower index wins
        j = (W // 2) * vs if W > 1 else V - 1
        x[j - 1] = x[j] = top
    elif kind == "max_last_of_last_rank":
        x[V - 1] = top
    elif kind == "max_first_of_other_rank":
        x[last] = top
    elif kind == "tie_inside_shard":                      # two indices of one shard owned by different threads
        x[last + vs // 3] = x[last + vs - 1] = top
    elif kind == "signed_zero_max":                       # -0.0 == +0.0: the lower index wins whatever its sign
        x.copy_(-1.0 - x.abs())
        x[vs // 2] = -0.0
        x[last + vs - 1] = 0.0
    elif kind == "inf_in_two_shards":
        x[vs // 2] = inf
        x[last + 1] = inf
    elif kind == "nan_before_max":                        # NaN never wins, however early it comes
        x[torch.rand(V, generator=g) < 0.05] = nan
        for s in range(W):
            x[s * vs:s * vs + 2] = nan
        x[last + vs - 1] = top
    elif kind == "nan_shard":                             # one shard entirely NaN, the others finite
        x[:vs if W > 1 else vs // 2] = nan
    elif kind == "neg_inf_shard":                         # one shard entirely -inf, the others finite
        x[last if W > 1 else vs // 2:] = -inf
    elif kind == "one_finite_entry":
        x.fill_(-inf)
        x[last + vs // 2] = -60000.0
    elif kind == "all_neg_inf":
        x.fill_(-inf)
    elif kind == "all_nan":
        x.fill_(nan)
    elif kind == "neg_inf_and_nan":
        x.copy_(torch.where(torch.rand(V, generator=g) < 0.5, torch.full_like(x, -inf), torch.full_like(x, nan)))
    else:
        assert kind == "random", kind


def _greedy_step(c, R, ref, dec, W, vs, batch, dt, kinds, g, step):
    """One step: rows of the given kinds, all W ranks, cts_greedy_advance on the whole rows; checks tokens and state on every rank."""
    x = torch.randn(batch, W * vs, generator=g) * 3.0
    for b in range(batch):
        _plant(x[b], kinds[b], W, vs, g)
    xd = x.to(dt)
    want = _rule(xd.float())
    full = xd.cuda()
    R.call([full[:, r * vs:(r + 1) * vs].contiguous() for r in range(W)], batch, dec)
    c.greedy_advance(full, batch, ref["out_tokens"], ref["step_ptr"], ref["cur_ids"], ref["positions"], ref["seq_lens"], ref["slot_map"],
                     ref["page_table"], PAGE)
    torch.cuda.synchronize()
    assert ref["out_tokens"][:batch, step].cpu().tolist() == want, f"step {step}: cts_greedy_advance disagrees with the rule"
    for r in range(W):
        got = dec[r]["out_tokens"][:batch, step].cpu().tolist()
        bad = [(b, kinds[b], got[b], want[b]) for b in range(batch) if got[b] != want[b]]
        assert not bad, f"step {step}, rank {r} of {W}: (row, kind, token, expected) {bad}"
        for k in STATE:
            assert torch.equal(dec[r][k], ref[k]), f"step {step}, rank {r} of {W}: {k} differs from cts_greedy_advance"


@pytest.mark.parametrize("batch", [1, 5, 16])
@pytest.mark.parametrize("vshard", [152064 // 8, 152064 // 4, 152064 // 2, 1000, 1003, 7])
@pytest.mark.parametrize("W", WORLDS, ids=W_IDS)
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_peer_greedy_matches_single_gpu_greedy(dt, W, vshard, batch):
    """Three steps on the same tables: every planted row kind, on every rank bit-identical to cts_greedy_advance on the whole row."""
    c = ctx()
    g = torch.Generator().manual_seed(W * 100003 + vshard * 17 + batch)
    max_b = batch + 3                                     # rows b >= batch of the tables and of the state stay untouched
    R = _GreedyRanks(c, W, max_b)
    init = _decode_state(max_b, g)
    ref, dec = _on_device(init), [_on_device(init) for _ in range(W)]
    slots0 = []
    for step in range(3):
        kinds = [PLANTED[(b + 5 * step) % len(PLANTED)] for b in range(batch)]
        _greedy_step(c, R, ref, dec, W, vshard, batch, dt, kinds, g, step)
        slots0.append(int(ref["slot_map"][0]))
    last_page = int(init["page_table"][0, MAX_PAGES - 1])
    assert slots0 == [last_page * PAGE, last_page * PAGE + 1, -1], slots0
    for r in range(W):
        assert dec[r]["step_ptr"].cpu().tolist() == [3, 0] and R.state[r].cpu().tolist() == [3, 0], f"rank {r}: step / epoch"
        assert bool((R.flags[r][:, :batch] == 3).all()), f"rank {r}: a candidate flag of this epoch is missing"
        assert not R.flags[r][:, batch:].any() and not R.cand[r][:, batch:].any(), f"rank {r}: rows past the batch were written"
        for k in STATE:
            if k != "step_ptr":
                assert torch.equal(dec[r][k][batch:].cpu(), init[k][batch:]), f"rank {r}: {k} rows past the batch changed"
    record("peer_greedy_advance", dtype=str(dt).split(".")[-1], W=W, vshard=vshard, batch=batch, steps=3, bit_exact_state=True)


@pytest.mark.parametrize("kind", NO_CANDIDATE)
@pytest.mark.parametrize("vshard", [152064 // 8, 1003, 7])
@pytest.mark.parametrize("W", WORLDS, ids=W_IDS)
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_peer_greedy_row_without_a_candidate_gives_token_0(dt, W, vshard, kind):
    """A row with no entry greater than -inf (every shard publishes "no candidate") gives token 0, as cts_greedy_advance does -- not
    the index one past a shard, which on the last rank is outside the vocabulary.  A random row beside it is unaffected."""
    c = ctx()
    g = torch.Generator().manual_seed(W * 7 + vshard)
    batch = 3
    R = _GreedyRanks(c, W, batch)
    init = _decode_state(batch, g)
    ref, dec = _on_device(init), [_on_device(init) for _ in range(W)]
    _greedy_step(c, R, ref, dec, W, vshard, batch, dt, [kind, "random", kind], g, 0)
    assert dec[0]["out_tokens"][[0, 2], 0].cpu().tolist() == [0, 0]
    record("peer_greedy_no_candidate", dtype=str(dt).split(".")[-1], W=W, vshard=vshard, kind=kind, token=0)


def test_peer_greedy_rejects_bad_arguments():
    """Refused before any launch (a launch with a missing rank would spin), so one rank's tables serve every world size here."""
    from chatts_b200._cabi import CtsError
    c = ctx()
    R = _GreedyRanks(c, 1, 4)
    d = _on_device(_decode_state(4, torch.Generator().manual_seed(1)))
    lg = torch.zeros(4, 64, dtype=torch.bfloat16, device="cuda")
    args = lambda: (d["out_tokens"], d["step_ptr"], d["cur_ids"], d["positions"], d["seq_lens"], d["slot_map"], d["page_table"])
    with pytest.raises(CtsError, match="sizes"):                                  # batch > max_batch
        c.peer_greedy_advance(torch.zeros(5, 64, dtype=torch.bfloat16, device="cuda"), 5, 0, 2, R.cand_ptrs, R.flag_ptrs, R.state[0], 4,
                              *args(), PAGE)
    huge = torch.zeros(1, 1, dtype=torch.bfloat16, device="cuda").expand(1, 1 << 30)  # vshard * W = 2^31: no int32 global index
    with pytest.raises(CtsError, match="sizes"):
        c.peer_greedy_advance(huge, 1, 0, 2, R.cand_ptrs, R.flag_ptrs, R.state[0], 4, *args(), PAGE)
    with pytest.raises(CtsError, match="rank / world"):
        c.peer_greedy_advance(lg, 1, 0, 33, R.cand_ptrs, R.flag_ptrs, R.state[0], 4, *args(), PAGE)
    with pytest.raises(CtsError, match="rank / world"):
        c.peer_greedy_advance(lg, 1, 2, 2, R.cand_ptrs, R.flag_ptrs, R.state[0], 4, *args(), PAGE)
    with pytest.raises(CtsError, match="paging"):
        c.peer_greedy_advance(lg, 1, 0, 2, R.cand_ptrs, R.flag_ptrs, R.state[0], 4, *args(), 0)
    torch.cuda.synchronize()
    assert not R.state[0].any() and not R.flags[0].any() and d["step_ptr"].cpu().tolist() == [0, 0]


# ---------------------------------------------------------------------------------------------------------------------------------
# cts_peer_allreduce_residual_rmsnorm (one-shot)
# ---------------------------------------------------------------------------------------------------------------------------------
class _OneShotRanks:
    """W ranks of the one-shot all-reduce, laid out as tp.PeerBuffers does: per rank two buffers, each rows fp32 [W][max_tokens][h]
    and flags int32 [W][max_tokens][8] (zeroed), the int64 pointer arrays every rank passes, and the rank's own state and stream."""

    def __init__(self, c, W, max_tokens, h):
        self.c, self.W, self.max_tokens = c, W, max_tokens
        self.rows = [[torch.zeros(W, max_tokens, h, device="cuda") for _ in range(W)] for _ in range(2)]
        self.flags = [[torch.zeros(W, max_tokens, 8, dtype=torch.int32, device="cuda") for _ in range(W)] for _ in range(2)]
        self.row_ptrs = [torch.tensor([t.data_ptr() for t in self.rows[b]], dtype=torch.int64, device="cuda") for b in range(2)]
        self.flag_ptrs = [torch.tensor([t.data_ptr() for t in self.flags[b]], dtype=torch.int64, device="cuda") for b in range(2)]
        self.state = [torch.zeros(2, dtype=torch.int32, device="cuda") for _ in range(W)]
        self.streams = [torch.cuda.Stream() for _ in range(W)] if W > 1 else None

    def call(self, which, parts, split, resid, norm_w, eps, xn, T):
        """parts[r]: fp32 [split, T, h] of rank r; resid[r] [T, h] is updated in place, xn[r] receives the norm."""
        torch.cuda.synchronize()
        for r in range(self.W):
            with _on(self.streams, r):
                self.c.peer_allreduce_residual_rmsnorm(parts[r], split, self.row_ptrs[which], self.flag_ptrs[which], self.state[r], r,
                                                       self.W, self.max_tokens, resid[r], resid[r], norm_w, eps, xn[r], T)
        torch.cuda.synchronize()


def _cluster(h):
    """The cluster width cts_peer_allreduce_residual_rmsnorm picks: CTAs per token."""
    return next((c for c in (8, 4, 2) if h % (8 * c) == 0 and h // (8 * c) >= 32), 1)


def _ll_cluster(h, W):
    """CTAs per token of cts_peer_allreduce_ll, or None where it does not take (W, h)."""
    if W not in (2, 4, 8) or h % (4 * W):
        return None
    hw = h // W
    return next((c for c in (8, 4, 2, 1) if hw % (4 * c) == 0 and 32 <= hw // (4 * c) <= 256), 1 if hw // 4 <= 256 else None)


_MANT = {torch.bfloat16: 7, torch.float16: 10}
_EMIN = {torch.bfloat16: -126, torch.float16: -14}


def _ulps(got, want, dt):
    """|got - want| per element in units of the last place of dt at want (fp64; subnormal spacing below the normal range)."""
    _, e = torch.frexp(want)                              # want = m * 2^e, 0.5 <= |m| < 1
    e = torch.where(want == 0, torch.full_like(e, _EMIN[dt] + 1), e)
    ulp = torch.ldexp(torch.ones_like(want), (e - 1).clamp_min(_EMIN[dt]) - _MANT[dt])
    return (got.double() - want).abs() / ulp


@pytest.mark.parametrize("h", [256, 512, 1024, 4096, 5120, 32768])
@pytest.mark.parametrize("split", [1, 3, 7])
@pytest.mark.parametrize("W", WORLDS, ids=W_IDS)
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_one_shot_allreduce_matches_rank_ordered_sum(dt, W, split, h):
    """Six calls alternating the two buffers as the model does (plus one repeated buffer), T changing between calls: h bit for bit the
    rank-ordered sum and the LL kernel's h, identical on every rank; norm_out identical on every rank and within 2 ulps of RMSNorm."""
    c = ctx()
    C, C_ll = _cluster(h), _ll_cluster(h, W)
    tm = min(16, 128 // (W * max(C, C_ll or 1)))          # co-resident: W x C x T <= 128 CTAs for both kernels
    g = torch.Generator().manual_seed(W * 1000 + split * 100 + h)
    R = _OneShotRanks(c, W, tm, h)
    L = _LLRanks(c, W, tm, h) if C_ll else None
    h0 = (torch.randn(tm, h, generator=g) * 0.5).to(dt).cuda()
    nw = (1.0 + 0.1 * torch.randn(h, generator=g)).to(dt).cuda()
    resid, resid_ll = [h0.clone() for _ in range(W)], [h0.clone() for _ in range(W)]
    xn, xn_ll = [torch.empty(tm, h, dtype=dt, device="cuda") for _ in range(W)], [torch.empty(tm, h, dtype=dt, device="cuda") for _ in range(W)]
    cur = h0.clone()
    worst = 0.0
    Ts = [tm, 1, max(1, tm // 2), tm, 1, max(1, (tm + 2) // 3)]
    for n, (which, T) in enumerate(zip([0, 1, 0, 1, 1, 0], Ts)):
        parts = [(torch.randn(split, T, h, generator=g) * 0.3).cuda() for _ in range(W)]
        for x in xn:
            x.fill_(float("nan"))
        R.call(which, parts, split, [x[:T] for x in resid], nw, 1e-6, [x[:T] for x in xn], T)
        cur[:T] = _expected(parts, split, cur[:T], dt)
        for r in range(W):
            assert torch.equal(resid[r], cur), f"call {n} (T={T}): h differs from the rank-ordered sum on rank {r}"
            assert torch.equal(xn[r][:T], xn[0][:T]), f"call {n}: norm_out differs between ranks 0 and {r}"
            assert bool(xn[r][T:].isnan().all()), f"call {n}: norm_out written past token {T} on rank {r}"
        if L is not None:
            L.call(which, parts, split, [x[:T] for x in resid_ll], nw, 1e-6, [x[:T] for x in xn_ll], T)
            for r in range(W):
                assert torch.equal(resid_ll[r], cur), f"call {n}: h of cts_peer_allreduce_ll differs on rank {r}"
        x = cur[:T].double().cpu()
        want = nw.double().cpu() * x / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)
        err = float(_ulps(xn[0][:T].cpu(), want, dt).max())
        worst = max(worst, err)
        assert err <= 2.0, f"call {n}: norm_out {err:.2f} ulps from the fp64 RMSNorm of h"
    for r in range(W):
        assert R.state[r].cpu().tolist() == [6, 0], f"rank {r}: the epoch advances once per call"
    # the kernel rounds x * inv to the dtype, multiplies by the weight in fp32 and rounds again: at most 1.5 ulps plus the fp32
    # statistic's error.  Measured worst case over all cases on an H100 80GB HBM3: 1.44 ulps (bf16), 1.46 ulps (fp16)
    record("peer_allreduce_one_shot", dtype=str(dt).split(".")[-1], W=W, split=split, h=h, cluster=C, max_tokens=tm, norm_ulps=worst,
           bit_exact_h=True, matches_ll=L is not None)


@pytest.mark.parametrize("h", [512, 5120])
@pytest.mark.parametrize("W", WORLDS, ids=W_IDS)
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_one_shot_allreduce_residual_only(dt, W, h):
    """norm_w = None: the residual add alone (no norm_out), T changing over the same buffers."""
    c = ctx()
    tm = min(8, 128 // (W * _cluster(h)))
    g = torch.Generator().manual_seed(W + h)
    R = _OneShotRanks(c, W, tm, h)
    for n, T in enumerate([tm, 1, max(1, tm // 2), tm]):
        h0 = (torch.randn(T, h, generator=g) * 0.5).to(dt).cuda()
        resid = [h0.clone() for _ in range(W)]
        parts = [(torch.randn(2, T, h, generator=g) * 0.3).cuda() for _ in range(W)]
        R.call(n % 2, parts, 2, resid, None, 1e-6, [None] * W, T)
        want = _expected(parts, 2, h0, dt)
        for r in range(W):
            assert torch.equal(resid[r], want), f"call {n}: h differs on rank {r}"


def test_one_shot_allreduce_rejects_bad_arguments():
    from chatts_b200._cabi import CtsError
    """Refused before any launch, so one rank's buffers serve every world size here."""
    c = ctx()
    R = _OneShotRanks(c, 1, 4, 256)
    dt = torch.bfloat16

    def run(h=256, t=1, rank=0, world=2, max_tokens=4, norm=True, norm_out=True):
        part = torch.zeros(1, max(t, 1), h, device="cuda")
        resid = torch.zeros(max(t, 1), h, dtype=dt, device="cuda")
        nw = torch.ones(h, dtype=dt, device="cuda") if norm else None
        xn = torch.empty(max(t, 1), h, dtype=dt, device="cuda") if norm_out else None
        c.peer_allreduce_residual_rmsnorm(part, 1, R.row_ptrs[0], R.flag_ptrs[0], R.state[0], rank, world, max_tokens, resid, resid, nw,
                                          1e-6, xn, t)

    with pytest.raises(CtsError, match="multiple of 8"):
        run(h=252)
    with pytest.raises(CtsError, match="h too large"):           # h % 16 != 0 gives one CTA per token: 4104 > 4096 columns
        run(h=4104)
    with pytest.raises(CtsError, match="1..max_tokens"):
        run(t=0)
    with pytest.raises(CtsError, match="1..max_tokens"):
        run(t=5)
    with pytest.raises(CtsError, match="rank / world"):
        run(world=17)
    with pytest.raises(CtsError, match="rank / world"):
        run(rank=2)
    with pytest.raises(CtsError, match="norm_w / norm_out"):
        run(norm_out=False)
    torch.cuda.synchronize()
    assert not R.state[0].any() and not R.flags[0][0].any()
