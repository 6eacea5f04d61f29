"""cts_sample_advance (csrc/sampling.cu) against the exact distribution of its statement (tests/cabi_double.py ``sample_reference``:
a float64 CDF over the kept set in index order), where an fp32 inverse CDF goes wrong: the far tail behind a dominant token, rows with
-inf (refused) and NaN logits, the top-k / top-p thresholds, degenerate rows, and the masks written by cts_struct_mask_apply and
cts_logit_proc_apply.

The kernel's uniform is a counter-based function of (seed, step, sequence), so every statistic below is deterministic for its seed;
the thresholds are wide (chi-square at p ~ 3e-7, means within 4 standard errors) and the statement's own draws at the same steps
must pass them too.

  T1  one dominant token, N(0, 1) tail, half the vocabulary at -inf, a few NaN: launched at the steps whose statement token lies in
      the tail -- every token has mass, and the tail picks follow the exact tail distribution (chi-square over bins of equal tail
      mass by logit, size-biased mean logit).  Matching the statement draw by draw is not a valid check there: the rounding of the
      cross-chunk prefix is about ulp(total), which spans tens of tail tokens.
  T2  1024 identical full-vocabulary rows x 64 steps: whole-row chi-square.
  T3  thresholds and edges: the observed tokens are a subset of the statement's kept set and every kept token expected 20 times
      appears; top_k = 1 and degenerate rows give cts_greedy_advance's token.
  T4  rows where every kept token holds >= 2^-12 of the kept mass: the statement's token draw by draw, up to a CDF boundary.
  T5  repeated launches are bit-identical; a captured graph replays the eager launches and their bookkeeping.
  T6  cts_struct_mask_apply / cts_logit_proc_apply (allowed_token_ids, min_tokens) -> cts_sample_advance: no refused id, ever.
"""
import math

import numpy as np
import pytest
import torch

from tests.cabi_double import TorchDouble
from tests.gpu_util import ctx, record
from tests.logit_proc_double import apply_reference
from tests.structured_double import pack_bits

pytestmark = pytest.mark.gpu

V_FULL = 152064
SEED = 7
STEP_RANGE = 1 << 22                       # steps searched for tail draws
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _on_device():
    """False on the CPU shim, where device tensors stay on the host and a launch costs milliseconds: the draw counts shrink there."""
    return torch.zeros(1).cuda().is_cuda


# ---------------------------------------------------------------------------------------------------------------------------------
# the statement's uniform and token, vectorised over steps
# ---------------------------------------------------------------------------------------------------------------------------------
def _splitmix64(z):
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def _uniforms(seed, steps, b):
    """u(seed, step, sequence) of the statement for arrays of steps / sequences, float64 in [0, 1)."""
    steps = np.asarray(steps, dtype=np.uint64)
    b = np.asarray(b, dtype=np.uint64)
    h = _splitmix64(np.uint64(seed) ^ _splitmix64((steps << np.uint64(32)) | b))
    return (h >> np.uint64(40)).astype(np.float64) / 16777216.0


def _statement_tokens(cdf, kept, u):
    t = np.searchsorted(cdf, u * cdf[-1], side="right")
    return np.minimum(t, int(np.nonzero(kept)[0][-1]))


_U_CACHE = {}


def _tail_steps(cdf, kept, dom, n):
    """The first n steps in [0, 2^22) whose statement token (sequence 0) is not the dominant one."""
    if "u" not in _U_CACHE:
        _U_CACHE["u"] = _uniforms(SEED, np.arange(STEP_RANGE), 0)
    u = _U_CACHE["u"]
    lo, hi = (cdf[dom - 1] if dom > 0 else 0.0), cdf[dom]
    t = u * cdf[-1]
    steps = np.nonzero((t < lo) | (t >= hi))[0][:n]
    toks = _statement_tokens(cdf, kept, u[steps])
    assert (toks != dom).all()
    return steps, toks


def _mass(cdf):
    return np.diff(np.concatenate([[0.0], cdf]))


def _chi2_limit(dof, z=5.0):
    """Wilson-Hilferty quantile of chi-square(dof) at z standard deviations (z = 5: p ~ 3e-7)."""
    return dof * (1 - 2 / (9 * dof) + z * math.sqrt(2 / (9 * dof))) ** 3


def _bins_by_logit(x, prob, n_bins, n_draws):
    """Bin id per token (-1: no mass): tokens sorted by logit, cut into bins of about equal mass, bins expected < 5 times merged
    into the previous one.  Returns (bin of token, expected fraction per bin)."""
    ids = np.nonzero(prob > 0)[0]
    order = ids[np.lexsort((ids, -x[ids]))]
    p = prob[order] / prob[order].sum()
    before = np.concatenate([[0.0], np.cumsum(p)[:-1]])
    raw = np.minimum((before * n_bins).astype(np.int64), n_bins - 1)
    _, raw = np.unique(raw, return_inverse=True)
    frac = np.bincount(raw, weights=p)
    merged, acc, cur = np.zeros(len(frac), dtype=np.int64), 0.0, 0
    for i, f in enumerate(frac):                      # fold small bins forward until each holds >= 5 expected draws
        merged[i] = cur
        acc += f
        if acc * n_draws >= 5 and i < len(frac) - 1:
            cur, acc = cur + 1, 0.0
    if acc * n_draws < 5 and cur > 0:
        merged[merged == cur] = cur - 1
    bin_of = np.full(x.shape[0], -1, dtype=np.int64)
    bin_of[order] = merged[raw]
    return bin_of, np.bincount(merged[raw], weights=p)


def _chi2(toks, bin_of, frac):
    n = len(toks)
    obs = np.bincount(bin_of[toks], minlength=len(frac)).astype(np.float64)
    exp = frac * n
    return float(((obs - exp) ** 2 / exp).sum()), len(frac) - 1


# ---------------------------------------------------------------------------------------------------------------------------------
# launches
# ---------------------------------------------------------------------------------------------------------------------------------
def _launch_at_steps(c, row, steps, temp, top_k=0, top_p=1.0):
    """One single-row launch per step (step_ptr = [step, 0], the token read from cur_ids); checks the step pointer's advance."""
    lg = row[None].contiguous().cuda()
    sp = torch.zeros(len(steps), 2, dtype=torch.int32)
    sp[:, 0] = torch.from_numpy(np.asarray(steps, dtype=np.int64)).to(torch.int32)
    sp = sp.cuda()
    cur = torch.full((len(steps),), -1, dtype=torch.int32).cuda()
    for i in range(len(steps)):
        c.sample_advance(lg, 1, temp, top_k, top_p, SEED, None, sp[i], cur[i:i + 1], None, None, None, None, 16)
    torch.cuda.synchronize()
    sp = sp.cpu()
    assert (sp[:, 0].numpy() == np.asarray(steps) + 1).all() and (sp[:, 1] == 0).all()
    return cur.cpu().numpy().astype(np.int64)


def _launch_rows(c, logits, temp, top_k, top_p, steps, seed=SEED):
    """All rows of ``logits`` for steps 0..steps-1 through the device step pointer; tokens [B, steps]."""
    B = logits.shape[0]
    out = torch.full((B, steps), -1, dtype=torch.int32).cuda()
    sp = torch.zeros(2, dtype=torch.int32).cuda()
    for _ in range(steps):
        c.sample_advance(logits, B, temp, top_k, top_p, seed, out, sp, None, None, None, None, None, 16)
    torch.cuda.synchronize()
    assert sp.cpu().tolist() == [steps, 0]
    return out.cpu().numpy().astype(np.int64)


def _draw_shape():
    return (128, 16) if _on_device() else (8, 8)


# ---------------------------------------------------------------------------------------------------------------------------------
# T1: support and tail distribution under precision stress
# ---------------------------------------------------------------------------------------------------------------------------------
DOM_POS = {"start": lambda V: 5, "middle": lambda V: V // 2 + 3, "end": lambda V: V - 7}


def _stress_row(dtype, pos, gap, temp, V=V_FULL, seed=11):
    """N(0, 1) logits, a random half of the vocabulary at -inf, 5 NaN, one token at ``gap``; everything times ``temp`` so that z =
    logit / temp is the same stress at every temperature."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(V, generator=g)
    x[torch.rand(V, generator=g) < 0.5] = float("-inf")
    x[torch.randint(0, V, (5,), generator=g)] = float("nan")
    dom = DOM_POS[pos](V)
    x[dom] = gap
    return (x * temp).to(dtype), dom


def _tail_stats(x, prob, dom, toks):
    """(refused picks, tail picks, chi-square, dof, mean tail logit, exact mean, standard error) of the draws ``toks``."""
    tail = prob.copy()
    tail[dom] = 0.0
    refused = int((prob[toks] == 0).sum())
    t = toks[(toks != dom) & (prob[toks] > 0)]
    bin_of, frac = _bins_by_logit(x, tail, 8, len(t))
    chi, dof = _chi2(t, bin_of, frac)
    w = tail / tail.sum()
    fin = w > 0
    mu = float((w[fin] * x[fin]).sum())
    sd = float(np.sqrt((w[fin] * (x[fin] - mu) ** 2).sum()))
    return refused, len(t), chi, dof, float(x[t].mean()), mu, sd / math.sqrt(max(len(t), 1))


def _assert_tail(name, stats, n):
    refused, n_tail, chi, dof, mean, mu, se = stats
    msg = f"{name}: {refused} refused of {n}, {n_tail} tail picks, chi2 {chi:.1f} (dof {dof}), mean tail logit {mean:.3f} vs {mu:.3f}"
    assert refused == 0, msg
    assert n_tail >= 0.98 * n, msg
    assert chi < _chi2_limit(dof), msg
    assert abs(mean - mu) < 4 * se, msg


@pytest.mark.parametrize("temp", [1.0, 0.2], ids=["t1", "t02"])
@pytest.mark.parametrize("gap", [15.0, 18.0], ids=["g15", "g18"])
@pytest.mark.parametrize("pos", ["start", "middle", "end"])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_tail_support_and_distribution(dt, pos, gap, temp):
    c = ctx()
    n = 4000 if _on_device() else 400
    row, dom = _stress_row(DTYPES[dt], pos, gap, temp)
    _, cdf, _, kept = TorchDouble.sample_reference(row, temp, 0, 1.0, SEED, 0, 0)
    steps, ref = _tail_steps(cdf, kept, dom, n)
    assert len(steps) == n
    for i in range(3):                                                   # the vectorised uniform is the statement's
        assert TorchDouble.sample_reference(row, temp, 0, 1.0, SEED, int(steps[i]), 0)[0] == ref[i]
    toks = _launch_at_steps(c, row, steps, temp)
    x, prob = row.float().numpy().astype(np.float64), _mass(cdf)
    assert ((toks >= 0) & (toks < V_FULL)).all()
    got, want = _tail_stats(x, prob, dom, toks), _tail_stats(x, prob, dom, ref)
    record("sample_tail", dtype=dt, pos=pos, gap=gap, temp=temp, n=n, refused=got[0], tail_picks=got[1], chi2=got[2], dof=got[3],
           mean_tail_logit=got[4], exact_mean=got[5], se=got[6], statement_chi2=want[2], statement_mean=want[4])
    _assert_tail("statement", want, n)
    assert np.isfinite(x[toks]).all(), f"{int((~np.isfinite(x[toks])).sum())} non-finite tokens returned"
    _assert_tail("kernel", got, n)


# ---------------------------------------------------------------------------------------------------------------------------------
# T2: whole-row chi-square at full vocabulary
# ---------------------------------------------------------------------------------------------------------------------------------
def _row(kind, V, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(V, generator=g)
    if kind == "randn3":
        x = x * 3
    elif kind == "peaked":
        x[V // 3] = 14.0                                                 # ~83 % of the mass on one token
    return x.to(dtype)


@pytest.mark.parametrize("kind,dt,temp,top_k,top_p", [
    ("randn3", "bf16", 1.0, 0, 1.0), ("randn3", "fp16", 1.0, 0, 1.0), ("peaked", "bf16", 1.0, 0, 1.0), ("peaked", "fp16", 1.0, 0, 0.95),
    ("randn", "bf16", 0.2, 0, 1.0), ("randn", "bf16", 0.2, 0, 0.9), ("randn", "bf16", 0.2, 50, 1.0), ("randn3", "fp16", 1.0, 50, 1.0),
])
def test_whole_row_chi_square(kind, dt, temp, top_k, top_p):
    c = ctx()
    B, S = 1024, 64
    row = _row(kind, V_FULL, DTYPES[dt], 3)
    _, cdf, _, kept = TorchDouble.sample_reference(row, temp, top_k, top_p, SEED, 0, 0)
    toks = _launch_rows(c, row[None].repeat(B, 1).cuda(), temp, top_k, top_p, S).reshape(-1)
    prob, x = _mass(cdf), row.float().numpy().astype(np.float64)
    assert (prob[toks] > 0).all() and kept[toks].all()
    bin_of, frac = _bins_by_logit(x, prob, 32, len(toks))
    chi, dof = _chi2(toks, bin_of, frac)
    u = _uniforms(SEED, np.repeat(np.arange(S), B), np.tile(np.arange(B), S))
    chi_ref, _ = _chi2(_statement_tokens(cdf, kept, u), bin_of, frac)
    record("sample_chi2", kind=kind, dtype=dt, temp=temp, top_k=top_k, top_p=top_p, chi2=chi, dof=dof, statement_chi2=chi_ref)
    assert dof >= 5 and chi_ref < _chi2_limit(dof) and chi < _chi2_limit(dof), (chi, chi_ref, dof)


# ---------------------------------------------------------------------------------------------------------------------------------
# T3: threshold edges against the statement's kept set
# ---------------------------------------------------------------------------------------------------------------------------------
def _support_and_coverage(row, temp, top_k, top_p, toks):
    """Every token drawn has mass in the statement's kept set, and every kept token expected >= 20 times was drawn.  Returns the
    statement's (mass, kept)."""
    _, cdf, _, kept = TorchDouble.sample_reference(row, temp, top_k, top_p, SEED, 0, 0)
    prob = _mass(cdf)
    toks = np.asarray(toks).reshape(-1)
    assert ((toks >= 0) & (toks < row.shape[0])).all()
    bad = toks[~(prob[toks] > 0)]
    assert len(bad) == 0, f"tokens outside the kept set: {sorted(set(bad.tolist()))[:10]}"
    want = np.nonzero(prob / prob.sum() * len(toks) >= 20)[0]
    missing = np.setdiff1d(want, toks)
    assert len(missing) == 0, f"kept tokens expected >= 20 times never drawn: {missing[:10].tolist()}"
    return prob, kept


def _draw(c, row, temp, top_k, top_p):
    B, S = _draw_shape()
    return _launch_rows(c, row[None].repeat(B, 1).cuda(), temp, top_k, top_p, S)


def _greedy(c, logits):
    B = logits.shape[0]
    cur = torch.full((B,), -1, dtype=torch.int32).cuda()
    c.greedy_advance(logits, B, None, None, cur, None, None, None, None, 16)
    torch.cuda.synchronize()
    return cur.cpu().numpy().astype(np.int64)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_ties_straddling_top_k_are_all_kept(dt):
    """top_k = 4 with two values above a 5-way tie: the 4th largest value is tied, so all 7 ids are kept (the statement, like
    transformers' TopKLogitsWarper, keeps every logit >= the k-th largest)."""
    c = ctx()
    row = _row("randn", 1000, torch.float32, 1).clamp(max=2.0)
    row[[10, 20]] = 3.5
    row[[3, 400, 401, 999, 77]] = 3.0
    row = row.to(DTYPES[dt])
    toks = _draw(c, row, 1.0, 4, 1.0)
    _, kept = _support_and_coverage(row, 1.0, 4, 1.0, toks)
    assert np.nonzero(kept)[0].tolist() == [3, 10, 20, 77, 400, 401, 999]


@pytest.mark.parametrize("V", [1000, 1003, 8193, 152064])
def test_top_k_one_is_greedy_and_a_tied_maximum_stays_tied(V):
    c = ctx()
    row = _row("randn3", V, torch.bfloat16, V)
    toks = _draw(c, row, 0.7, 1, 1.0)
    g = _greedy(c, row[None].cuda())[0]
    assert (toks == g).all(), (g, sorted(set(toks.reshape(-1).tolist())))
    tied = [V // 7, V // 2, V - 1]
    row[tied] = (row.float().max() + 1.0).to(row.dtype)
    toks = _draw(c, row, 0.7, 1, 1.0)
    _support_and_coverage(row, 0.7, 1, 1.0, toks)
    assert set(toks.reshape(-1).tolist()) == set(tied)


@pytest.mark.parametrize("V", [1000, 8192])
def test_top_k_at_or_above_vocab_is_no_filter(V):
    """top_k >= V keeps every non-NaN logit: draw for draw the same tokens as top_k = 0."""
    c = ctx()
    row = _row("randn", V, torch.float32, 2)
    row[:: 17] = float("-inf")
    row[5:: 101] = float("nan")
    row = row.to(torch.bfloat16)
    base = _draw(c, row, 1.0, 0, 1.0)
    _support_and_coverage(row, 1.0, 0, 1.0, base)
    for k in (V, V + 7):
        assert (_draw(c, row, 1.0, k, 1.0) == base).all()


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_top_p_extremes(dt):
    """A tiny top_p keeps only the maximum and its ties; top_p = 1 - 2^-24 cuts only the far tail."""
    c = ctx()
    row = _row("randn", 8193, torch.float32, 4)
    row[[100, 6000]] = 4.5
    row = row.to(DTYPES[dt])
    toks = _draw(c, row, 1.0, 0, 1e-7)
    _, kept = _support_and_coverage(row, 1.0, 0, 1e-7, toks)
    assert np.nonzero(kept)[0].tolist() == [100, 6000] and set(toks.reshape(-1).tolist()) == {100, 6000}
    top_p = float(np.float32(1 - 2 ** -24))
    toks = _draw(c, row, 1.0, 0, top_p)
    _support_and_coverage(row, 1.0, 0, top_p, toks)


@pytest.mark.parametrize("temp", [0.05, 0.2, 3.0])
@pytest.mark.parametrize("top_k,top_p", [(0, 1.0), (0, 0.9), (40, 0.8)])
def test_temperatures(temp, top_k, top_p):
    c = ctx()
    row = _row("randn", 8193, torch.float32, 5).mul(2).to(torch.bfloat16)
    _support_and_coverage(row, temp, top_k, top_p, _draw(c, row, temp, top_k, top_p))


def test_fp16_rows_near_the_largest_finite_value():
    """Logits within a few hundred of +65504 (spacing 32 there), a block at -65504; temperature 400 spreads the top ones."""
    c = ctx()
    g = torch.Generator().manual_seed(6)
    V = 4096
    row = 65504.0 - 32.0 * torch.randint(0, 40, (V,), generator=g).float()
    row[torch.rand(V, generator=g) < 0.3] = -65504.0
    row = row.to(torch.float16)
    assert torch.isfinite(row).all() and float(row.float().max()) == 65504.0
    for temp, top_k, top_p in ((400.0, 0, 1.0), (400.0, 0, 0.7), (400.0, 300, 1.0), (1.0, 0, 1.0)):
        _support_and_coverage(row, temp, top_k, top_p, _draw(c, row, temp, top_k, top_p))


@pytest.mark.parametrize("dt,temp,top_k", [("fp16", 1e-5, 0), ("fp16", 1e-5, 30), ("bf16", 1.0, 50)])
def test_subnormal_logits(dt, temp, top_k):
    """All logits subnormal (and +-0): the keys order them exactly; fp16 subnormals are normal in fp32, so a small temperature
    spreads their probabilities; bf16 subnormals at temperature 1 are uniform over the top-k set."""
    c = ctx()
    g = torch.Generator().manual_seed(8)
    V = 1003
    tiny = torch.finfo(DTYPES[dt]).tiny
    row = (torch.rand(V, generator=g) * 2 - 1) * tiny
    row[:3] = torch.tensor([0.0, -0.0, tiny / 4])
    row = row.to(DTYPES[dt])
    r = row.float()
    assert (r.abs() <= tiny).all() and (r.abs() < tiny).sum() > V // 2 and (r != 0).sum() > V // 2
    _support_and_coverage(row, temp, top_k, 1.0, _draw(c, row, temp, top_k, 1.0))


@pytest.mark.parametrize("V", [1000, 1003, 8192, 8193, 151936, 152064])
def test_degenerate_rows_follow_greedy(V):
    """All -inf, all NaN, -inf and NaN mixed, a single finite logit among -inf or among NaN: cts_greedy_advance's token (index 0
    for a row without a finite logit), at every step."""
    c = ctx()
    g = torch.Generator().manual_seed(V)
    rows = torch.full((5, V), float("-inf"))
    rows[1] = float("nan")
    rows[2, torch.rand(V, generator=g) < 0.5] = float("nan")
    rows[3, V - 2] = -3.0
    rows[4] = float("nan")
    rows[4, V // 3] = 2.0
    for dt in (torch.bfloat16, torch.float16):
        lg = rows.to(dt).cuda()
        want = _greedy(c, lg)
        assert want.tolist() == [0, 0, 0, V - 2, V // 3]
        for temp, top_k, top_p in ((1.0, 0, 1.0), (0.2, 50, 0.9)):
            toks = _launch_rows(c, lg, temp, top_k, top_p, 3)
            assert (toks == want[:, None]).all(), (toks.tolist(), want.tolist())


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("V", [1000, 1003, 8192, 8193, 151936, 152064])
def test_vocab_sizes(V, dt):
    """Empty chunks (V = 1000: threads past the end own nothing), the scalar path (V % 8 != 0), one element past a multiple of 8,
    the checkpoint's padded vocabulary and the lm_head's."""
    c = ctx()
    row = _row("randn", V, torch.float32, V + 1).mul(2)
    row[V - 1] = row.max() + 0.5                                         # the last index is the most probable one
    row = row.to(DTYPES[dt])
    for temp, top_k, top_p in ((0.7, 0, 0.9), (1.0, 40, 1.0)):
        _support_and_coverage(row, temp, top_k, top_p, _draw(c, row, temp, top_k, top_p))


# ---------------------------------------------------------------------------------------------------------------------------------
# T4: draw for draw where every kept token holds >= 2^-12 of the kept mass
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("V,scale,temp,top_k,top_p", [(1000, 1.0, 1.0, 0, 1.0), (1003, 1.0, 0.5, 0, 0.5), (8193, 0.3, 1.0, 300, 1.0),
                                                      (152064, 0.3, 1.0, 1000, 1.0), (152064, 1.0, 0.2, 0, 0.9)])
def test_draw_for_draw(V, scale, temp, top_k, top_p, dt):
    c = ctx()
    g = torch.Generator().manual_seed(V + top_k)
    row = (torch.rand(V, generator=g) if V < 2000 else torch.randn(V, generator=g)).mul(scale).to(DTYPES[dt])
    _, cdf, _, kept = TorchDouble.sample_reference(row, temp, top_k, top_p, SEED, 0, 0)
    prob = _mass(cdf)
    share = prob[kept] / cdf[-1]
    assert share.min() >= 2 ** -12, share.min()                          # the precondition of an exact comparison
    B, S = (64, 32) if _on_device() else (8, 8)
    toks = _launch_rows(c, row[None].repeat(B, 1).cuda(), temp, top_k, top_p, S)
    s_idx, b_idx = np.meshgrid(np.arange(S), np.arange(B))
    u = _uniforms(SEED, s_idx.reshape(-1), b_idx.reshape(-1))
    ref = _statement_tokens(cdf, kept, u).reshape(B, S)
    target = (u * cdf[-1]).reshape(B, S)
    order = np.cumsum(kept) - 1                                          # position of a token in kept index order
    tol = 64 * float(np.spacing(np.float32(cdf[-1])))
    bad = []
    for b, s in zip(*np.nonzero(toks != ref)):
        t, r = int(toks[b, s]), int(ref[b, s])
        edge = cdf[min(t, r)]                                            # the CDF boundary between two adjacent kept tokens
        if not (kept[t] and abs(int(order[t]) - int(order[r])) == 1 and abs(target[b, s] - edge) <= tol):
            bad.append((int(b), int(s), t, r, float(target[b, s] - edge)))
    record("sample_draw_for_draw", V=V, dtype=dt, temp=temp, top_k=top_k, top_p=top_p, draws=B * S,
           boundary=int((toks != ref).sum()) - len(bad), bad=len(bad))
    assert not bad, bad[:5]


# ---------------------------------------------------------------------------------------------------------------------------------
# T5: determinism, graphs and bookkeeping
# ---------------------------------------------------------------------------------------------------------------------------------
def test_repeated_launches_are_bit_identical():
    c = ctx()
    row, dom = _stress_row(torch.bfloat16, "start", 18.0, 1.0)
    _, cdf, _, kept = TorchDouble.sample_reference(row, 1.0, 0, 1.0, SEED, 0, 0)
    steps, _ = _tail_steps(cdf, kept, dom, 1000)
    assert (_launch_at_steps(c, row, steps, 1.0) == _launch_at_steps(c, row, steps, 1.0)).all()
    logits = _row("randn3", V_FULL, torch.bfloat16, 3)[None].repeat(1024, 1).cuda()
    for temp, top_k, top_p in ((1.0, 0, 1.0), (0.2, 50, 0.9)):
        assert (_launch_rows(c, logits, temp, top_k, top_p, 64) == _launch_rows(c, logits, temp, top_k, top_p, 64)).all()


def test_graph_replay_matches_eager_launches_and_bookkeeping():
    c = ctx()
    B, S, page, max_pages, step0 = 1024, 32, 16, 8, 5
    g = torch.Generator().manual_seed(9)
    logits = (torch.randn(B, V_FULL, generator=g) * 2).to(torch.bfloat16).cuda()
    pos0 = torch.randint(0, page * max_pages - S - 1, (B,), generator=g).to(torch.int32)
    pt = torch.randperm(B * max_pages, generator=g).to(torch.int32).view(B, max_pages)

    def state():
        return dict(out=torch.full((B, 64), -1, dtype=torch.int32, device="cuda"),
                    sp=torch.tensor([step0, 0], dtype=torch.int32, device="cuda"), cur=torch.full((B,), -1, dtype=torch.int32, device="cuda"),
                    pos=pos0.clone().cuda(), sl=(pos0 + 1).cuda(), slot=torch.full((B,), -7, dtype=torch.int32, device="cuda"),
                    pt=pt.clone().cuda())

    def launch(s):
        c.sample_advance(logits, B, 0.8, 50, 0.95, 1234, s["out"], s["sp"], s["cur"], s["pos"], s["sl"], s["slot"], s["pt"], page)

    eager, graphed = state(), state()
    for _ in range(S):
        launch(eager)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch(graphed)
    torch.cuda.synchronize()
    assert graphed["sp"].cpu().tolist() == [step0, 0] and (graphed["out"] == -1).all()          # capture launches nothing
    for _ in range(S):
        graph.replay()
    torch.cuda.synchronize()
    for k in ("out", "sp", "cur", "pos", "sl", "slot"):
        assert torch.equal(graphed[k].cpu(), eager[k].cpu()), k
    assert graphed["sp"].cpu().tolist() == [step0 + S, 0]
    pos = pos0 + S
    assert torch.equal(graphed["pos"].cpu(), pos) and torch.equal(graphed["sl"].cpu(), pos + 1)
    want_slot = pt[torch.arange(B), (pos // page).long()] * page + pos % page
    assert torch.equal(graphed["slot"].cpu(), want_slot)
    out = graphed["out"].cpu()
    assert (out[:, :step0] == -1).all() and (out[:, step0 + S:] == -1).all() and torch.equal(out[:, step0 + S - 1], graphed["cur"].cpu())
    for b in (0, 511, 1023):
        _, cdf, _, kept = TorchDouble.sample_reference(logits[b].cpu(), 0.8, 50, 0.95, 1234, 0, b)
        assert kept[out[b, step0:step0 + S].numpy()].all()


# ---------------------------------------------------------------------------------------------------------------------------------
# T6: the kernels that write refusals, chained into the sampler
# ---------------------------------------------------------------------------------------------------------------------------------
def _chunk_ends(V):
    """The last index of each thread's chunk in sample_advance_kernel (1024 threads, chunks rounded up to multiples of 8): where a
    walk that rounding leaves short ends up."""
    per = ((V + 1023) // 1024 + 7) // 8 * 8
    return np.arange(per - 1, V, per)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("chain,n_allowed,gap", [("struct", 64, 15.0), ("struct", V_FULL // 3, 18.0), ("allowed_ids", V_FULL // 3, 18.0),
                                                 ("min_tokens", 0, 18.0)])
def test_refused_ids_are_never_sampled(chain, n_allowed, gap, dt):
    c = ctx()
    row, dom = _stress_row(DTYPES[dt], "start", gap, 1.0, seed=21)
    x = row.float().numpy()
    g = np.random.default_rng(5)
    finite = np.nonzero(np.isfinite(x))[0]
    lg = row[None].clone().cuda()
    want = row[None].clone()
    if chain in ("struct", "allowed_ids"):
        allowed = np.zeros(V_FULL, dtype=bool)
        allowed[g.choice(finite, n_allowed, replace=False)] = True
        allowed[dom] = True
        if chain == "struct":
            words = torch.from_numpy(pack_bits(allowed[None]))
            c.struct_mask_apply(lg, 1, torch.zeros(1, dtype=torch.int32).cuda(), words.cuda())
            want[0, torch.from_numpy(~allowed)] = float("-inf")
        else:
            bias = torch.zeros(1, V_FULL)
            bias[0, torch.from_numpy(~allowed)] = float("-inf")
            args = [torch.ones(1), torch.zeros(1), torch.zeros(1), torch.zeros(1, (V_FULL + 31) // 32, dtype=torch.int32), None, bias,
                    torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32), None]
            apply_reference(want, 1, *args)
            c.logit_proc_apply(lg, 1, *[a.cuda() if a is not None else None for a in args])
    else:
        # 64 stop ids at finite chunk ends behind the dominant token, banned while n_generated < min_tokens
        ends = _chunk_ends(V_FULL)
        ends = ends[(ends > dom) & np.isfinite(x[ends])]
        stops = torch.from_numpy(g.choice(ends, 64, replace=False).astype(np.int32))[None]
        args = [torch.ones(1), torch.zeros(1), torch.zeros(1), torch.zeros(1, (V_FULL + 31) // 32, dtype=torch.int32), None, None,
                torch.full((1,), -1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32), torch.full((1,), 5, dtype=torch.int32), stops]
        apply_reference(want, 1, *args)
        c.logit_proc_apply(lg, 1, *[a.cuda() if a is not None else None for a in args])
    torch.cuda.synchronize()
    masked = lg.cpu()[0]
    nan = masked.isnan()
    assert torch.equal(nan, want[0].isnan()) and torch.equal(masked.view(torch.int16)[~nan], want[0].view(torch.int16)[~nan])
    _, cdf, _, kept = TorchDouble.sample_reference(masked, 1.0, 0, 1.0, SEED, 0, 0)
    steps, _ = _tail_steps(cdf, kept, dom, 1000 if _on_device() else 100)
    assert len(steps) >= 50, len(steps)
    toks = _launch_at_steps(c, masked, steps, 1.0)
    xm = masked.float().numpy()
    refused = ~np.isfinite(xm[toks])
    record("sample_chain_refusals", chain=chain, n_allowed=n_allowed, dtype=dt, draws=len(steps), refused=int(refused.sum()))
    assert not refused.any(), f"{int(refused.sum())} refused ids of {len(steps)} draws: {sorted(set(toks[refused].tolist()))[:10]}"
    assert (_mass(cdf)[toks] > 0).all()
