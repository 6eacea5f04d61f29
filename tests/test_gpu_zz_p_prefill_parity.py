"""Prefill parity at the ChatTS-14B and ChatTS-8B widths: every prefill kernel, in every regime the dispatch picks for a packed prompt
of T positions, element by element against its own statement evaluated in float64.

What a prefill layer launches depends on T (chatts_b200/model.py _layers, cts_gemm and cts_gemm_suggest_split in
csrc/gemm_tcgen05.cu, cts_reduce_residual_rmsnorm and cts_qkv_rope_cache in csrc/elementwise.cu): the streaming GEMM, gemm_tn_kernel
with or without split-K partial planes, the persistent GEMM with its L2-grouped raster, the scalar or the vector RoPE kernel, and the
cluster, generic or one-warp-per-row RMSNorm.  _regimes() restates those predicates, scans T and takes the smallest, an interior and
the largest T of every band of identical launches, so a change of heuristic or of SM count moves the T values, not the coverage.

Bounds are element-wise.  Every stage's reference applies the dtype rounding at the kernel's own rounding points; an element may
differ from it by one ulp (of the output dtype, at the reference value) per rounding point, each carried to the output through the
derivative of what follows, plus 2^-20 * sum_k |x_k| |w_k| + 2^-23 * ceil(K / 16) * |sum_k x_k w_k| for every GEMM feeding the element
(fp32 accumulation in the tensor cores, see TRUNC).  Attention is
bounded per query row and head by a multiple of one ulp of max |v| over the row's keys.  Each case records its worst error / bound.

The model-level cases run a two-layer model at full width through prefills whose packed T lands in each regime and compare the logits
(last and every position) and every KV row the prefill wrote with a GPU restatement of oracle.decoder.forward_hidden in float64 and in
the model dtype (the comparative gate of tests/gpu_util.py).

On the CPU shim (tools/shim_gpu_tests.py) the widths shrink to a table that still reaches the generic RMSNorm with two or three
vector slots, the RoPE chunk loop past 65535 rows and a persistent GEMM with more than one L2 group and an uneven last one."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import decoder as od
from tests.gpu_util import ctx, parity_gate, record

pytestmark = pytest.mark.gpu
BF, FP, F64 = torch.bfloat16, torch.float16, torch.float64
DTS = pytest.mark.parametrize("dt", [BF, FP], ids=["bf16", "fp16"])
MANT = {BF: 7, FP: 10}
TINY = {BF: 2.0 ** -133, FP: 2.0 ** -24}           # smallest subnormal: the ulp of zero
ACC = 2.0 ** -20                                   # fp32 accumulation allowance per unit of sum |x_k| |w_k|
# ... plus 2^-23 * ceil(K / 16) * |x w|: the wgmma accumulator does not round each addition to nearest.  A k16 step's products are
# aligned to the largest exponent and truncated into the fp32 running sum, so every step can lose up to one fp32 ulp of that sum, all in
# the same direction.  Without this term the down_proj partial planes (K = 4608 per plane, |x w| = 0.17 sum |x_k| |w_k|) measured up
# to 1.19 x the first allowance alone on an H100; the random-walk part of the error stays inside the first term.
TRUNC = 2.0 ** -23
# The RMSNorm statistic: a lane sums at most 8 x 24 squares in fp32, then a warp / block tree adds <= 13 levels, so the relative
# error of the sum of squares is below 210 * 2^-24 < 2^-16, and 1/sqrtf(.) adds a few fp32 ulps: 2^-16 relative on x * inv.
NORM_REL = 2.0 ** -16
SILU_REL = 2.0 ** -20                              # silu_f = x / (1 + expf(-x)) in fp32: a few fp32 ulps
SILU_D = 1.1                                       # max |silu'(x)| = 1.0998...
ATTN_ULPS = 2.0                                    # see _attn_statement
EPS = 1e-6


def _on_device():
    """False on the CPU shim, where device tensors stay on the host and a GEMM costs seconds: the widths shrink there."""
    return torch.zeros(1).cuda().is_cuda


def _dev():
    return "cuda" if _on_device() else "cpu"


@pytest.fixture(autouse=True, scope="module")
def _peak_memory():
    """Records the file's peak device memory and wall time (it shares the GPU: the references are chunked to stay well under 16 GB)."""
    import time
    t0 = time.time()
    if _on_device():
        torch.cuda.reset_peak_memory_stats()
    yield
    if _on_device():
        record("prefill_parity_file", peak_allocated_gb=torch.cuda.max_memory_allocated() / 2 ** 30, wall_s=time.time() - t0)


# ---------------------------------------------------------------------------------------------------------------- shapes
def _shape(kind):
    """Layer widths.  On the GPU: ChatTS-14B (Qwen2, qkv bias) and ChatTS-8B (Qwen3, q/k norm).  On the shim: the same head layouts and
    head_dim at hidden 1024 / intermediate 768 (a persistent GEMM of k >= 16384 is what reaches uneven L2 groups there, see
    test_persistent_gemm_l2_groups)."""
    from chatts_b200 import ChatTSConfig
    cfg = ChatTSConfig.chatts_14b() if kind == "14b" else ChatTSConfig.chatts_8b()
    s = dict(H=cfg.hidden_size, I=cfg.intermediate_size, nh=cfg.num_attention_heads, nkv=cfg.num_key_value_heads, d=cfg.head_dim,
             bias=cfg.attention_bias, qk_norm=cfg.qk_norm, max_pos=cfg.max_position_embeddings, V=cfg.vocab_size, theta=cfg.rope_theta)
    if not _on_device():
        s.update(H=1024, I=768, V=1000)
    return s


def _cfg(s, layers=2, vocab=512):
    from chatts_b200 import ChatTSConfig
    return ChatTSConfig(hidden_size=s["H"], intermediate_size=s["I"], num_hidden_layers=layers, num_attention_heads=s["nh"],
                        num_key_value_heads=s["nkv"], head_dim=s["d"], vocab_size=vocab, max_position_embeddings=s["max_pos"],
                        rope_theta=s["theta"], attention_bias=s["bias"], qk_norm=s["qk_norm"], ts_token_start_index=vocab - 12,
                        eos_token_id=vocab - 2, pad_token_id=vocab - 1)


# ---------------------------------------------------------------------------------------------------------------- regimes
def _splits(c, s, T):
    """The split-K factors _layers uses (Context.suggest_split, called through the library so the shim's stand-in answers the same)."""
    def sug(n, k, dual=False):
        return int(c.lib.cts_gemm_suggest_split(c.h, n, k, T, int(dual)))
    nqkv = (s["nh"] + 2 * s["nkv"]) * s["d"]
    return dict(qkv=sug(nqkv, s["H"]), o=sug(s["H"], s["nh"] * s["d"]), gu=sug(s["I"], s["H"], True), d=sug(s["H"], s["I"]))


def _signature(c, s, T):
    """The kernels a prefill layer of T packed positions launches, restating the dispatch of _layers, cts_gemm (t <= 32 streaming
    kernel for partials and split-1 EPI_NONE; t > 128 at split 1 persistent; else gemm_tn_kernel), cts_qkv_rope_cache (partials with
    head_dim / 2 a multiple of 32: scalar kernel) and cts_reduce_residual_rmsnorm (a cluster at t <= 256, one warp per row for
    t > 256 without partials, the generic kernel with partials at t > 256)."""
    sp = _splits(c, s, T)

    def partial_gemm():
        return "stream" if T <= 32 else "tn_partial"

    qkv = partial_gemm() if sp["qkv"] > 1 else ("stream" if T <= 32 else "tn" if T <= 128 else "persistent")
    rope = "scalar" if sp["qkv"] > 1 and (s["d"] // 2) % 32 == 0 else "vector"

    def tail(split):
        if split > 1:
            return partial_gemm(), "cluster" if T <= 256 else "generic_partials"
        return ("tn" if T <= 128 else "persistent"), "cluster" if T <= 256 else "rows"
    o, o_norm = tail(sp["o"])
    d, d_norm = tail(sp["d"])
    gu = "persistent_swiglu_il" if T > 128 else partial_gemm() + "+reduce_swiglu"
    return (qkv, rope, o, o_norm, gu, d, d_norm)


# the rows of the regime table at the 14B / 8B widths on an H100 SXM (132 SMs); _regimes asserts that each is hit on this card
TABLE = [("stream", "scalar", "stream", "cluster", "stream+reduce_swiglu", "stream", "cluster"),
         ("tn_partial", "scalar", "tn_partial", "cluster", "tn_partial+reduce_swiglu", "tn_partial", "cluster"),
         ("tn_partial", "scalar", "tn_partial", "cluster", "persistent_swiglu_il", "tn_partial", "cluster"),
         ("persistent", "vector", "tn_partial", "generic_partials", "persistent_swiglu_il", "tn_partial", "generic_partials"),
         ("persistent", "vector", "persistent", "rows", "persistent_swiglu_il", "persistent", "rows")]
T_TOP = 2464


def _regimes(c, s, t_top=T_TOP):
    """[(signature, [T...])]: every band of consecutive T in [1, t_top] with one signature, with its smallest, one interior and its
    largest T."""
    bands, prev = [], None
    for T in range(1, t_top + 1):
        sig = _signature(c, s, T)
        if sig != prev:
            bands.append([sig, T, T])
            prev = sig
        else:
            bands[-1][2] = T
    return [(sig, sorted({lo, (lo + hi) // 2, hi})) for sig, lo, hi in bands]


# ---------------------------------------------------------------------------------------------------------------- rounding
def _ulp(v, dt):
    """One ulp of dt at |v| (v fp64)."""
    a = v.abs()
    _, e = torch.frexp(a)
    u = torch.ldexp(torch.ones_like(a), (e - 1 - MANT[dt]).to(torch.int32))
    return torch.where(a > 0, u, torch.zeros_like(u)).clamp_min(TINY[dt])


def _rnd(v, dt):
    return v.to(torch.float32).to(dt).to(F64)


def _u(v, allow, dt):
    """The ulp of a rounding point whose input is v give or take ``allow`` (the upper binade when v sits next to a power of two)."""
    return _ulp(v.abs() + allow, dt)


def _ratio(got, ref, bound, what):
    """Worst |got - ref| / bound; a non-finite element counts as infinitely far."""
    got = got.to(F64)
    err = (got - ref).abs()
    err = torch.where(torch.isfinite(got), err, torch.full_like(err, float("inf")))
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    worst = float(r.max()) if r.numel() else 0.0
    if not worst <= 1.0:
        i = int(r.flatten().argmax())
        idx = np.unravel_index(i, tuple(r.shape))
        raise AssertionError(f"{what}: error / bound {worst:.3g} at {tuple(int(j) for j in idx)}: got {float(got.flatten()[i])!r}, "
                             f"statement {float(ref.flatten()[i])!r}, bound {float(bound.flatten()[i]):.3g}")
    return worst


class _Case:
    """Collects the worst error / bound of every stage of one case and records them."""

    def __init__(self, name, **meta):
        self.name, self.meta, self.worst = name, meta, {}

    def check(self, stage, got, ref, bound):
        self.worst[stage] = max(self.worst.get(stage, 0.0), _ratio(got, ref, bound, f"{self.name} {self.meta} {stage}"))

    def done(self):
        record(self.name, worst_error_over_bound=max(self.worst.values(), default=0.0), **self.meta,
               **{f"ratio_{k}": v for k, v in self.worst.items()})


# ---------------------------------------------------------------------------------------------------------------- statements
CHUNK = 4096


def _gemm_chunks(x, w, k0=0, k1=None, chunk=CHUNK):
    """(n0, n1, y, allow) over chunks of the weight rows: y = x @ w^T in fp64 over K columns [k0, k1) and its fp32-accumulation
    allowance ACC |x| @ |w|^T + TRUNC ceil(K / 16) |y|."""
    k1 = x.shape[1] if k1 is None else k1
    x64 = x[:, k0:k1].to(F64)
    ax = x64.abs()
    steps = -(-(k1 - k0) // 16)
    for n0 in range(0, w.shape[0], chunk):
        wc = w[n0:n0 + chunk, k0:k1].to(F64)
        y = x64 @ wc.T
        yield n0, n0 + wc.shape[0], y, ACC * (ax @ wc.abs().T) + TRUNC * steps * y.abs()


def _check_gemm(case, stage, x, w, out, dt, bias=None, residual=None):
    """out = rnd(x w^T + bias) (EPI_NONE) or rnd(rnd(x w^T) + residual) (EPI_RESIDUAL; ``residual`` is the input before an in-place
    call)."""
    for n0, n1, y, allow in _gemm_chunks(x, w):
        if bias is not None:
            b = bias[n0:n1].to(F64)
            allow = allow + ACC * b.abs()
            y = y + b
        p = _rnd(y, dt)
        bound = _u(y, allow, dt) + allow
        if residual is not None:
            r = residual[:, n0:n1].to(F64)
            ref = _rnd(p + r, dt)
            bound = bound + _u(p + r, bound, dt)
        else:
            ref = p
        case.check(stage, out[:, n0:n1], ref, bound)


def _check_swiglu_il(case, stage, x, w, out, dt):
    """out = rnd(rnd(silu(rnd(g))) * rnd(u)) with gate row 128 j + i and up row 128 j + 64 + i of the interleaved weight -> column
    64 j + i."""
    for n0, n1, y, a in _gemm_chunks(x, w, chunk=CHUNK // 128 * 128):
        T = y.shape[0]
        y4, a4 = y.view(T, -1, 2, 64), a.view(T, -1, 2, 64)
        g, u, ag, au = y4[:, :, 0].reshape(T, -1), y4[:, :, 1].reshape(T, -1), a4[:, :, 0].reshape(T, -1), a4[:, :, 1].reshape(T, -1)
        _swiglu_statement(case, stage, g, u, ag, au, out[:, n0 // 2:n1 // 2], dt)


def _swiglu_statement(case, stage, g, u, ag, au, got, dt):
    gr, ur = _rnd(g, dt), _rnd(u, dt)
    sg = gr * torch.sigmoid(gr)
    s = _rnd(sg, dt)
    ref = _rnd(s * ur, dt)
    bound = (SILU_D * (ur.abs() + au) * (_u(g, ag, dt) + ag)
             + (ur.abs() + au) * (_ulp(sg, dt) + SILU_REL * sg.abs())
             + s.abs() * (_u(u, au, dt) + au))
    bound = bound + _u(s * ur, bound, dt)
    case.check(stage, got, ref, bound)


def _check_partials(case, stage, x, w, ws, split):
    """Plane s of EPI_PARTIAL_F32 = the fp32 product over K blocks [kb s / S, kb (s + 1) / S)."""
    K, N, T = x.shape[1], w.shape[0], x.shape[0]
    kb = -(-K // 64)
    planes = ws[:split * T * N].view(split, T, N)
    for sidx in range(split):
        k0, k1 = min(K, kb * sidx // split * 64), min(K, kb * (sidx + 1) // split * 64)
        for n0, n1, y, allow in _gemm_chunks(x, w, k0, k1):
            case.check(stage, planes[sidx, :, n0:n1], y, allow + 2.0 ** -140)


def _sum_partials(ws, split, T, N):
    p = ws[:split * T * N].view(split, T, N).to(F64)
    return p.sum(0), ACC * p.abs().sum(0)


def _norm_statement(r, w, dt, allow_r=None):
    """rnd(w * rnd(r * inv)), inv = 1 / sqrt(mean(r^2) + eps) over the last dimension; r fp64.  -> (statement, bound)."""
    inv = 1.0 / torch.sqrt((r * r).mean(-1, keepdim=True) + EPS)
    v = r * inv
    w64 = w.to(F64)
    dv = NORM_REL * v.abs()
    if allow_r is not None:                                 # r carries an allowance: d(r_i inv)/dr_j = inv d_ij - r_i r_j inv^3 / n
        dv = dv + inv * allow_r + r.abs() * inv ** 3 / r.shape[-1] * (r.abs() * allow_r).sum(-1, keepdim=True)
    ref = _rnd(w64 * _rnd(v, dt), dt)
    bound = w64.abs() * (_u(v, dv, dt) + dv)
    return ref, bound + _u(w64 * v, bound, dt)


def _check_norm(case, stage, x, w, out, dt):
    ref, bound = _norm_statement(x.to(F64), w, dt)
    case.check(stage, out, ref, bound)


def _check_reduce_norm(case, stage, ws, split, resid_before, resid_after, w, xn, dt):
    """cts_reduce_residual_rmsnorm with partials: resid_after = rnd(resid + rnd(sum_s part_s)), xn = the norm of resid_after."""
    T, H = resid_before.shape
    P, allow = _sum_partials(ws, split, T, H)
    pr = _rnd(P, dt)
    r = resid_before.to(F64)
    ref = _rnd(r + pr, dt)
    bound = _u(P, allow, dt) + allow
    bound = bound + _u(r + pr, bound, dt)
    case.check(stage + "_residual", resid_after, ref, bound)
    _check_norm(case, stage + "_norm", resid_after, w, xn, dt)


def _rope_statement(x, ax, nh, nkv, d, positions, cos, sin, qn, kn, dt):
    """q / k / v [T, heads, d] as cts_qkv_rope_cache writes them from the rounded projection x (fp64, with allowance ax): the optional
    per-head q / k RMSNorm, then RoPE with every product and the sum rounded.  -> (statement, bound) [T, nh + 2 nkv, d]."""
    T = x.shape[0]
    heads = nh + 2 * nkv
    x, ax = x.reshape(T, heads, d).clone(), ax.reshape(T, heads, d).clone()
    if qn is not None:
        for sl, w in ((slice(0, nh), qn), (slice(nh, nh + nkv), kn)):
            ref, bound = _norm_statement(x[:, sl], w, dt, ax[:, sl])
            x[:, sl], ax[:, sl] = ref, bound
    h = d // 2
    pos = positions.long()
    c, s = cos[pos].to(F64)[:, None], sin[pos].to(F64)[:, None]         # [T, 1, d/2]
    qk = slice(0, nh + nkv)
    x0, x1, a0, a1 = x[:, qk, :h], x[:, qk, h:], ax[:, qk, :h], ax[:, qk, h:]
    out, bnd = x.clone(), ax.clone()
    for dst, xa, xb, aa, ab, sg in ((slice(0, h), x0, x1, a0, a1, -1.0), (slice(h, d), x1, x0, a1, a0, 1.0)):
        pa, pb = xa * c, sg * xb * s
        ra, rb = _rnd(pa, dt), _rnd(pb, dt)
        b = c.abs() * aa + s.abs() * ab
        b = b + _u(pa, c.abs() * aa, dt) + _u(pb, s.abs() * ab, dt)
        out[:, qk, dst] = _rnd(ra + rb, dt)
        bnd[:, qk, dst] = b + _u(ra + rb, b, dt)
    return out, bnd


def _check_rope(case, stage, x, ax, q_out, k_lin, v_lin, kc, vc, slots, page, s, positions, cos, sin, qn, kn, dt):
    nh, nkv, d = s["nh"], s["nkv"], s["d"]
    T = x.shape[0]
    ref, bound = _rope_statement(x, ax, nh, nkv, d, positions, cos, sin, qn, kn, dt)
    case.check(stage + "_q", q_out[:T].view(T, nh, d), ref[:, :nh], bound[:, :nh])
    case.check(stage + "_k", k_lin[:T].view(T, nkv, d), ref[:, nh:nh + nkv], bound[:, nh:nh + nkv])
    case.check(stage + "_v", v_lin[:T].view(T, nkv, d), ref[:, nh + nkv:], bound[:, nh + nkv:])
    _check_cache(case, kc, vc, k_lin[:T], v_lin[:T], slots, page, nkv, d)


def _check_cache(case, kc, vc, k_lin, v_lin, slots, page, nkv, d):
    """Every slot of slot_map holds its row of the linear K / V bit for bit, and every other slot still holds the NaN it was filled
    with."""
    sl = slots.long()
    live = sl >= 0
    for cache, lin in ((kc, k_lin), (vc, v_lin)):
        flat = cache.view(-1, nkv, page, d).transpose(1, 2).reshape(-1, nkv, d)   # slot-major
        got = flat[sl[live]]
        assert torch.equal(got.view(torch.int16), lin.view(-1, nkv, d)[live].view(torch.int16)), f"{case.name}: cache rows differ"
        untouched = torch.ones(flat.shape[0], dtype=torch.bool, device=flat.device)
        untouched[sl[live]] = False
        assert bool(torch.isnan(flat[untouched]).all()), f"{case.name}: a cache slot outside slot_map was written"


# ---------------------------------------------------------------------------------------------------------------- fixtures
def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


def _randn(g, *shape, std=1.0, dt=BF):
    return (torch.randn(*shape, generator=g, device=_dev(), dtype=torch.float32) * std).to(dt).cuda()


def _layer_weights(s, dt, seed):
    """One decoder layer, scaled as synthetic_state_dict scales it (N(0, 0.02^2) projections and biases, U(0.5, 1.5) norms), gate/up
    interleaved per 64 rows as the model stores it."""
    g = _gen(seed)
    H, I, nh, nkv, d = s["H"], s["I"], s["nh"], s["nkv"], s["d"]
    nq = (nh + 2 * nkv) * d
    norm = lambda n: (torch.rand(n, generator=g, device=_dev()) + 0.5).to(dt).cuda()     # noqa: E731
    return dict(wqkv=_randn(g, nq, H, std=0.02, dt=dt), bqkv=_randn(g, nq, std=0.02, dt=dt) if s["bias"] else None,
                wo=_randn(g, H, nh * d, std=0.02, dt=dt), wgu=_randn(g, 2 * I, H, std=0.02, dt=dt), wd=_randn(g, H, I, std=0.02, dt=dt),
                ln1=norm(H), ln2=norm(H), qn=norm(d) if s["qk_norm"] else None, kn=norm(d) if s["qk_norm"] else None)


def _rope_tabs(s, dt, n_pos):
    from chatts_b200.model import rope_tables
    return rope_tables(_cfg(s), n_pos, dt, _dev())


# ---------------------------------------------------------------------------------------------------------------- regimes test
@pytest.mark.parametrize("kind", ["14b", "8b"])
def test_every_regime_of_the_table_is_hit(kind):
    """The band scan finds each row of the regime table on this card (a change of card or heuristic that drops one fails here)."""
    c, s = ctx(), _shape(kind)
    regs = _regimes(c, s)
    sigs = [sig for sig, _ in regs]
    record("prefill_regimes", kind=kind, bands=[dict(sig="/".join(sig), T=ts) for sig, ts in regs])
    if _on_device():
        for row in TABLE:
            assert row in sigs, f"{kind}: regime {row} is not reached by any T <= {T_TOP}; bands: {regs}"


# ---------------------------------------------------------------------------------------------------------------- stage tests
def _layer_stage_case(c, s, W, dt, T, kind, g):
    """One prefill layer at T packed positions, each stage launched as _layers launches it and checked on its own inputs."""
    H, I, nh, nkv, d = s["H"], s["I"], s["nh"], s["nkv"], s["d"]
    nq = (nh + 2 * nkv) * d
    sp = _splits(c, s, T)
    sig = _signature(c, s, T)
    case = _Case("prefill_stage", kind=kind, dtype=str(dt).split(".")[-1], T=T, regime="/".join(sig), splits=str(sp))
    from chatts_b200._cabi import EPI_NONE, EPI_PARTIAL_F32, EPI_RESIDUAL, EPI_SWIGLU_IL
    page, n_pos = 64, s["max_pos"]
    cos, sin = _rope_tabs(s, dt, n_pos)
    h = _randn(g, T, H, dt=dt)
    xn = torch.full((T, H), float("nan"), device=h.device, dtype=dt)
    ws_n = max(sp["qkv"] * T * nq, sp["o"] * T * H, sp["gu"] * T * 2 * I, sp["d"] * T * H, T * H)
    ws = torch.full((ws_n,), float("nan"), device=h.device)
    positions = torch.randint(0, n_pos, (T,), generator=g, device=_dev()).to(torch.int32).cuda()
    n_pages = -(-T // page) + 2
    perm = torch.randperm(n_pages * page, generator=g, device=_dev())[:T].to(torch.int32)
    perm[::7] = -1
    slots = perm.cuda()
    kc = torch.full((n_pages, nkv, page, d), float("nan"), device=h.device, dtype=dt)
    vc = torch.full_like(kc, float("nan"))
    q = torch.full((T, nh * d), float("nan"), device=h.device, dtype=dt)
    k_lin = torch.full((T, nkv * d), float("nan"), device=h.device, dtype=dt)
    v_lin = torch.full_like(k_lin, float("nan"))

    # input RMSNorm
    c.reduce_residual_rmsnorm(None, 0, h, None, W["ln1"], EPS, xn, t=T)
    _check_norm(case, "norm_in", h, W["ln1"], xn, dt)
    # QKV + bias + RoPE + KV write
    rope = (positions, cos, sin, slots, q, kc, vc, k_lin, v_lin, T, nh, nkv, d, page, W["qn"], W["kn"], EPS)
    if sp["qkv"] > 1:
        c.gemm(xn, W["wqkv"], ws, epilogue=EPI_PARTIAL_F32, split_k=sp["qkv"], t=T)
        _check_partials(case, "qkv_partials", xn, W["wqkv"], ws, sp["qkv"])
        c.qkv_rope_cache(ws, True, sp["qkv"], W["bqkv"], *rope)
        P, allow = _sum_partials(ws, sp["qkv"], T, nq)
        if W["bqkv"] is not None:
            b = W["bqkv"].to(F64)
            P, allow = P + b, allow + ACC * b.abs()
        x, ax = _rnd(P, dt), _u(P, allow, dt) + allow
    else:
        qkv = torch.full((T, nq), float("nan"), device=h.device, dtype=dt)
        c.gemm(xn, W["wqkv"], qkv, bias=W["bqkv"], epilogue=EPI_NONE, t=T)
        _check_gemm(case, "qkv", xn, W["wqkv"], qkv, dt, bias=W["bqkv"])
        c.qkv_rope_cache(qkv, False, 1, None, *rope)
        x, ax = qkv.to(F64), torch.zeros(T, nq, dtype=F64, device=h.device)
        if W["qn"] is None:                                # the same tables and rounding points as the oracle: bit for bit
            oc, osn = torch.cat([cos, cos], -1)[positions.long()], torch.cat([sin, sin], -1)[positions.long()]
            qe, ke = od.apply_rope(qkv[:, :nh * d].view(T, nh, d), qkv[:, nh * d:(nh + nkv) * d].view(T, nkv, d), oc, osn)
            assert torch.equal(q.view(T, nh, d), qe) and torch.equal(k_lin.view(T, nkv, d), ke)
    _check_rope(case, "rope", x, ax, q, k_lin, v_lin, kc, vc, slots, page, s, positions, cos, sin, W["qn"], W["kn"], dt)
    # o_proj + residual + post-attention RMSNorm (the attention output is any 16-bit input here: test_attn_prefill checks it)
    ao = _randn(g, T, nh * d, dt=dt)
    h0 = h.clone()
    if sp["o"] > 1:
        c.gemm(ao, W["wo"], ws, epilogue=EPI_PARTIAL_F32, split_k=sp["o"], t=T)
        _check_partials(case, "o_partials", ao, W["wo"], ws, sp["o"])
        c.reduce_residual_rmsnorm(ws, sp["o"], h, h, W["ln2"], EPS, xn, t=T)
        _check_reduce_norm(case, "o_tail", ws, sp["o"], h0, h, W["ln2"], xn, dt)
    else:
        c.gemm(ao, W["wo"], h, residual=h, epilogue=EPI_RESIDUAL, t=T)
        _check_gemm(case, "o_residual", ao, W["wo"], h, dt, residual=h0)
        c.reduce_residual_rmsnorm(None, 0, h, None, W["ln2"], EPS, xn, t=T)
        _check_norm(case, "o_norm", h, W["ln2"], xn, dt)
    # gate/up + SwiGLU
    act = torch.full((T, I), float("nan"), device=h.device, dtype=dt)
    if T > 128:
        c.gemm(xn, W["wgu"], act, epilogue=EPI_SWIGLU_IL, t=T)
        _check_swiglu_il(case, "swiglu_il", xn, W["wgu"], act, dt)
    else:
        c.gemm(xn, W["wgu"], ws, epilogue=EPI_PARTIAL_F32, split_k=sp["gu"], t=T)
        _check_partials(case, "gu_partials", xn, W["wgu"], ws, sp["gu"])
        c.reduce_swiglu(ws, sp["gu"], T, I, act, interleaved=True)
        P, allow = _sum_partials(ws, sp["gu"], T, 2 * I)
        P4, A4 = P.view(T, -1, 2, 64), allow.view(T, -1, 2, 64)
        _swiglu_statement(case, "reduce_swiglu", P4[:, :, 0].reshape(T, I), P4[:, :, 1].reshape(T, I), A4[:, :, 0].reshape(T, I),
                          A4[:, :, 1].reshape(T, I), act, dt)
    # down_proj + residual + the next layer's input RMSNorm
    h0 = h.clone()
    if sp["d"] > 1:
        c.gemm(act, W["wd"], ws, epilogue=EPI_PARTIAL_F32, split_k=sp["d"], t=T)
        _check_partials(case, "down_partials", act, W["wd"], ws, sp["d"])
        c.reduce_residual_rmsnorm(ws, sp["d"], h, h, W["ln1"], EPS, xn, t=T)
        _check_reduce_norm(case, "down_tail", ws, sp["d"], h0, h, W["ln1"], xn, dt)
    else:
        c.gemm(act, W["wd"], h, residual=h, epilogue=EPI_RESIDUAL, t=T)
        _check_gemm(case, "down_residual", act, W["wd"], h, dt, residual=h0)
        c.reduce_residual_rmsnorm(None, 0, h, None, W["ln1"], EPS, xn, t=T)
        _check_norm(case, "down_norm", h, W["ln1"], xn, dt)
    case.done()
    return case


def _stage_ts(c, s):
    if _on_device():
        return [t for _, ts in _regimes(c, s) for t in ts]
    return [5, 40, 131, 300]                                # the shim: one T per kind of launch at the reduced widths


@DTS
@pytest.mark.parametrize("kind", ["14b", "8b"])
def test_prefill_layer_stages_in_every_regime(kind, dt):
    """Every stage of a prefill layer (input norm, QKV with bias or partial planes, RoPE + KV write with the q/k norm of the 8B, o_proj
    EPI_RESIDUAL in place or partials + reduce_residual_rmsnorm, gate_up EPI_SWIGLU_IL or partials + reduce_swiglu(interleaved),
    down_proj likewise) at the smallest, an interior and the largest T of every regime band, against its fp64 statement."""
    c, s = ctx(), _shape(kind)
    W = _layer_weights(s, dt, seed=11 if kind == "14b" else 12)
    g = _gen(5)
    seen = set()
    for T in _stage_ts(c, s):
        seen.add(_layer_stage_case(c, s, W, dt, T, kind, g).meta["regime"])
    if _on_device():
        assert {"/".join(r) for r in TABLE} <= seen


# ---------------------------------------------------------------------------------------------------------------- lm_head
@DTS
@pytest.mark.parametrize("kind", ["14b", "8b"])
def test_lm_head_at_the_full_vocabulary(kind, dt):
    """logits = rnd(xn @ lm_head^T) at n = 152064 / 151936: T = B last positions (streaming kernel), a 100-row and a 1024-row chunk
    of the prompt-logprob path (gemm_tn_kernel / persistent) and every position of a 2464-position prompt (persistent, 75 L2 groups
    with an uneven last one)."""
    from chatts_b200._cabi import EPI_NONE
    c, s = ctx(), _shape(kind)
    g = _gen(21)
    lm = _randn(g, s["V"], s["H"], std=0.02, dt=dt)
    for T in ([4, 100, 1024, T_TOP] if _on_device() else [4, 40]):
        xn = _randn(g, T, s["H"], dt=dt)
        logits = torch.full((T, s["V"]), float("nan"), device=lm.device, dtype=dt)
        c.gemm(xn, lm, logits, epilogue=EPI_NONE, t=T)
        case = _Case("prefill_lm_head", kind=kind, dtype=str(dt).split(".")[-1], T=T, n=s["V"])
        _check_gemm(case, "lm_head", xn, lm, logits, dt)
        case.done()


# ---------------------------------------------------------------------------------------------------------------- RMSNorm
@DTS
@pytest.mark.parametrize("h", [4096, 5120])
@pytest.mark.parametrize("kernel", ["cluster", "generic_partials", "generic_plain", "rows"])
def test_rmsnorm_kernels(kernel, h, dt):
    """The three RMSNorm kernels as the model calls them (resid_out == resid_in), at the 8B and 14B widths: the cluster kernel
    (t <= 256, with and without partials), the generic one-CTA-per-token kernel with NV = 2 / 3 vector slots (partials at t > 256, and
    without partials when resid_out is a different buffer), the one-warp-per-row kernel (t > 256, no partials)."""
    c = ctx()
    g = _gen(31 + h)
    T = {"cluster": 256, "generic_partials": 300, "generic_plain": 259, "rows": 1000}[kernel]
    split = 3 if kernel in ("cluster", "generic_partials") else 0
    resid = _randn(g, T, h, dt=dt)
    w = (torch.rand(h, generator=g, device=_dev()) + 0.5).to(dt).cuda()
    xn = torch.full((T, h), float("nan"), device=resid.device, dtype=dt)
    case = _Case("prefill_rmsnorm", kernel=kernel, h=h, dtype=str(dt).split(".")[-1], T=T)
    r0 = resid.clone()
    if split:
        ws = (torch.randn(split * T * h, generator=g, device=_dev()) * 0.3).cuda()
        c.reduce_residual_rmsnorm(ws, split, resid, resid, w, EPS, xn, t=T)
        _check_reduce_norm(case, kernel, ws, split, r0, resid, w, xn, dt)
    elif kernel == "generic_plain":
        out = torch.full_like(resid, float("nan"))
        c.reduce_residual_rmsnorm(None, 0, resid, out, w, EPS, xn, t=T)
        assert torch.equal(out, r0)
        _check_norm(case, kernel, r0, w, xn, dt)
    else:
        c.reduce_residual_rmsnorm(None, 0, resid, resid, w, EPS, xn, t=T)
        assert torch.equal(resid, r0)
        _check_norm(case, kernel, r0, w, xn, dt)
    case.done()


# ---------------------------------------------------------------------------------------------------------------- RoPE / KV write
@DTS
@pytest.mark.parametrize("partial", [True, False], ids=["partials", "plain"])
@pytest.mark.parametrize("kind", ["14b", "8b"])
def test_qkv_rope_cache_at_full_width(kind, partial, dt):
    """Both RoPE kernels at 40/8 (qkv bias) and 32/8 heads (Qwen3 q/k norm), positions drawn over [0, max_position_embeddings) with
    the model's tables: q, the linear K / V rows and every cache slot against the statement; no other slot written."""
    c, s = ctx(), _shape(kind)
    nh, nkv, d, page = s["nh"], s["nkv"], s["d"], 16
    nq = (nh + 2 * nkv) * d
    T = 300 if _on_device() else 37
    g = _gen(41)
    cos, sin = _rope_tabs(s, dt, s["max_pos"])
    positions = torch.randint(0, s["max_pos"], (T,), generator=g, device=_dev()).to(torch.int32)
    positions[:3] = torch.tensor([0, s["max_pos"] - 1, 1], dtype=torch.int32)
    positions = positions.cuda()
    n_pages = -(-T // page) + 3
    slots = torch.randperm(n_pages * page, generator=g, device=_dev())[:T].to(torch.int32)
    slots[1::5] = -1
    slots = slots.cuda()
    bias = _randn(g, nq, std=0.02, dt=dt) if s["bias"] else None
    qn = (torch.rand(d, generator=g, device=_dev()) + 0.5).to(dt).cuda() if s["qk_norm"] else None
    kn = (torch.rand(d, generator=g, device=_dev()) + 0.5).to(dt).cuda() if s["qk_norm"] else None
    kc = torch.full((n_pages, nkv, page, d), float("nan"), device=positions.device, dtype=dt)
    vc = torch.full_like(kc, float("nan"))
    q = torch.full((T, nh * d), float("nan"), device=positions.device, dtype=dt)
    k_lin = torch.full((T, nkv * d), float("nan"), device=positions.device, dtype=dt)
    v_lin = torch.full_like(k_lin, float("nan"))
    case = _Case("prefill_rope", kind=kind, partial=partial, dtype=str(dt).split(".")[-1], T=T)
    if partial:
        S = 3
        ws = (torch.randn(S, T, nq, generator=g, device=_dev()) * 0.7).cuda()
        c.qkv_rope_cache(ws, True, S, bias, positions, cos, sin, slots, q, kc, vc, k_lin, v_lin, T, nh, nkv, d, page, qn, kn, EPS)
        P, allow = _sum_partials(ws.view(-1), S, T, nq)
        if bias is not None:
            P, allow = P + bias.to(F64), allow + ACC * bias.to(F64).abs()
        x, ax = _rnd(P, dt), _u(P, allow, dt) + allow
    else:
        src = _randn(g, T, nq, dt=dt)
        c.qkv_rope_cache(src, False, 1, None, positions, cos, sin, slots, q, kc, vc, k_lin, v_lin, T, nh, nkv, d, page, qn, kn, EPS)
        x, ax = src.to(F64), torch.zeros(T, nq, dtype=F64, device=src.device)
    _check_rope(case, "rope", x, ax, q, k_lin, v_lin, kc, vc, slots, page, s, positions, cos, sin, qn, kn, dt)
    case.done()


@DTS
def test_qkv_rope_cache_past_65535_rows(dt):
    """t > 65535 folds into chunks of the y grid dimension: every chunk must offset src, positions, slot_map, q and the linear K / V by
    its first row.  Every q row, every linear K / V row and every cache slot is written, and no other slot."""
    c = ctx()
    nh, nkv, d, page = 2, 1, 64, 16
    s = dict(nh=nh, nkv=nkv, d=d, max_pos=4096, theta=1e6, H=nh * d, I=64, bias=False, qk_norm=False)
    T = 65535 + 700
    g = _gen(51)
    from chatts_b200.model import rope_tables
    from chatts_b200 import ChatTSConfig
    cos, sin = rope_tables(ChatTSConfig.tiny(head_dim=d, num_attention_heads=nh, num_key_value_heads=nkv, rope_theta=1e6), 4096, dt, _dev())
    positions = torch.randint(0, 4096, (T,), generator=g, device=_dev()).to(torch.int32).cuda()
    n_pages = -(-T // page) + 2
    slots = torch.randperm(n_pages * page, generator=g, device=_dev())[:T].to(torch.int32)
    slots[::101] = -1
    slots = slots.cuda()
    src = _randn(g, T, (nh + 2 * nkv) * d, dt=dt)
    kc = torch.full((n_pages, nkv, page, d), float("nan"), device=src.device, dtype=dt)
    vc = torch.full_like(kc, float("nan"))
    q = torch.full((T, nh * d), float("nan"), device=src.device, dtype=dt)
    k_lin = torch.full((T, nkv * d), float("nan"), device=src.device, dtype=dt)
    v_lin = torch.full_like(k_lin, float("nan"))
    c.qkv_rope_cache(src, False, 1, None, positions, cos, sin, slots, q, kc, vc, k_lin, v_lin, T, nh, nkv, d, page)
    case = _Case("prefill_rope_chunked", dtype=str(dt).split(".")[-1], T=T)
    oc, osn = torch.cat([cos, cos], -1)[positions.long()], torch.cat([sin, sin], -1)[positions.long()]
    qe, ke = od.apply_rope(src[:, :nh * d].view(T, nh, d), src[:, nh * d:(nh + nkv) * d].view(T, nkv, d), oc, osn)
    assert torch.equal(q.view(T, nh, d), qe), "q rows differ from oracle.decoder.apply_rope"
    assert torch.equal(k_lin.view(T, nkv, d), ke), "linear K rows differ from oracle.decoder.apply_rope"
    assert torch.equal(v_lin, src[:, (nh + nkv) * d:]), "linear V rows differ from the input"
    _check_cache(case, kc, vc, k_lin, v_lin, slots, page, nkv, d)
    case.worst["rope"] = 0.0
    case.done()


# ---------------------------------------------------------------------------------------------------------------- persistent GEMM
def _l2_groups(n, k):
    """(groups, feature tiles per group, tiles in the last group) of launch_persistent's L2 raster."""
    tiles = -(-n // 128)
    gmax = max(1, (20 << 20) // (128 * k * 2))
    groups = -(-tiles // gmax)
    gm = -(-tiles // groups)
    return groups, gm, tiles - (groups - 1) * gm


@DTS
@pytest.mark.parametrize("epi", ["none_bias", "residual", "swiglu_il"])
def test_persistent_gemm_l2_groups(epi, dt):
    """The persistent GEMM with several L2 groups and an uneven last one (tile_coords' gm_here branch), every epilogue it serves in a
    prefill, on an output pre-filled with NaN: a tile computed twice or never shows.  On the GPU at 14B widths (o_proj 40 tiles in
    14/14/12, gate_up 216 tiles in 13 x 16 + 8; the QKV width 7168 over down_proj's K = 13824, 56 tiles in 11 x 5 + 1, for the bias on
    the last feature tile); on the shim at the smallest weight over 20 MB."""
    from chatts_b200._cabi import EPI_NONE, EPI_RESIDUAL, EPI_SWIGLU_IL
    c = ctx()
    g = _gen(61)
    if _on_device():
        n, k, T = {"none_bias": (7168, 13824), "residual": (5120, 5120), "swiglu_il": (27648, 5120)}[epi] + (700,)
    else:
        n, k, T = (640, 20480, 200) if epi != "swiglu_il" else (640, 20480, 130)
    groups, gm, last = _l2_groups(n, k)
    assert groups > 1 and last < gm, (n, k, groups, gm, last)
    x = _randn(g, T, k, dt=dt)
    w = _randn(g, n, k, std=0.02, dt=dt)
    case = _Case("prefill_persistent_gemm", epi=epi, dtype=str(dt).split(".")[-1], T=T, n=n, k=k, groups=groups, group_m=gm, last=last)
    if epi == "swiglu_il":
        out = torch.full((T, n // 2), float("nan"), device=x.device, dtype=dt)
        c.gemm(x, w, out, epilogue=EPI_SWIGLU_IL, t=T)
        _check_swiglu_il(case, epi, x, w, out, dt)
    elif epi == "residual":
        out = _randn(g, T, n, dt=dt)
        r0 = out.clone()
        c.gemm(x, w, out, residual=out, epilogue=EPI_RESIDUAL, t=T)
        _check_gemm(case, epi, x, w, out, dt, residual=r0)
    else:
        bias = _randn(g, n, std=0.5, dt=dt)
        out = torch.full((T, n), float("nan"), device=x.device, dtype=dt)
        c.gemm(x, w, out, bias=bias, epilogue=EPI_NONE, t=T)
        _check_gemm(case, epi, x, w, out, dt, bias=bias)
    case.done()


# ---------------------------------------------------------------------------------------------------------------- attention
def _attn_statement(q, k, v, lens, nh, nkv, d, scale, dt):
    """Causal GQA attention per sequence in fp64, and the per (row, head) bound ATTN_ULPS ulps of max |v| over the row's keys.  The
    kernel rounds the probabilities to the model dtype for the P V product (the oracle rounds them after normalising), which moves an
    output by at most half an ulp of max |v| (relative 2^-9 / 2^-12 of sum_j p_j |v_j|); the output rounding adds half an ulp of the
    output <= max |v|.  Two ulps leave room for the fp32 scores and the online-softmax rescaling."""
    T = q.shape[0]
    out = torch.empty(T, nh, d, dtype=F64, device=q.device)
    bound = torch.empty(T, nh, 1, dtype=F64, device=q.device)
    rep = nh // nkv
    c0 = 0
    for L in lens:
        qs = q[c0:c0 + L].view(L, nh, d).to(F64)
        ks, vs = k[c0:c0 + L].view(L, nkv, d).to(F64), v[c0:c0 + L].view(L, nkv, d).to(F64)
        causal = torch.ones(L, L, dtype=torch.bool, device=q.device).triu(1)
        for j in range(nkv):
            sc = torch.einsum("trd,sd->rts", qs[:, j * rep:(j + 1) * rep], ks[:, j]) * scale
            p = torch.softmax(sc.masked_fill(causal, float("-inf")), -1)
            out[c0:c0 + L, j * rep:(j + 1) * rep] = torch.einsum("rts,sd->trd", p, vs[:, j])
            vmax = vs[:, j].abs().amax(-1).cummax(0).values
            bound[c0:c0 + L, j * rep:(j + 1) * rep] = ATTN_ULPS * _ulp(vmax, dt)[:, None, None]
            del sc, p
        c0 += L
    return out, bound


ATTN_LENS = {"edges": [1, 63, 64, 65, 127, 128, 129], "576x8": [576] * 8, "2464x2": [2464] * 2, "long": [4500, 37]}


@DTS
@pytest.mark.parametrize("lens", list(ATTN_LENS), ids=list(ATTN_LENS))
@pytest.mark.parametrize("kind", ["14b", "8b"])
def test_attn_prefill_ragged_and_isolated(kind, lens, dt):
    """cts_attn_prefill at 40/8 and 32/8 heads over a ragged batch, with q / k / v buffers longer than the batch (as the model passes
    its activation buffers): the output of every row and head against the fp64 statement; bit-identical when every row past T holds
    NaN, or +-the largest finite value, instead of zero; finite; the rows past T of the output untouched.  A neighbour sequence whose V
    rows sit next to the largest finite value leaves the other sequences' outputs bit-identical."""
    c, s = ctx(), _shape(kind)
    nh, nkv, d = s["nh"], s["nkv"], s["d"]
    lens = ATTN_LENS[lens] if _on_device() else [1, 63, 64, 65, 129]
    T, pad = sum(lens), 160
    g = _gen(71)
    scale = 1.0 / math.sqrt(d)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32).cuda()
    q, k, v = (_randn(g, T + pad, n * d, dt=dt) for n in (nh, nkv, nkv))
    fmax = torch.finfo(dt).max

    def run(fill, vv=None):
        bufs = [t.clone() for t in (q, k, v if vv is None else vv)]
        for b in bufs:
            if fill == "nan":
                b[T:] = float("nan")
            elif fill == "max":
                b[T:] = fmax
                b[T:, 1::2] = -fmax
            else:
                b[T:] = 0
        out = torch.full((T + pad, nh * d), 3.0, device=q.device, dtype=dt)
        c.attn_prefill(bufs[0], bufs[1], bufs[2], cu, len(lens), max(lens), nh, nkv, d, scale, out)
        assert bool((out[T:] == 3.0).all()), "cts_attn_prefill wrote rows past the batch"
        return out[:T]

    base = run("zero")
    assert bool(torch.isfinite(base).all())
    for fill in ("nan", "max"):
        assert torch.equal(run(fill), base), f"rows past T filled with {fill} moved the output"
    ref, bound = _attn_statement(q[:T], k[:T], v[:T], lens, nh, nkv, d, scale, dt)
    case = _Case("prefill_attention", kind=kind, lens=str(lens[:8]), dtype=str(dt).split(".")[-1], T=T)
    case.check("attention", base.view(T, nh, d), ref, bound.expand_as(ref))
    # a neighbour sequence (the second) whose V rows are next to the largest finite value
    b0, b1 = int(cu[1]), int(cu[2])
    v2 = v.clone()
    v2[b0:b1] = (fmax * 0.99) * torch.sign(v2[b0:b1].float()).to(dt)
    big = run("zero", v2)
    assert torch.equal(big[:b0], base[:b0]) and torch.equal(big[b1:], base[b1:]), "a neighbour's V rows moved another sequence"
    case.done()


# ---------------------------------------------------------------------------------------------------------------- model level
def _forward_hidden(x, Wf, cfg):
    """oracle.decoder.forward_hidden for one sequence from position 0, on the device of x (the oracle builds its causal mask on the
    CPU): the same statement, the attention evaluated a KV head at a time.  Wf(name) -> the weight in the evaluation dtype.
    -> (final-norm hidden [T, H], [K per layer], [V per layer])."""
    nh, nkv, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    eps = float(cfg.rms_norm_eps)
    T = x.shape[0]
    cos, sin = od.rope_tables(cfg.to_dict(), T, x.dtype)
    cos, sin = cos.to(x.device), sin.to(x.device)
    causal = torch.ones(T, T, dtype=torch.bool, device=x.device).triu(1)
    rep = nh // nkv
    h, ks, vs = x, [], []
    for l in range(cfg.num_hidden_layers):
        pre = f"model.layers.{l}."
        r = h
        a = od.rms_norm(h, Wf(pre + "input_layernorm.weight"), eps)
        q = F.linear(a, Wf(pre + "self_attn.q_proj.weight"), Wf(pre + "self_attn.q_proj.bias")).view(T, nh, d)
        k = F.linear(a, Wf(pre + "self_attn.k_proj.weight"), Wf(pre + "self_attn.k_proj.bias")).view(T, nkv, d)
        v = F.linear(a, Wf(pre + "self_attn.v_proj.weight"), Wf(pre + "self_attn.v_proj.bias")).view(T, nkv, d)
        if cfg.qk_norm:
            q = od.rms_norm(q, Wf(pre + "self_attn.q_norm.weight"), eps)
            k = od.rms_norm(k, Wf(pre + "self_attn.k_norm.weight"), eps)
        q, k = od.apply_rope(q, k, cos, sin)
        ks.append(k)
        vs.append(v)
        o = torch.empty(T, nh, d, dtype=x.dtype, device=x.device)
        for j in range(nkv):                               # modeling_qwen2.py eager attention, one KV head's query group at a time
            w = torch.einsum("thd,sd->hts", q[:, j * rep:(j + 1) * rep], k[:, j]) * (d ** -0.5)
            w = F.softmax(w.masked_fill(causal, float("-inf")), dim=-1, dtype=torch.float32).to(x.dtype)
            o[:, j * rep:(j + 1) * rep] = torch.einsum("hts,sd->thd", w, v[:, j])
            del w
        h = r + F.linear(o.reshape(T, nh * d), Wf(pre + "self_attn.o_proj.weight"))
        r = h
        a = od.rms_norm(h, Wf(pre + "post_attention_layernorm.weight"), eps)
        gt = F.silu(F.linear(a, Wf(pre + "mlp.gate_proj.weight"))) * F.linear(a, Wf(pre + "mlp.up_proj.weight"))
        h = r + F.linear(gt, Wf(pre + "mlp.down_proj.weight"))
    return od.rms_norm(h, Wf("model.norm.weight"), eps), ks, vs


MODEL_CASES = {"20": [20], "100": [100], "129+100": [129, 100], "300": [300], "576x8": [576] * 8, "2464": [2464]}
# Fixed bounds of the comparative gate (tests/gpu_util.py, gate (b)) against the same-dtype restatement, two full-width layers, a
# 512-token vocabulary; gate (a) against the fp64 restatement is the one that scales with the model's own rounding floor
MODEL_BOUND = {BF: dict(logits=4e-2, kv=3e-2), FP: dict(logits=5e-3, kv=4e-3)}
KV_RATIO = 1.5          # as in test_gpu_zz_g_decode_parity: the KV rows are gated element-wise and carry the earlier layer's rounding


@DTS
@pytest.mark.parametrize("kind", ["14b", "8b"])
def test_model_prefill_in_every_regime_matches_the_oracle(kind, dt):
    """A two-layer full-width model prefills packed batches whose T lands in each regime; the last-position logits, every position's
    logits (all_logits, as forward(logits_to_keep=0) asks) and every KV row the prefill wrote, against the restated oracle in fp64 and
    in the model dtype.  This is what shows that _layers wires each regime: the partial buffer, the split and t=."""
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    s = _shape(kind)
    cfg = _cfg(s)
    sd = synthetic_state_dict(cfg, seed=77, device=_dev(), dtype=dt)
    sd = {k2: v2 for k2, v2 in sd.items() if not k2.startswith("ts_encoder.")}
    cases = MODEL_CASES if _on_device() else {"20": [20], "129+100": [129, 100]}
    maxb, maxs = max(len(v2) for v2 in cases.values()), max(max(v2) for v2 in cases.values()) + 64
    model = ChatTSForCausalLM(cfg, sd, dtype=dt, max_batch=maxb, max_seq_len=maxs, page_size=64, use_cuda_graph=False)
    c = ctx()
    f64 = lambda name: None if name not in sd else sd[name].to(F64)        # noqa: E731
    same = lambda name: sd.get(name)                                       # noqa: E731
    lm_name = "lm_head.weight" if "lm_head.weight" in sd else "model.embed_tokens.weight"
    g = torch.Generator().manual_seed(3)
    for cname, lens in cases.items():
        T = sum(lens)
        sig = "/".join(_signature(c, s, T))
        ids = [torch.randint(0, cfg.ts_token_start_index - 20, (L,), generator=g) for L in lens]
        mx = max(lens)
        inp = torch.full((len(lens), mx), cfg.pad_token_id, dtype=torch.long)
        am = torch.zeros(len(lens), mx, dtype=torch.long)
        for b, t in enumerate(ids):
            inp[b, mx - len(t):], am[b, mx - len(t):] = t, 1
        _, _, counts, lay = model._prepare_inputs(inp, am, None)
        pts, held = model._alloc_pages(lay.lens, 0)
        try:
            last = model._prefill(lay, counts, None, pts).float().cpu()
            every = model._prefill(lay, counts, None, pts, all_logits=True).float().cpu()
            kv = model.kv.clone()
        finally:
            model.pool.release(held)
        got_l, got_a, r_l, r_a, r64_l, r64_a = [], [], [], [], [], []
        kv_got, kv_ref, kv_64 = [[] for _ in range(2)], [[] for _ in range(2)], [[] for _ in range(2)]
        c0 = 0
        for b, t in enumerate(ids):
            L = len(t)
            emb = sd["model.embed_tokens.weight"][t.to(sd["model.embed_tokens.weight"].device)]
            outs = []
            for Wf, x in ((same, emb), (f64, emb.to(F64))):
                hn, ks, vs = _forward_hidden(x, Wf, cfg)
                lg = F.linear(hn, Wf(lm_name)).float().cpu()
                outs.append((lg, ks, vs))
                del hn
            got_l.append(last[b]); r_l.append(outs[0][0][-1]); r64_l.append(outs[1][0][-1])
            got_a.append(every[c0:c0 + L]); r_a.append(outs[0][0]); r64_a.append(outs[1][0])
            pos = torch.arange(L)
            pg = torch.from_numpy(pts[b]).long()[pos // 64].to(kv.device)
            for l in range(cfg.num_hidden_layers):
                for i in range(2):
                    kv_got[l].append(kv[l, i, pg, :, (pos % 64).to(kv.device)].float().cpu())
                    kv_ref[l].append((outs[0][1] if i == 0 else outs[0][2])[l].float().cpu())
                    kv_64[l].append((outs[1][1] if i == 0 else outs[1][2])[l].float().cpu())
            c0 += L
        name = f"prefill_model_{kind}_{cname}"
        bnd = MODEL_BOUND[dt]
        parity_gate(name + "_last_logits", got_l, r_l, r64_l, dt, bnd["logits"], T=T, regime=sig)
        parity_gate(name + "_all_logits", got_a, r_a, r64_a, dt, bnd["logits"], T=T, regime=sig)
        for l in range(cfg.num_hidden_layers):
            parity_gate(name + f"_kv_layer{l}", kv_got[l], kv_ref[l], kv_64[l], dt, bnd["kv"], ratio=KV_RATIO, T=T, regime=sig)
