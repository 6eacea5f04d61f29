"""cts_sample_advance_rows (csrc/sampling.cu: the sampling kernel with every parameter read per row) and the continuous engine's
per-request sampling on the GPU.

  K1  uniform parameters with draw_key[b] = b and draw_step[b] = step_ptr[0]: bit-identical tokens and advance state to
      cts_sample_advance, on the far-tail, edge and odd-vocabulary rows of test_gpu_zz_n_sampling_dist.py, in bf16 and fp16.
  K2  one launch mixing greedy rows (ties, all -inf, NaN) and sampled rows of different temperature / top_k / top_p / seed / draw:
      greedy rows are cts_greedy_advance's token, sampled rows the statement's draw (tests/cabi_double.py ``sample_reference``) where
      the draw-for-draw precondition holds, and draw_step advances by exactly 1 on every row.
  K3  a chi-square per row group over many launches at V = 152 064, -inf tails included; the statement's own draws pass the same
      thresholds and no token of zero mass is ever returned.
  K4  cts_struct_mask_apply / cts_logit_proc_apply followed by the rows kernel never returns a refused id.
  K5  200 captured launches replay bit-identically.
  E1  the continuous engine: greedy and sampled requests with different parameters and seeds, one with processors and one with
      logprobs, give exactly what each gets served alone at the same width, in any submission order, and the pool is returned.
"""
import numpy as np
import pytest
import torch

from tests.cabi_double import TorchDouble
from tests.gpu_util import ctx, record
from tests.structured_double import pack_bits
from tests.test_gpu_zz_n_sampling_dist import (DTYPES, SEED, V_FULL, _bins_by_logit, _chi2, _chi2_limit, _greedy, _mass, _on_device,
                                               _row, _statement_tokens, _stress_row, _uniforms)

pytestmark = pytest.mark.gpu
I32 = dict(dtype=torch.int32, device="cuda")


def _state(B, page=16, max_pages=8, seed=3):
    g = torch.Generator().manual_seed(seed)
    pos = torch.randint(0, page * max_pages - 40, (B,), generator=g).to(torch.int32)
    return dict(out=torch.full((B, 48), -1, **I32), sp=torch.tensor([2, 0], **I32), cur=torch.full((B,), -1, **I32), pos=pos.cuda(),
                sl=(pos + 1).cuda(), slot=torch.full((B,), -7, **I32),
                pt=torch.randperm(B * max_pages, generator=g).to(torch.int32).view(B, max_pages).cuda())


def _params(B, temp, top_k, top_p, seed, key=None, step=0):
    """Per-row parameter tensors; scalars are broadcast."""
    t = lambda v, dt: torch.as_tensor(v, dtype=dt).expand(B).contiguous().cuda() if np.ndim(v) == 0 else torch.as_tensor(v, dtype=dt).cuda()
    return dict(temperature=t(temp, torch.float32), top_k=t(top_k, torch.int32), top_p=t(top_p, torch.float32), seed=t(seed, torch.int64),
                draw_key=t(np.arange(B) if key is None else key, torch.int32), draw_step=t(step, torch.int32))


def _rows_launch(c, logits, B, p, s, page=16):
    c.sample_advance_rows(logits, B, p["temperature"], p["top_k"], p["top_p"], p["seed"], p["draw_key"], p["draw_step"], s["out"], s["sp"],
                          s["cur"], s["pos"], s["sl"], s["slot"], s["pt"], page)


def _scalar_launch(c, logits, B, temp, top_k, top_p, seed, s, page=16):
    c.sample_advance(logits, B, temp, top_k, top_p, seed, s["out"], s["sp"], s["cur"], s["pos"], s["sl"], s["slot"], s["pt"], page)


def _uniform_pair(c, logits, temp, top_k, top_p, steps=6, seed=SEED):
    """K1: ``steps`` launches of each kernel over every row; the rows kernel's draw_step is set to step_ptr[0] before each launch."""
    B = logits.shape[0]
    a, b = _state(B), _state(B)
    for _ in range(steps):
        _scalar_launch(c, logits, B, temp, top_k, top_p, seed, a)
        p = _params(B, temp, top_k, top_p, seed)
        p["draw_step"].copy_(b["sp"][0].expand(B))
        _rows_launch(c, logits, B, p, b)
        torch.cuda.synchronize()
        assert (p["draw_step"].cpu() == b["sp"][0].cpu()).all()             # advanced by exactly one, like the step pointer
    for k in ("out", "sp", "cur", "pos", "sl", "slot"):
        assert torch.equal(a[k].cpu(), b[k].cpu()), k
    return a["out"].cpu()


# ---------------------------------------------------------------------------------------------------------------------------------
# K1: uniform parameters are cts_sample_advance, bit for bit
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("temp", [1.0, 0.2])
@pytest.mark.parametrize("pos", ["start", "middle", "end"])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_uniform_rows_equal_scalar_kernel_far_tail(dt, pos, temp):
    c = ctx()
    row, _ = _stress_row(DTYPES[dt], pos, 15.0, temp)
    B = 64 if _on_device() else 4
    _uniform_pair(c, row[None].repeat(B, 1).cuda(), temp, 0, 1.0)


def _edge_rows(V, dt):
    """Rows of the edge cases: top-k ties, a tied maximum, fp16 near 65504, subnormals, degenerate rows."""
    g = torch.Generator().manual_seed(V)
    rows = torch.randn(8, V, generator=g) * 2
    rows[0] = rows[0].clamp(max=2.0)
    rows[0, [10, 20]] = 3.5
    rows[0, [3, 400 % V, 401 % V, V - 1, 77]] = 3.0
    rows[1, [V // 7, V // 2, V - 1]] = rows[1].max() + 1.0
    rows[2] = torch.rand(V, generator=g) * 8 + (65504.0 - 16.0 if dt == torch.float16 else 30.0)
    rows[3] = torch.rand(V, generator=g) * (1e-6 if dt == torch.float16 else 1e-38)
    rows[4] = float("-inf")
    rows[5] = float("nan")
    rows[6, torch.rand(V, generator=g) < 0.5] = float("nan")
    rows[7] = float("-inf")
    rows[7, V - 2] = -3.0
    return rows.to(dt)


@pytest.mark.parametrize("temp,top_k,top_p", [(1.0, 4, 1.0), (0.7, 1, 1.0), (1.0, 1 << 20, 1.0), (1.0, 0, 1e-4), (1.0, 0, 0.999999),
                                              (0.05, 0, 1.0), (3.0, 40, 0.8), (1e-5, 30, 1.0)])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_uniform_rows_equal_scalar_kernel_edges(dt, temp, top_k, top_p):
    c = ctx()
    _uniform_pair(c, _edge_rows(1000, DTYPES[dt]).cuda(), temp, top_k, top_p)


@pytest.mark.parametrize("V", [1000, 1003, 8192, 8193, 151936, 152064])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_uniform_rows_equal_scalar_kernel_vocab_sizes(V, dt):
    c = ctx()
    row = _row("randn", V, torch.float32, V + 1).mul(2)
    row[V - 1] = row.max() + 0.5
    logits = row.to(DTYPES[dt])[None].repeat(8, 1).cuda()
    for temp, top_k, top_p in ((0.7, 0, 0.9), (1.0, 40, 1.0)):
        _uniform_pair(c, logits, temp, top_k, top_p, steps=3)


# ---------------------------------------------------------------------------------------------------------------------------------
# K2: mixed rows in one launch
# ---------------------------------------------------------------------------------------------------------------------------------
GREEDY_TEMPS = [0.0, -1.0, float("nan"), 0.0, 0.0, 0.0]
SAMPLED = [(0.2, 0, 1.0), (1.0, 1, 1.0), (1.7, 50, 0.9), (1.0, 0, 0.5), (0.2, 50, 0.5), (1.7, 1 << 20, 1.0), (1.0, 0, 0.9),
           (1.7, 0, 1.0)]


def _mixed(V, dt):
    """Greedy rows (plain, a tie, all -inf, all NaN, NaN mixed in, -0 / +0 tie) then sampled rows (uniform logits in [0, 1)) with
    parameters and draws of their own; where every kept token holds >= 2^-12 of the kept mass the draw is compared draw for draw."""
    g = torch.Generator().manual_seed(V + 5)
    nG = len(GREEDY_TEMPS)
    x = torch.randn(nG, V, generator=g) * 2
    x[1, [V // 5, V // 3]] = x[1].max() + 1.0
    x[2] = float("-inf")
    x[3] = float("nan")
    x[4, torch.rand(V, generator=g) < 0.3] = float("nan")
    x[5] = float("-inf")
    x[5, [7, 9]] = torch.tensor([-0.0, 0.0])
    s = torch.rand(len(SAMPLED), V, generator=g)
    logits = torch.cat([x, s]).to(dt)
    temps = GREEDY_TEMPS + [t for t, _, _ in SAMPLED]
    ks = [0] * nG + [k for _, k, _ in SAMPLED]
    ps = [1.0] * nG + [p for _, _, p in SAMPLED]
    B = logits.shape[0]
    seeds = [SEED + 1000 * b for b in range(B)]
    keys = [(7 * b + 3) % 11 for b in range(B)]
    steps = [b * 13 for b in range(B)]
    return logits, _params(B, temps, ks, ps, seeds, keys, steps), temps, ks, ps, seeds, keys, steps


@pytest.mark.parametrize("V", [1000, 8193, 152064])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_mixed_rows_in_one_launch(V, dt):
    c = ctx()
    logits, p, temps, ks, ps, seeds, keys, steps = _mixed(V, DTYPES[dt])
    B, nG = logits.shape[0], len(GREEDY_TEMPS)
    lg = logits.cuda()
    greedy = _greedy(c, lg)
    n_launch = 16 if _on_device() else 3
    s = _state(B)
    bad = []
    for j in range(n_launch):
        _rows_launch(c, lg, B, p, s)
        torch.cuda.synchronize()
        assert p["draw_step"].cpu().tolist() == [st + j + 1 for st in steps]
        toks = s["cur"].cpu().numpy()
        assert toks[:nG].tolist() == greedy[:nG].tolist(), (toks[:nG], greedy[:nG])
        for b in range(nG, B):
            tok, cdf, target, kept = TorchDouble.sample_reference(logits[b], temps[b], ks[b], ps[b], seeds[b], steps[b] + j, keys[b])
            if tok == toks[b]:
                continue
            if (_mass(cdf)[kept] / cdf[-1]).min() < 2 ** -12:              # no draw-for-draw precondition: the kept set only
                if not _mass(cdf)[toks[b]] > 0:
                    bad.append((j, b, int(toks[b]), tok))
                continue
            order = np.cumsum(kept) - 1
            edge = cdf[min(tok, toks[b])]
            if not (kept[toks[b]] and abs(int(order[tok]) - int(order[toks[b]])) == 1
                    and abs(target - edge) <= 64 * float(np.spacing(np.float32(cdf[-1])))):
                bad.append((j, b, int(toks[b]), tok))
    assert greedy[:nG].tolist()[2:4] == [0, 0] and greedy[5] == 7
    assert s["sp"].cpu().tolist() == [2 + n_launch, 0]
    assert not bad, bad[:5]


# ---------------------------------------------------------------------------------------------------------------------------------
# K3: distribution per row group
# ---------------------------------------------------------------------------------------------------------------------------------
K3_GROUPS = [("randn3", 1.0, 0, 1.0), ("tail", 1.0, 0, 1.0), ("randn", 0.2, 0, 0.9), ("randn", 0.2, 50, 1.0), ("peaked", 1.7, 0, 0.95),
             ("tail", 0.7, 0, 0.9), ("randn3", 1.3, 2000, 1.0), ("greedy", 0.0, 0, 1.0)]


def _k3_row(kind, dt, seed):
    if kind == "tail":
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(V_FULL, generator=g)
        x[torch.rand(V_FULL, generator=g) < 0.5] = float("-inf")
        return x.to(dt)
    return _row("randn" if kind == "greedy" else kind, V_FULL, dt, seed)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_chi_square_per_row_group(dt):
    c = ctx()
    R, S = (16, 64) if _on_device() else (2, 4)             # rows per group, launches
    rows, temps, ks, ps, seeds = [], [], [], [], []
    for gi, (kind, t, k, p) in enumerate(K3_GROUPS):
        row = _k3_row(kind, DTYPES[dt], 40 + gi)
        rows += [row] * R
        temps += [t] * R; ks += [k] * R; ps += [p] * R; seeds += [SEED + gi] * R
    B = len(rows)
    keys = list(range(B))
    logits = torch.stack(rows).cuda()
    prm = _params(B, temps, ks, ps, seeds, keys, 0)
    st = _state(B)
    toks = np.zeros((B, S), dtype=np.int64)
    for j in range(S):
        _rows_launch(c, logits, B, prm, st)
        toks[:, j] = st["cur"].cpu().numpy()
    assert prm["draw_step"].cpu().tolist() == [S] * B
    for gi, (kind, t, k, p) in enumerate(K3_GROUPS):
        row = rows[gi * R]
        got = toks[gi * R:(gi + 1) * R].reshape(-1)
        if kind == "greedy":
            assert (got == _greedy(c, row[None].cuda())[0]).all()
            continue
        _, cdf, _, kept = TorchDouble.sample_reference(row, t, k, p, seeds[gi * R], 0, 0)
        prob, x = _mass(cdf), row.float().numpy().astype(np.float64)
        assert (prob[got] > 0).all(), f"group {gi}: a token of zero mass"
        if not _on_device():
            continue
        bin_of, frac = _bins_by_logit(x, prob, 16, len(got))
        chi, dof = _chi2(got, bin_of, frac)
        b_idx = np.arange(gi * R, (gi + 1) * R)
        u = _uniforms(seeds[gi * R], np.tile(np.arange(S), R), np.repeat(b_idx, S))
        chi_ref, _ = _chi2(_statement_tokens(cdf, kept, u), bin_of, frac)
        record("sample_rows_chi2", dtype=dt, kind=kind, temp=t, top_k=k, top_p=p, chi2=chi, dof=dof, statement_chi2=chi_ref)
        assert dof >= 5 and chi_ref < _chi2_limit(dof) and chi < _chi2_limit(dof), (gi, chi, chi_ref, dof)


# ---------------------------------------------------------------------------------------------------------------------------------
# K4: refusals chained into the rows kernel
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chain", ["struct", "allowed_ids", "min_tokens"])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_refused_ids_are_never_sampled(chain, dt):
    c = ctx()
    B = 16 if _on_device() else 3
    row, dom = _stress_row(DTYPES[dt], "start", 15.0, 1.0, seed=23)
    x = row.float().numpy()
    rng = np.random.default_rng(7)
    finite = np.nonzero(np.isfinite(x))[0]
    lg = row[None].repeat(B, 1).cuda()
    vw = (V_FULL + 31) // 32
    if chain == "min_tokens":
        stops = torch.from_numpy(rng.choice(finite[finite != dom], 64, replace=False).astype(np.int32))
        refused = np.zeros(V_FULL, dtype=bool)
        refused[stops.numpy()] = True
        args = [torch.ones(B), torch.zeros(B), torch.zeros(B), torch.zeros(B, vw, dtype=torch.int32), None, None,
                torch.full((B,), -1, dtype=torch.int32), torch.zeros(B, dtype=torch.int32), torch.full((B,), 5, dtype=torch.int32),
                stops[None].repeat(B, 1).contiguous()]
    else:
        allowed = np.zeros(V_FULL, dtype=bool)
        allowed[rng.choice(finite, V_FULL // 3, replace=False)] = True
        refused = ~allowed
        if chain == "allowed_ids":
            bias = torch.zeros(1, V_FULL)
            bias[0, torch.from_numpy(refused)] = float("-inf")
            args = [torch.ones(B), torch.zeros(B), torch.zeros(B), torch.zeros(B, vw, dtype=torch.int32), None, bias,
                    torch.zeros(B, dtype=torch.int32), torch.zeros(B, dtype=torch.int32), torch.zeros(B, dtype=torch.int32), None]
    if chain == "struct":
        c.struct_mask_apply(lg, B, torch.zeros(B, **I32), torch.from_numpy(pack_bits(allowed[None])).cuda())
    else:
        c.logit_proc_apply(lg, B, *[a.cuda() if a is not None else None for a in args])
    temps = [1.0, 0.7, 1.7, 0.0] * (B // 4) + [1.0] * (B % 4)
    prm = _params(B, temps, [0, 0, 50, 0] * (B // 4) + [0] * (B % 4), 1.0, [SEED + b for b in range(B)])
    st = _state(B)
    n = 64 if _on_device() else 4
    got = []
    for _ in range(n):
        _rows_launch(c, lg, B, prm, st)
        got.append(st["cur"].cpu().numpy())
    got = np.stack(got)
    assert not refused[got].any(), f"{int(refused[got].sum())} refused ids of {got.size}"
    assert np.isfinite(x[got]).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# K5: CUDA graphs
# ---------------------------------------------------------------------------------------------------------------------------------
def test_graph_replay_is_bit_identical():
    c = ctx()
    B, S = 32, 200
    g = torch.Generator().manual_seed(9)
    logits = (torch.randn(B, V_FULL, generator=g) * 2).to(torch.bfloat16).cuda()
    temps = [0.0, 0.2, 1.0, 1.7] * (B // 4)
    mk = lambda: _params(B, temps, [0, 50, 0, 1 << 20] * (B // 4), [1.0, 0.9, 0.5, 1.0] * (B // 4), [11 * b for b in range(B)],
                         [b ^ 5 for b in range(B)], [3 * b for b in range(B)])
    big = lambda: dict(_state(B), out=torch.full((B, S + 8), -1, **I32))
    eager, graphed = (mk(), big()), (mk(), big())
    for _ in range(S):
        _rows_launch(c, logits, B, *eager)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _rows_launch(c, logits, B, *graphed)
    torch.cuda.synchronize()
    assert (graphed[1]["out"] == -1).all()                                    # capture launches nothing
    for _ in range(S):
        graph.replay()
    torch.cuda.synchronize()
    for k in ("out", "sp", "cur", "pos", "sl", "slot"):
        assert torch.equal(graphed[1][k].cpu(), eager[1][k].cpu()), k
    assert torch.equal(graphed[0]["draw_step"].cpu(), eager[0]["draw_step"].cpu())
    assert graphed[0]["draw_step"].cpu().tolist() == [3 * b + S for b in range(B)]


# ---------------------------------------------------------------------------------------------------------------------------------
# E1: the continuous engine
# ---------------------------------------------------------------------------------------------------------------------------------
def _engine_model():
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig.tiny()
    sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=torch.bfloat16, std=0.05)
    model = ChatTSForCausalLM(cfg, sd, dtype=torch.bfloat16, max_batch=4, max_seq_len=256, page_size=16, use_cuda_graph=True)
    return model, ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)


def test_engine_requests_match_solo_runs_in_any_order():
    from chatts_b200.engine import ContinuousEngine
    model, proc = _engine_model()
    x = np.arange(200)
    specs = [("A <ts><ts/> ?", [np.sin(x / 9) * 4], 9, {}),
             ("plain text", [], 8, dict(temperature=0.8, top_p=0.9, seed=5)),
             ("B <ts><ts/>", [np.cos(x / 5)[:77]], 11, dict(temperature=1.7, top_k=50, seed=17)),
             ("processors", [], 7, dict(temperature=1.0, seed=3, presence_penalty=0.8, logit_bias={5: 2.0})),
             ("with logprobs", [], 6, dict(temperature=0.2, top_k=1 << 20, seed=9, logprobs=3)),
             ("greedy too", [], 5, dict(logprobs=2))]
    encs = [(proc(text=[t], timeseries=s, return_tensors="pt"), n, kw) for t, s, n, kw in specs]

    def run(order, width=4):
        eng = ContinuousEngine(model, slots=width, steps_per_round=3, max_prefill_batch=1)
        rid = {}
        for i in order:
            enc, n, kw = encs[i]
            rid[eng.add_request(enc["input_ids"][0], enc["timeseries"], max_new_tokens=n, ignore_eos=True, **kw)] = i
        done = eng.run()
        eng.close()
        return {rid[r.rid]: (r.tokens, r.token_logprobs) for r in done}

    solo = {}
    for i in range(len(encs)):
        solo.update(run([i]))
    pages0 = len(model.pool.free)
    crowded = run(range(len(encs)))
    assert crowded == solo
    assert run([5, 3, 1, 0, 4, 2]) == solo
    assert len(model.pool.free) == pages0
    # greedy requests: the same tokens when nobody samples
    quiet = run([0, 5])
    assert quiet[0] == solo[0] and quiet[5] == solo[5]
    # a sampled request's first token: batch-1 generate(seed=...) with the same parameters
    for i in (1, 2, 4):
        enc, n, kw = encs[i]
        S = enc["input_ids"].shape[1]
        g = model.generate(**enc, max_new_tokens=1, ignore_eos=True, do_sample=True, temperature=kw["temperature"],
                           top_k=kw.get("top_k"), top_p=kw.get("top_p"), seed=kw["seed"])
        assert g[0, S].item() == solo[i][0][0], i
    assert len(model.pool.free) == pages0
