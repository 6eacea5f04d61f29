"""Prefix caching (chatts_b200/prefix_cache.py, ChatTSForCausalLM(enable_prefix_caching=True)) on the GPU: a cold call is the uncached
call bit for bit; a warm call that shares series and differs in its question hits the expected pages, and its prefill logits, decode
logits and every KV row it reads or wrote pass the oracle gate (the oracle runs the WHOLE prompt, teacher-forced on the produced
tokens); the same token ids with other series share nothing; eviction, invalidation by merge_lora, and ContinuousEngine admissions
that share a prefix."""
import numpy as np
import pytest
import torch

from oracle import decoder as od
from oracle import merge as om
from oracle import ts_encoder as ote
from tests.gpu_util import DecodeRun, parity_gate, record, rel_err

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
DTS = [pytest.param(BF, id="bf16"), pytest.param(FP, id="fp16")]
STEPS = 4
_LETTERS = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz ,.?", dtype=np.uint8)


def _cfg(kind):
    from chatts_b200 import ChatTSConfig
    if kind == "small128":                                   # ChatTS-14B proportions at a small width: head_dim 128, GQA group 5
        cfg = ChatTSConfig.tiny(hidden_size=1280, intermediate_size=3456, num_attention_heads=10, num_key_value_heads=2, head_dim=128,
                                vocab_size=2000, ts_token_start_index=1990, eos_token_id=1998, pad_token_id=1999)
        cfg.ts = dict(cfg.ts, hidden_size=1280)
        return cfg
    if kind == "l14b":                                       # one decoder layer at the ChatTS-14B shapes, small vocabulary, no encoder
        return ChatTSConfig(num_hidden_layers=1, vocab_size=512, ts_token_start_index=500, eos_token_id=510, pad_token_id=511,
                            max_position_embeddings=1024)
    cfg = ChatTSConfig.tiny()
    if kind == "tiny_q3":
        cfg.qk_norm, cfg.attention_bias = True, False
    return cfg


_SD = {}


def _weights(kind, dt):
    from chatts_b200.weights import synthetic_state_dict
    if (kind, dt) not in _SD:
        _SD.clear()
        cfg = _cfg(kind)
        sd = synthetic_state_dict(cfg, seed=4243, device="cpu", dtype=dt, std=0.02 if kind == "l14b" else 0.05)
        if kind == "l14b":
            sd = {k: v for k, v in sd.items() if not k.startswith("ts_encoder.")}
        _SD[(kind, dt)] = (cfg, sd)
    return _SD[(kind, dt)]


def _model(kind, dt, cached, page=16, max_batch=4, max_seq_len=512, sd=None):
    from chatts_b200.model import ChatTSForCausalLM
    cfg, sd0 = _weights(kind, dt)
    return ChatTSForCausalLM(cfg, sd if sd is not None else sd0, dtype=dt, max_batch=max_batch, max_seq_len=max_seq_len, page_size=page,
                             enable_prefix_caching=cached)


def _proc(cfg):
    from chatts_b200 import ChatTSProcessor, SimpleTokenizer
    return ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)


def _series(seed, n=160):
    rng = np.random.default_rng(seed)
    return np.sin(np.arange(n) / (3.0 + seed % 5)) * (1 + seed % 3) + rng.normal(size=n) * 0.1


def _text(seed, n):
    return _LETTERS[np.random.default_rng(seed).integers(0, 30, n)].tobytes().decode()


def _row(kind, question, series_seed=1, lead=5):
    """(text, [series]) of one prompt: ``lead`` letters, two series, then the question (text only for the model without encoder)."""
    if kind == "l14b":
        return _text(77, 150) + " " + _text(question, 20), []
    return (_text(77, lead) + " <ts><ts/> and <ts><ts/> q: " + _text(question, 20),
            [_series(series_seed), _series(series_seed + 10, 96)])


def _encode(proc, rows):
    series = [s for _, ss in rows for s in ss]
    return proc(text=[t for t, _ in rows], timeseries=series or None, padding=True, return_tensors="pt")


def _drive(model, enc, steps):
    """generate()'s path (prefix-cache allocation, prefill, registration, graph-replayed greedy decode) keeping every step's logits."""
    ts = enc.get("timeseries")
    _, _, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], ts)
    B = lay.cu_seqlens.shape[0] - 1
    pts, held, keys, cached = model._alloc_prompt(lay, ts, steps + 1)
    try:
        pre = model._prefill(lay, counts, ts, pts, cached=cached)
        model._prefix_register(keys, pts, lay.lens, cached)
        st = model._decode_state(B, steps + 1)
        lens32 = torch.from_numpy(lay.lens.astype(np.int32))
        st.page_table.copy_(torch.from_numpy(pts)); st.positions.copy_(lens32 - 1); st.seq_lens.copy_(lens32); st.step_ptr.zero_()
        model.ctx.greedy_advance(pre, B, st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.page_table,
                                 model.page_size)
        prefill = pre[:B].float().cpu().clone()
        logits = []
        for _ in range(steps):
            model._decode_step(st, sample=True)
            logits.append(st.full_logits[:B].float().cpu().clone())
        torch.cuda.synchronize()
        return DecodeRun(prefill=prefill, logits=torch.stack(logits), tokens=st.out_tokens[:, :steps + 1].cpu().clone(), lens=lay.lens.copy(),
                         page_table=st.page_table.cpu().clone(), seq_lens=st.seq_lens.cpu().clone(),
                         cached=None if cached is None else cached.copy(), lay=lay)
    finally:
        model.pool.release(held)


def _oracle(cfg, w, dt, fp32, proc, row, tokens, mode="insert"):
    """Oracle on the whole prompt of ``row``, then teacher-forced on ``tokens``: (prefill logits, per-step logits, State)."""
    text, series = row
    enc = proc(text=[text], timeseries=series or None, return_tensors="pt")
    feats, pc = None, []
    if series:
        ts_w = {k[len("ts_encoder."):]: v for k, v in w.items() if k.startswith("ts_encoder.")}
        x = enc["timeseries"].to(dt)
        feats, pc = ote.forward(x.float() if fp32 else x, cfg.ts, ts_w)
        pc = pc.tolist()
    emb = om.hf_merge(enc["input_ids"], enc["attention_mask"], w["model.embed_tokens.weight"], feats, pc, cfg.ts_token_start_index, mode)[0]
    st = od.State(cfg.num_hidden_layers)
    pre = od.logits(od.forward_hidden(emb, w, cfg.to_dict(), st)[-1:], w)[0]
    lg = [od.logits(od.forward_hidden(w["model.embed_tokens.weight"][t][None], w, cfg.to_dict(), st), w)[0] for t in tokens]
    return pre, lg, st


def _common_pages(lay_a, lay_b, ts_same, page):
    """Full pages the warm prompt (b) shares with the cold one (a): merged positions equal in id and in series content, capped so that
    the warm prompt's last position is recomputed."""
    a, b = lay_a.ids, lay_b.ids
    n = 0
    while n < min(a.shape[0], b.shape[0]) and a[n] == b[n] and (a[n] >= 0 or ts_same):
        n += 1
    return min(n // page, (b.shape[0] - 1) // page)


# Fixed bounds against the same-dtype oracle (logits: prefill and decode steps; kv: every cache row of the warm sequence, the shared
# pages included), the decode-parity bounds of the same configurations.  Measured warm calls on an H100 80GB HBM3 (700 W), max over
# cases (tiny: also the hit boundary inside a series):
#   tiny      bf16 logits 1.24e-2 kv 9.3e-3    fp16 logits 1.40e-3 kv 1.24e-3
#   tiny_q3   bf16 logits 1.40e-2 kv 1.30e-2   fp16 logits 1.61e-3 kv 1.62e-3
#   small128  bf16 logits 2.79e-2 kv 2.05e-2   fp16 logits 3.71e-3 kv 2.50e-3
#   l14b      bf16 logits 1.16e-2 kv 2.5e-3    fp16 logits 1.89e-3 kv 5.5e-4
BOUND = {("tiny", BF): dict(logits=2.2e-2, kv=1.7e-2), ("tiny", FP): dict(logits=2.7e-3, kv=2.4e-3),
         ("tiny_q3", BF): dict(logits=2.2e-2, kv=1.7e-2), ("tiny_q3", FP): dict(logits=2.7e-3, kv=2.4e-3),
         ("small128", BF): dict(logits=4e-2, kv=2.3e-2), ("small128", FP): dict(logits=6.2e-3, kv=3.1e-3),
         ("l14b", BF): dict(logits=2.1e-2, kv=4e-3), ("l14b", FP): dict(logits=2.3e-3, kv=1e-3)}
KV_RATIO = 1.5          # element-wise KV rows: the comparative factor of the decode-parity gate (tests/test_gpu_zz_g_decode_parity.py)


def _gate_warm(name, kind, dt, model, proc, row, run, mode="insert"):
    cfg, sd = _weights(kind, dt)
    toks = run.tokens[0].tolist()
    outs = [_oracle(cfg, w, dt, f32, proc, row, toks[:STEPS], mode)
            for w, f32 in ((sd, False), ({k: v.float() for k, v in sd.items()}, True))]
    b = BOUND[(kind, dt)]
    got = [run.prefill[0]] + [run.logits[i, 0] for i in range(STEPS)]
    parity_gate(f"{name}-logits", got, [outs[0][0]] + outs[0][1], [outs[1][0]] + outs[1][1], dt, b["logits"])
    for i in range(STEPS):                                   # each token is the argmax of the logits the model computed
        assert toks[i + 1] == int(run.logits[i, 0].argmax())
    pos = torch.arange(int(run.seq_lens[0]) - 1)
    pg = run.page_table[0].long()[pos // model.page_size]
    kv = model.kv.cpu()
    for l in range(cfg.num_hidden_layers):
        got = [kv[l, 0, pg, :, pos % model.page_size], kv[l, 1, pg, :, pos % model.page_size]]
        parity_gate(f"{name}-kv-l{l}", got, [outs[0][2].k[l], outs[0][2].v[l]], [outs[1][2].k[l], outs[1][2].v[l]], dt, b["kv"],
                    ratio=KV_RATIO)


KINDS = ["tiny", "small128", "l14b"]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("kind", KINDS)
def test_cold_call_is_the_uncached_call_bit_for_bit(kind, dt):
    cfg, _ = _weights(kind, dt)
    proc = _proc(cfg)
    enc = _encode(proc, [_row(kind, 1), _row(kind, 2, series_seed=3), _row(kind, 4)])
    runs = []
    for cached in (False, True):
        m = _model(kind, dt, cached)
        runs.append((_drive(m, enc, STEPS), m.generate(**enc, max_new_tokens=6, ignore_eos=True)))
        del m
    (a, ga), (b, gb) = runs
    assert b.cached is not None and int(b.cached.sum()) == 0      # within one batch nothing is shared (registration follows the prefill)
    assert torch.equal(a.prefill, b.prefill) and torch.equal(a.logits, b.logits) and torch.equal(a.tokens, b.tokens)
    assert torch.equal(ga, gb)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("kind,page,mode", [("tiny", 16, "insert"), ("tiny", 32, "overwrite"), ("tiny_q3", 64, "insert"),
                                             ("small128", 16, "insert"), ("small128", 64, "overwrite"), ("l14b", 16, "insert")])
def test_warm_call_hits_and_matches_the_oracle(kind, page, mode, dt, monkeypatch):
    """Same series, another question: the hit count is the shared full pages (capped), and the warm call's prefill logits, decode
    logits and KV rows pass the oracle gate, the oracle running the whole prompt."""
    monkeypatch.setenv("CTS_TS_MERGE_MODE", mode)
    cfg, _ = _weights(kind, dt)
    proc = _proc(cfg)
    m = _model(kind, dt, True, page=page)
    cold_row, warm_row = _row(kind, 1, lead=37), _row(kind, 2, lead=37)
    cold = _drive(m, _encode(proc, [cold_row]), STEPS)
    warm = _drive(m, _encode(proc, [warm_row]), STEPS)
    want = _common_pages(cold.lay, warm.lay, True, page)
    assert want >= 1 and int(warm.cached[0]) == want * page, (int(warm.cached[0]), want)
    st = m.prefix_cache_stats()
    assert st["hit_positions"] == want * page and st["queried_positions"] == int(cold.lens.sum() + warm.lens.sum())
    record("prefix_cache_warm", kind=kind, page=page, mode=mode, dtype=str(dt), hit=want * page, prompt=int(warm.lens[0]))
    _gate_warm(f"prefix-warm-{kind}-p{page}-{mode}", kind, dt, m, proc, warm_row, warm, mode)


@pytest.mark.parametrize("dt", DTS)
def test_hit_boundary_inside_a_series(dt):
    """The cached prefix ends inside the first series' patch rows: that series is encoded whole, its cached rows discarded."""
    kind, page = "tiny", 16
    cfg, _ = _weights(kind, dt)
    proc = _proc(cfg)
    m = _model(kind, dt, True, page=page)
    cold_row, warm_row = _row(kind, 1, lead=5), _row(kind, 2, lead=5)
    _drive(m, _encode(proc, [cold_row]), STEPS)
    warm = _drive(m, _encode(proc, [warm_row]), STEPS)
    rows, hit = warm.lay.row_map, int(warm.cached[0])
    spans = [rows[:10], rows[10:]]                          # 160 points / patch 16, then 96 points
    assert any(r.min() < hit <= r.max() for r in spans), (hit, [(int(r.min()), int(r.max())) for r in spans])
    _gate_warm("prefix-boundary-in-series", kind, dt, m, proc, warm_row, warm)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("kind", ["tiny", "small128"])
def test_same_ids_other_series_share_nothing(kind, dt):
    """The same input ids with other series (of the same lengths): exactly the full pages in front of the first patch row are shared,
    nothing from the page that holds it on, and the output is the uncached model's within the logits bound."""
    cfg, _ = _weights(kind, dt)
    proc = _proc(cfg)
    m, ref = _model(kind, dt, True, page=64), _model(kind, dt, False, page=64)
    enc1 = _encode(proc, [_row(kind, 1, series_seed=1, lead=1)])
    enc2 = dict(enc1, timeseries=_encode(proc, [_row(kind, 1, series_seed=2, lead=1)])["timeseries"])
    assert not torch.equal(enc1["timeseries"], enc2["timeseries"])
    _drive(m, enc1, STEPS)
    b = _drive(m, enc2, STEPS)
    first_row = int(np.nonzero(b.lay.ids < 0)[0][0])
    assert int(b.cached[0]) == first_row // m.page_size * m.page_size
    a = _drive(ref, enc2, STEPS)
    e = rel_err(b.prefill, a.prefill)
    record("prefix_cache_other_series_vs_uncached", kind=kind, dtype=str(dt), err=e, hit=int(b.cached[0]))
    assert e < BOUND[(kind, dt)]["logits"]
    assert torch.equal(a.tokens[:, :1], b.tokens[:, :1])


def test_fp8_model_warm_call():
    """FP8 weights (prefill on the dequantised projections): the warm call against the uncached FP8 model's full prefill."""
    dt, kind = BF, "tiny"
    cfg, _ = _weights(kind, dt)
    proc = _proc(cfg)
    m, ref = _model(kind, dt, True).quantize_fp8(), _model(kind, dt, False).quantize_fp8()
    _drive(m, _encode(proc, [_row(kind, 1, lead=37)]), STEPS)
    enc = _encode(proc, [_row(kind, 2, lead=37)])
    warm, full = _drive(m, enc, STEPS), _drive(ref, enc, STEPS)
    assert int(warm.cached[0]) > 0
    e = rel_err(warm.prefill, full.prefill)
    record("prefix_cache_fp8_warm_vs_full", err=e)
    assert e < BOUND[(kind, dt)]["logits"]


@pytest.mark.parametrize("dt", DTS)
def test_eviction_keeps_results_and_stats_consistent(dt):
    """A pool of 6 pages: the second prompt evicts the first one's cached pages; a third call of the first prompt recomputes what
    was evicted and still matches the uncached model bit for bit where nothing was hit."""
    kind, page = "tiny", 16
    cfg, _ = _weights(kind, dt)
    proc = _proc(cfg)
    m = _model(kind, dt, True, page=page, max_batch=1, max_seq_len=320)
    ref = _model(kind, dt, False, page=page, max_batch=1, max_seq_len=320)
    rows = [_row(kind, 1, series_seed=1), _row(kind, 1, series_seed=21), _row(kind, 1, series_seed=41)]
    for r in rows + rows[:1]:
        enc = _encode(proc, [r])
        b, a = _drive(m, enc, STEPS), _drive(ref, enc, STEPS)
        st = m.prefix_cache_stats()
        assert m.pool.available() == m.pool.num_pages                           # nothing held between calls
        assert st["cached_pages"] == len(m.pool.evictable) <= m.pool.num_pages
        if int(b.cached[0]) == 0:
            assert torch.equal(a.prefill, b.prefill) and torch.equal(a.tokens, b.tokens)
        else:
            assert rel_err(b.prefill, a.prefill) < BOUND[(kind, dt)]["logits"]
    assert st["evictions"] > 0
    assert st["queried_positions"] >= st["hit_positions"] >= 0


def test_merge_lora_invalidates():
    dt, kind = BF, "tiny"
    cfg, sd = _weights(kind, dt)
    proc = _proc(cfg)
    g = torch.Generator().manual_seed(5)
    H, r = cfg.hidden_size, 4
    nq = cfg.num_attention_heads * cfg.head_dim
    ad = {"base_model.model.model.layers.0.self_attn.q_proj.lora_A.weight": torch.randn(r, H, generator=g) * 0.05,
          "base_model.model.model.layers.0.self_attn.q_proj.lora_B.weight": torch.randn(nq, r, generator=g) * 0.05}
    m, ref = _model(kind, dt, True), _model(kind, dt, False)
    enc = _encode(proc, [_row(kind, 1, lead=37)])
    _drive(m, enc, STEPS)
    m.merge_lora(ad, lora_alpha=8, r=r)
    ref.merge_lora(ad, lora_alpha=8, r=r)
    b = _drive(m, enc, STEPS)
    assert int(b.cached[0]) == 0 and m.prefix_cache_stats()["cached_pages"] == (int(b.lens[0]) // m.page_size)
    a = _drive(ref, enc, STEPS)
    assert torch.equal(a.prefill, b.prefill) and torch.equal(a.logits, b.logits) and torch.equal(a.tokens, b.tokens)


@pytest.mark.parametrize("dt", DTS)
def test_continuous_engine_shared_prefix(dt):
    """Requests that share a prefix, admitted in overlapping groups while earlier ones decode: every produced token is the oracle's
    argmax or within the logits bound of it (the oracle teacher-forced on the request's whole prompt and tokens), some admissions hit,
    and the pool is whole again once the engine closes."""
    from chatts_b200.engine import ContinuousEngine
    kind, page = "tiny", 16
    cfg, sd = _weights(kind, dt)
    proc = _proc(cfg)
    m = _model(kind, dt, True, page=page, max_batch=4)
    eng = ContinuousEngine(m, slots=4, steps_per_round=2, max_prefill_batch=2)
    rows = [_row(kind, q, lead=37) for q in range(6)]
    reqs = []
    for i, row in enumerate(rows):
        enc = proc(text=[row[0]], timeseries=row[1], return_tensors="pt")
        reqs.append(eng.add_request(enc["input_ids"][0], enc["timeseries"], max_new_tokens=5 + i % 3, ignore_eos=True))
        if i % 2:
            eng.step()
    eng.run()
    done = {r.rid: r for r in eng.finished}
    eng.close()
    assert m.pool.available() == m.pool.num_pages
    assert sum(done[rid].cached_positions > 0 for rid in reqs) >= 3
    w = {k: v.float() for k, v in sd.items()}
    for rid, row in zip(reqs, rows):
        r = done[rid]
        assert r.error is None
        pre, lg, _ = _oracle(cfg, w, dt, True, proc, row, r.tokens[:-1])
        for i, logits in enumerate([pre] + lg):
            gap = float(logits.max() - logits[r.tokens[i]])
            assert gap <= 2 * BOUND[(kind, dt)]["logits"] * float(logits.abs().max()), (rid, i, gap)
