"""Decode parity: every decode step's logits and every KV-cache row the run wrote, against the oracle run teacher-forced on the tokens the
model produced (in the model dtype and in fp32), on every decode path and batch width; plus the isolation of a request from cache rows it
does not own.

The paths (chatts_b200/model.py): the multi-kernel step (streaming GEMM at t <= 32; split-1 QKV with bias, EPI_RESIDUAL o/down and
gemm_tn gate_up at 32 < t <= 128; the persistent EPI_SWIGLU_IL GEMM at t > 128), with and without CUDA graph replay and with the
next-GEMM L2 hint (CTS_NEXT_PREFETCH_MB, gemm_tn_kernel); the native C++ step; the decode chain; the cluster-fused decode at levels 1
and 2; FP8 weights (oracle on W' = fp32(code) * scale); W4A16 through both kernels (oracle on the dequantised weights).  The prompts are
left-padded and ragged, some rows carry a time series, and rows 0-3 are p-1, p, p+1 and 2p-3 positions long for page size p, so their
KV writes cross a page boundary at different steps."""
import numpy as np
import pytest
import torch

from oracle import decoder as od
from oracle import merge as om
from oracle import ts_encoder as ote
from tests.gpu_util import decode_run, parity_gate, record

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
STEPS = 6
_LETTERS = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz ,.?", dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------------------- models
def _cfg(kind):
    from chatts_b200 import ChatTSConfig
    if kind == "tiny_w4":                                    # the mma W4 kernel needs every K a multiple of 128
        return ChatTSConfig.tiny(intermediate_size=768)
    if kind == "small128":                                   # ChatTS-14B proportions at a small width: head_dim 128, GQA group 5
        cfg = ChatTSConfig.tiny(hidden_size=1280, intermediate_size=3456, num_attention_heads=10, num_key_value_heads=2, head_dim=128,
                                vocab_size=2000, ts_token_start_index=1990, eos_token_id=1998, pad_token_id=1999)
        cfg.ts = dict(cfg.ts, hidden_size=1280)
        return cfg
    if kind == "l14b":                                       # one decoder layer at the ChatTS-14B shapes, small vocabulary
        return ChatTSConfig(num_hidden_layers=1, vocab_size=512, ts_token_start_index=500, eos_token_id=510, pad_token_id=511,
                            max_position_embeddings=1024)
    cfg = ChatTSConfig.tiny()
    if kind == "tiny_q3":                                    # Qwen3 (ChatTS-8B family): q/k RMSNorm, no qkv bias
        cfg.qk_norm, cfg.attention_bias = True, False
    return cfg


_SD = {}


def _weights(kind, dt):
    from chatts_b200.weights import synthetic_state_dict
    if (kind, dt) not in _SD:
        for k in [k for k in _SD if k[0] != kind]:          # one configuration at a time (the 14B layer is ~1 GB per dtype)
            del _SD[k]
        cfg = _cfg(kind)
        sd = synthetic_state_dict(cfg, seed=4242, device="cpu", dtype=dt, std=0.02 if kind == "l14b" else 0.05)
        if kind == "l14b":
            sd = {k: v for k, v in sd.items() if not k.startswith("ts_encoder.")}
        _SD[(kind, dt)] = (cfg, sd, {k: v.float() for k, v in sd.items()}, {})      # the last dict caches the oracle's prefill states
    return _SD[(kind, dt)]


def _model(kind, dt, path, B, page, max_seq_len=512):
    from chatts_b200.model import ChatTSForCausalLM
    cfg, sd, sd32, cache = _weights(kind, dt)
    model = ChatTSForCausalLM(cfg, sd, dtype=dt, max_batch=B, max_seq_len=max_seq_len, page_size=page, use_cuda_graph=path != "eager",
                              use_chain=path == "chain", use_native_step=path == "native",
                              use_fused_decode=int(path[-1]) if path.startswith("fused") else 0)
    if path == "fp8":
        model.quantize_fp8()
    elif path.startswith("w4"):
        model.quantize_w4_synthetic(group_size=64)
        assert model.w4["kernel"] == path[3:]
    return cfg, (sd, sd32), cache, model


def _dense_state_dict(model, sd, dt):
    """The checkpoint with every decoder projection replaced by the model's own dense weights (after quantize_w4_synthetic: the
    dequantised values), (in the model dtype, in fp32)."""
    H, I, d, nh, nkv = model.H, model.I, model.d, model.nh, model.nkv
    same, f32 = dict(sd), {k: v.float() for k, v in sd.items()}
    for l in range(model.L):
        q_, k_, v_ = model.wqkv[l].cpu().split([nh * d, nkv * d, nkv * d])
        gu = model.wgu[l].cpu().view(-1, 2, 64, H)
        parts = {"self_attn.q_proj": q_, "self_attn.k_proj": k_, "self_attn.v_proj": v_, "self_attn.o_proj": model.wo[l].cpu(),
                 "mlp.gate_proj": gu[:, 0].reshape(I, H), "mlp.up_proj": gu[:, 1].reshape(I, H), "mlp.down_proj": model.wd[l].cpu()}
        for name, t in parts.items():
            same[f"model.layers.{l}.{name}.weight"], f32[f"model.layers.{l}.{name}.weight"] = t.to(dt).contiguous(), t.float().contiguous()
    return same, f32


# ---------------------------------------------------------------------------------------------------------------- prompts
def _rows(B, page, with_ts=True, long=False):
    """(text, series or None) per row.  Rows 0-3: text only, p-1, p, p+1 and 2p-3 positions; then every third row carries a time
    series, the others are ragged text.  A row's content depends only on its index (and, for rows 0-3, the page size), so the oracle
    prefill of a row is shared by every batch width."""
    out = []
    for b in range(B):
        rng = np.random.default_rng(1000 + b)
        if long:
            # > 600 merged positions: at max_seq_len 2048 the step has 32 attention splits, more than 8 of them live
            out.append(("long: " + _LETTERS[rng.integers(0, 30, 640)].tobytes().decode() + " <ts><ts/> ?",
                        np.cumsum(rng.normal(size=256))))
        elif b < 4 and B > 1:
            out.append((_LETTERS[rng.integers(0, 30, [page - 1, page, page + 1, 2 * page - 3][b])].tobytes().decode(), None))
        elif with_ts and (b % 3 == 1 or B == 1):
            n = 48 + 16 * (b % 5)
            out.append((f"s{b} <ts><ts/> " + _LETTERS[rng.integers(0, 30, 3 + b % 11)].tobytes().decode(),
                        np.sin(np.arange(n) / (3.0 + b % 7)) * (1 + b % 4) + rng.normal(size=n) * 0.1))
        else:
            n = 5 + (53 * b) % (40 if not with_ts else 150)
            out.append((_LETTERS[rng.integers(0, 30, n)].tobytes().decode(), None))
    return out


def _encode(proc, rows):
    return proc(text=[t for t, _ in rows], timeseries=[s for _, s in rows if s is not None], padding=True, return_tensors="pt")


def _proc(cfg):
    from chatts_b200 import ChatTSProcessor, SimpleTokenizer
    return ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)


def _oracle_prefill(cfg, w, dt, fp32, proc, row):
    """The oracle's State after the row's prompt (the merged embeddings of the row alone)."""
    text, series = row
    enc = proc(text=[text], timeseries=[series] if series is not None else None, return_tensors="pt")
    feats, pc = None, []
    if series is not None:
        ts_w = {k[len("ts_encoder."):]: v for k, v in w.items() if k.startswith("ts_encoder.")}
        x = enc["timeseries"].to(dt)
        feats, pc = ote.forward(x.float() if fp32 else x, cfg.ts, ts_w)
        pc = pc.tolist()
    emb = om.hf_merge(enc["input_ids"], enc["attention_mask"], w["model.embed_tokens.weight"], feats, pc, cfg.ts_token_start_index)[0]
    st = od.State(cfg.num_hidden_layers)
    od.forward_hidden(emb, w, cfg.to_dict(), st)
    return st


def _oracle(cfg, w, dt, fp32, proc, row, tokens, cache, key):
    """Logits of every decode step (the oracle fed the tokens the model produced) and the oracle's KV cache after them."""
    if key not in cache:
        cache[key] = _oracle_prefill(cfg, w, dt, fp32, proc, row)
    st0 = cache[key]
    st = od.State(cfg.num_hidden_layers)
    st.k, st.v, st.len = list(st0.k), list(st0.v), st0.len
    lg = [od.logits(od.forward_hidden(w["model.embed_tokens.weight"][t][None], w, cfg.to_dict(), st), w)[0] for t in tokens]
    return lg, st


def _kv_rows(kv, page, run, b, l):
    """K and V [seq_len - 1, nkv, d] of row b in layer l of the cache ``kv``, read through the final page table: every row the prefill
    and the decode steps wrote."""
    pos = torch.arange(int(run.seq_lens[b]) - 1)
    pg = run.page_table[b].long()[pos // page]
    return kv[l, 0, pg, :, pos % page], kv[l, 1, pg, :, pos % page]


def _live_slots(model, run):
    live = torch.zeros(model.kv.shape[2], model.page_size, dtype=torch.bool)
    for b in range(run.page_table.shape[0]):
        pos = torch.arange(int(run.seq_lens[b]) - 1)
        live[run.page_table[b].long()[pos // model.page_size], pos % model.page_size] = True
    return live


# ---------------------------------------------------------------------------------------------------------------- parity
def _case(kind, path, B, page, **kw):
    return dict(kind=kind, path=path, B=B, page=page, **kw)


CASES = ([_case("tiny", "default", B, p) for B, p in ((1, 16), (8, 32), (32, 64), (33, 16), (64, 32), (129, 64))]
         + [_case("tiny", "default", 1, 64, long=True, max_seq_len=2048),
            _case("tiny", "default", 8, 32, splits=1), _case("tiny", "default", 8, 16, splits=32),
            _case("tiny", "eager", 8, 16), _case("tiny", "default", 8, 64, prefetch=True)]
         + [_case("tiny", "native", B, p) for B, p in ((1, 64), (8, 16), (32, 32), (64, 64))]
         + [_case("tiny", "native", 8, 32, splits=32)]
         + [_case("tiny", "chain", B, p) for B, p in ((1, 32), (8, 64), (32, 16))]
         + [_case("tiny", f"fused{lv}", B, p) for lv in (1, 2) for B, p in ((1, 16), (8, 32), (32, 64))]
         + [_case("tiny", "fp8", B, p) for B, p in ((1, 32), (8, 16), (32, 64))]
         + [_case("tiny_w4", f"w4_{k}", B, p) for k in ("mma", "tc5") for B, p in ((1, 16), (8, 64))]
         + [_case("tiny_q3", path, 8, 32) for path in ("default", "fused2")]
         + [_case("small128", "default", B, p) for B, p in ((1, 64), (8, 16), (32, 32))]
         + [_case("l14b", "default", B, 16, ts=False) for B in (1, 8, 32)])


def _id(c):
    extra = "".join(f"-{k}{'' if v is True else v}" for k, v in c.items() if k not in ("kind", "path", "B", "page", "ts"))
    return f"{c['kind']}-{c['path']}-b{c['B']}-p{c['page']}{extra}"


# Fixed bounds against the same-dtype oracle, worst case over the cases of a configuration (tiny: also Qwen3 and the W4 width), over
# steps and checked rows (logits) and over rows, K and V (each layer's cache).  Measured on an H100 80GB HBM3 (700 W), max over cases:
#   tiny      bf16 logits 1.68e-2 kv 1.32e-2   fp16 logits 2.06e-3 kv 1.87e-3
#   small128  bf16 logits 3.14e-2 kv 1.73e-2   fp16 logits 4.82e-3 kv 2.41e-3   (same-dtype oracle vs fp32 oracle: 4.3e-2 / 4.3e-3)
#   l14b      bf16 logits 1.60e-2 kv 2.84e-3   fp16 logits 1.73e-3 kv 7.1e-4
BOUND = {("tiny", BF): dict(logits=2.2e-2, kv=1.7e-2), ("tiny", FP): dict(logits=2.7e-3, kv=2.4e-3),
         ("small128", BF): dict(logits=4e-2, kv=2.3e-2), ("small128", FP): dict(logits=6.2e-3, kv=3.1e-3),
         ("l14b", BF): dict(logits=2.1e-2, kv=4e-3), ("l14b", FP): dict(logits=2.3e-3, kv=1e-3)}
# The KV rows are gated element-wise (no dot product over the hidden width averages their rounding), and a later layer's K / V carry
# every earlier layer's rounding: the GPU's worst element is up to 1.30x (measured, Qwen3 bf16 layer 1) as far from the fp32 oracle
# as the same-dtype oracle's own worst element, so their comparative factor is 1.5 instead of the logits' 1.25
KV_RATIO = 1.5


@pytest.mark.parametrize("dt", [BF, FP], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", CASES, ids=_id)
def test_decode_steps_and_kv_cache_match_the_oracle(case, dt, monkeypatch):
    """Per-step logits of every checked row against both oracles (the comparative gate of tests/gpu_util.py), each produced token is
    the argmax of the logits the step computed, each layer's KV rows against the oracle's cache, and no cache row outside the live
    slots moved."""
    kind, path, B, page = case["kind"], case["path"], case["B"], case["page"]
    monkeypatch.setenv("CTS_NEXT_PREFETCH_MB", "8" if case.get("prefetch") else "0")
    monkeypatch.setenv("CTS_W4_KERNEL", path[3:] if path.startswith("w4") else "mma")
    if case.get("splits"):
        monkeypatch.setenv("CTS_ATTN_SPLITS", str(case["splits"]))
    else:
        monkeypatch.delenv("CTS_ATTN_SPLITS", raising=False)
    cfg, sd, cache, model = _model(kind, dt, path, B, page, case.get("max_seq_len", 512))
    if case.get("prefetch"):
        assert model.next_prefetch_bytes > 0
    proc = _proc(cfg)
    rows = _rows(B, page, with_ts=case.get("ts", True), long=case.get("long", False))
    enc = _encode(proc, rows)
    g = torch.Generator(device=model.device).manual_seed(B + page)
    model.kv.copy_(torch.randn(model.kv.shape, generator=g, device=model.device, dtype=torch.float32).to(dt))   # finite, not zero
    snap = model.kv.clone()
    run = decode_run(model, enc, STEPS)
    st = model._steps[B]
    if case.get("long"):
        assert st.attn_splits == 32 and -(-int(run.seq_lens[0]) // 64) > 8, (st.attn_splits, run.seq_lens)
    if case.get("splits"):
        assert st.attn_splits == case["splits"]

    # the in-graph argmax: every produced token is a maximum of the logits it was picked from
    lgs = torch.cat([run.prefill[None], run.logits])
    picked = lgs.gather(2, run.tokens.t().long()[:, :, None])[..., 0]
    assert torch.equal(picked, lgs.max(2).values)
    assert bool(torch.isfinite(run.logits).all())

    # no cache row outside the live slots moved, every live slot was written
    moved = (model.kv != snap).any(-1).cpu()                                   # [L, 2, pages, nkv, page]
    live = _live_slots(model, run)
    assert torch.equal(moved, live[None, None, :, None, :].expand_as(moved))
    assert int(run.seq_lens.sum()) == int(run.lens.sum()) + B * (STEPS + 1)

    wkind = "fp8" if path == "fp8" else ("w4" if path.startswith("w4") else "dense")
    if wkind == "fp8":
        from tests.test_gpu_fp8 import _fp8_state_dict
        ws = _fp8_state_dict(model, sd[0], dt)
    elif wkind == "w4":
        ws = _dense_state_dict(model, sd[0], dt)
    else:
        ws = sd
    checked = sorted({0, B // 2, B - 1} if kind == "l14b" else {0, 1, 2, 3, 4, B // 2, B - 1} & set(range(B)))
    got, ref, ref32 = [], [], []
    kv_got, kv_ref, kv_ref32 = [[] for _ in range(cfg.num_hidden_layers)], [[] for _ in range(cfg.num_hidden_layers)], [[] for _ in range(cfg.num_hidden_layers)]
    kv = model.kv.cpu()
    for b in checked:
        toks = run.tokens[b, :STEPS].tolist()
        outs = [_oracle(cfg, w, dt, fp32, proc, rows[b], toks, cache, (wkind, fp32, rows[b][0])) for fp32, w in ((False, ws[0]), (True, ws[1]))]
        assert outs[0][1].len == int(run.seq_lens[b]) - 1
        for i in range(STEPS):
            got.append(run.logits[i, b]); ref.append(outs[0][0][i]); ref32.append(outs[1][0][i])
        for l in range(cfg.num_hidden_layers):
            k, v = _kv_rows(kv, page, run, b, l)
            kv_got[l] += [k, v]
            kv_ref[l] += [outs[0][1].k[l], outs[0][1].v[l]]
            kv_ref32[l] += [outs[1][1].k[l], outs[1][1].v[l]]
    name = "decode_parity_" + _id(case)
    bound = BOUND[(kind.split("_")[0], dt)]
    parity_gate(name + "_logits", got, ref, ref32, dt, bound["logits"], rows=str(checked), steps=STEPS)
    for l in range(cfg.num_hidden_layers):
        parity_gate(name + f"_kv_layer{l}", kv_got[l], kv_ref[l], kv_ref32[l], dt, bound["kv"], ratio=KV_RATIO, rows=str(checked))


# ---------------------------------------------------------------------------------------------------------------- isolation
@pytest.mark.parametrize("fill", ["nan", "large"])
@pytest.mark.parametrize("path", ["default", "native"])
@pytest.mark.parametrize("page", [16, 64])
@pytest.mark.parametrize("dt", [BF, FP], ids=["bf16", "fp16"])
def test_decode_does_not_depend_on_cache_rows_it_does_not_own(dt, page, path, fill, monkeypatch):
    """The same batch decoded twice: once on a zeroed KV cache, once on a cache first filled with NaN (or with +-the largest finite
    value).  The prefill writes only the live rows, so a row past a sequence's end in its last page, and a page past its allocated ones
    (page-table entry 0), hold whatever the cache held before; the logits and tokens must be bit-identical and finite."""
    monkeypatch.delenv("CTS_ATTN_SPLITS", raising=False)
    monkeypatch.setenv("CTS_NEXT_PREFETCH_MB", "0")
    cfg, _, _, model = _model("tiny", dt, path, 8, page)
    enc = _encode(_proc(cfg), _rows(8, page))
    model.kv.zero_()
    a = decode_run(model, enc, STEPS)
    if fill == "nan":
        model.kv.fill_(float("nan"))
    else:
        model.kv.fill_(torch.finfo(dt).max)
        model.kv[..., 1::2].neg_()
    b = decode_run(model, enc, STEPS)
    record("decode_isolation", dtype=str(dt), page=page, path=path, fill=fill,
           max_abs_diff=float((a.logits - b.logits).abs().nan_to_num(float("inf")).max()))
    assert bool(torch.isfinite(b.logits).all()) and bool(torch.isfinite(b.prefill).all())
    assert torch.equal(a.prefill, b.prefill)
    assert torch.equal(a.logits, b.logits) and torch.equal(a.tokens, b.tokens)
