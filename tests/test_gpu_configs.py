"""BASELINE.json configs as parity cases (tiny decoder so the CPU oracle finishes in seconds; the TS side at the
configs' real series counts / lengths), plus full-size-shape checks against the oracle where the CPU can afford it."""
import os

import numpy as np
import pytest
import torch

from oracle import decoder as od
from oracle import merge as om
from oracle import ts_encoder as ote
from tests.gpu_util import parity_gate, record, rel_err

pytestmark = pytest.mark.gpu
DT = torch.bfloat16


BOTH = pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])       # fp16 = the dtype the reference runs (SURVEY.md F5)


def _mk(seed=0, max_batch=32, max_seq_len=1024, dt=DT, **kw):
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig.tiny(**kw)
    cfg.ts = dict(cfg.ts, max_sequence_length=1024)
    sd = synthetic_state_dict(cfg, seed=77 + seed, device="cpu", dtype=dt, std=0.05)
    model = ChatTSForCausalLM(cfg, sd, dtype=dt, max_batch=max_batch, max_seq_len=max_seq_len, page_size=64)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    return cfg, sd, model, proc


def _oracle_last_logits(cfg, sd, enc, samples, fp32=False):
    """Next-token logits of the given samples by the oracle, in the dtype of ``sd`` (the reference's rounding points) or, with
    fp32=True, with every weight and activation in fp32 (same 16-bit weight VALUES, the series as the model dtype sees them)."""
    dt = sd["model.embed_tokens.weight"].dtype
    if fp32:
        sd = {k: v.float() for k, v in sd.items()}
    ts_w = {k[len("ts_encoder."):]: v for k, v in sd.items() if k.startswith("ts_encoder.")}
    x = enc["timeseries"].to(dt)
    feats, pc = ote.forward(x.float() if fp32 else x, cfg.ts, ts_w)
    embeds = om.hf_merge(enc["input_ids"], enc["attention_mask"], sd["model.embed_tokens.weight"], feats, pc.tolist(),
                         cfg.ts_token_start_index)
    out = {}
    for b in samples:
        st = od.State(cfg.num_hidden_layers)
        out[b] = (od.logits(od.forward_hidden(embeds[b], sd, cfg.to_dict(), st)[-1:], sd)[0], embeds[b].shape[0])
    return out, pc


def _gate(name, lg, cfg, sd, enc, samples, dt, fixed, **extra):
    """Comparative parity gate (tests/gpu_util.py:parity_gate) on the next-token logits of ``samples``."""
    ref, pc = _oracle_last_logits(cfg, sd, enc, samples)
    ref32, _ = _oracle_last_logits(cfg, sd, enc, samples, fp32=True)
    parity_gate(name, [lg[b] for b in samples], [ref[b][0] for b in samples], [ref32[b][0] for b in samples], dt, fixed, **extra)
    return ref, pc


@BOTH
def test_config2_batch32_variable_length_series_prefill(dt):
    """configs[2]: batch-32 prefill, 8 variable-length series (64-1024) per sample, sp-mask path."""
    cfg, sd, model, proc = _mk(max_seq_len=2048, dt=dt)
    rng = np.random.default_rng(2)
    prompts, series = [], []
    for b in range(32):
        lens = rng.integers(64, 1025, size=8)
        prompts.append(" ".join(f"s{k} <ts><ts/>" for k in range(8)) + f" q{b}?" * int(rng.integers(1, 4)))
        series += [rng.normal(size=int(n)) * rng.uniform(0.1, 30) + rng.uniform(-5, 5) for n in lens]
    enc = proc(text=prompts, timeseries=series, padding=True, return_tensors="pt")
    lens_all = [len(s) for s in series]
    lg = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0]

    ref, pc = _gate("config2_batch32_varlen_prefill", lg, cfg, sd, enc, [0, 13, 31], dt, 1.85e-2 if dt == torch.bfloat16 else 2.1e-3)
    assert pc.tolist() == [(n + 15) // 16 for n in lens_all]                 # bit-exact patch counts for 256 ragged series


def test_config3_batch8_30_series_len512_decode():
    """configs[3] workload on one GPU: batch-8 decode, 30 series x len-512 per sample (960 patch rows each)."""
    cfg, sd, model, proc = _mk(seed=1, max_batch=8, max_seq_len=4608, max_position_embeddings=8192)
    rng = np.random.default_rng(3)
    prompts = [" ".join(f"m{k}: <ts><ts/>" for k in range(30)) + " summarize." for _ in range(8)]
    series = [np.cumsum(rng.normal(size=512)) for _ in range(8 * 30)]
    enc = proc(text=prompts, timeseries=series, padding=True, return_tensors="pt")
    new = 6
    ids = model.generate(**enc, max_new_tokens=new, ignore_eos=True)
    S = enc["input_ids"].shape[1]
    ts_w = {k[len("ts_encoder."):]: v for k, v in sd.items() if k.startswith("ts_encoder.")}
    feats, pc = ote.forward(enc["timeseries"].to(DT), cfg.ts, ts_w)
    assert pc.tolist() == [32] * 240
    embeds = om.hf_merge(enc["input_ids"], enc["attention_mask"], sd["model.embed_tokens.weight"], feats, pc.tolist(),
                         cfg.ts_token_start_index)
    worst = 0.0
    for b in (0, 7):
        assert embeds[b].shape[0] == int(enc["attention_mask"][b].sum()) + 960
        st = od.State(cfg.num_hidden_layers)
        lg = od.logits(od.forward_hidden(embeds[b], sd, cfg.to_dict(), st)[-1:], sd)[0].float()
        for tok in ids[b, S:].tolist():
            worst = max(worst, float((lg.max() - lg[tok]) / lg.abs().max()))
            lg = od.logits(od.forward_hidden(sd["model.embed_tokens.weight"][tok][None], sd, cfg.to_dict(), st), sd)[0].float()
    record("config3_batch8_30x512_decode", worst_gap_rel=worst)
    assert worst < 1e-2      # every produced token is the oracle's argmax or within 1e-2 of max|logit| of it (measured: 0)


def test_config1_single_series_128_new_tokens():
    """configs[1]: 1 series len-256, max_new_tokens=128 (tiny decoder): teacher-forced agreement with the oracle."""
    cfg, sd, model, proc = _mk(seed=2, max_batch=2, max_seq_len=512)
    x = np.arange(256)
    enc = proc(text=["What happens in <ts><ts/>?"], timeseries=[np.sin(x / 10) * 5], return_tensors="pt")
    ids = model.generate(**enc, max_new_tokens=128, ignore_eos=True)
    S = enc["input_ids"].shape[1]
    assert ids.shape == (1, S + 128)
    ts_w = {k[len("ts_encoder."):]: v for k, v in sd.items() if k.startswith("ts_encoder.")}
    feats, pc = ote.forward(enc["timeseries"].to(DT), cfg.ts, ts_w)
    e = om.hf_merge(enc["input_ids"], enc["attention_mask"], sd["model.embed_tokens.weight"], feats, pc.tolist(), cfg.ts_token_start_index)[0]
    st = od.State(cfg.num_hidden_layers)
    lg = od.logits(od.forward_hidden(e, sd, cfg.to_dict(), st)[-1:], sd)[0].float()
    worst, exact = 0.0, 0
    for tok in ids[0, S:].tolist():
        worst = max(worst, float((lg.max() - lg[tok]) / lg.abs().max()))
        exact += int(int(lg.argmax()) == tok)
        lg = od.logits(od.forward_hidden(sd["model.embed_tokens.weight"][tok][None], sd, cfg.to_dict(), st), sd)[0].float()
    record("config1_128_new_tokens", worst_gap_rel=worst, exact=exact)
    assert worst < 1e-2 and exact >= 118


def test_vllm_layout_overwrite_matches_oracle():
    """vLLM surface layout (chatts_vllm.py:405-415,569-573): P copies of <ts> overwritten in order."""
    from chatts_b200 import layout as L
    cfg, sd, model, proc = _mk(seed=3, max_batch=2, max_seq_len=512)
    x = np.arange(100)
    v = proc(text=["a <ts><ts/> b <ts><ts/> c"], timeseries=[np.sin(x / 5), x * 0.1], vllm_flag=True)
    toks = proc.tokenizer.encode(v["text"][0])
    enc_ts = torch.from_numpy(np.concatenate([np.pad(e[1], ((0, 0), (0, 200 - e[1].shape[1]), (0, 0))) for e in v["timeseries"]])).float()
    pcs = [7, 7]
    # replace every [<ts>, <ts/>] by P placeholders (the prefix tokens are already in the text)
    exp = L.expand_prompt_vllm(toks, [[cfg.ts_token_start_index]] * 2, pcs, cfg.ts_token_start_index)
    ids = torch.tensor([exp])
    lg = model.forward(ids, None, enc_ts, layout_kind="vllm").logits[0, 0]
    ts_w = {k[len("ts_encoder."):]: v2 for k, v2 in sd.items() if k.startswith("ts_encoder.")}
    feats, pc = ote.forward(enc_ts.to(DT), cfg.ts, ts_w)
    assert pc.tolist() == pcs
    emb = om.vllm_merge(ids, sd["model.embed_tokens.weight"], feats, cfg.ts_token_start_index)
    st = od.State(cfg.num_hidden_layers)
    ref = od.logits(od.forward_hidden(emb, sd, cfg.to_dict(), st)[-1:], sd)[0]
    e = rel_err(lg, ref)
    record("vllm_layout", err=e)
    assert e < 1e-2


def test_from_pretrained_safetensors_roundtrip(tmp_path):
    import json
    from safetensors.torch import save_file
    from chatts_b200.model import ChatTSForCausalLM
    cfg, sd, model, proc = _mk(seed=4, max_batch=2, max_seq_len=256)
    d = tmp_path / "ckpt"
    d.mkdir()
    json.dump(cfg.to_dict(), open(d / "config.json", "w"))
    names = sorted(sd)
    save_file({k: sd[k].contiguous() for k in names[: len(names) // 2]}, str(d / "model-00001-of-00002.safetensors"))
    save_file({k: sd[k].contiguous() for k in names[len(names) // 2:]}, str(d / "model-00002-of-00002.safetensors"))
    m2 = ChatTSForCausalLM.from_pretrained(str(d), device_map=0, torch_dtype="bfloat16", max_batch=2, max_seq_len=256, page_size=64)
    ids = torch.randint(0, 900, (1, 20))
    assert torch.equal(model.forward(ids).logits, m2.forward(ids).logits)
    assert m2.config.ts["patch_size"] == 16


def test_full_size_ts_encoder_vs_oracle():
    """The metric workload's TS encoder at the real ChatTS-14B shapes (5 x 5120-wide layers, 8 series x 256 points =
    128 patch rows) against the CPU oracle in bf16."""
    from chatts_b200 import ChatTSConfig
    from chatts_b200.ts_encoder import TimeSeriesEmbedding
    from chatts_b200.weights import synthetic_state_dict, ts_encoder_shapes
    cfg = ChatTSConfig.chatts_14b()
    g = torch.Generator().manual_seed(5)
    w = {k: (torch.randn(s, generator=g) * 0.02).to(DT) for k, s in ts_encoder_shapes(cfg).items()}
    enc = TimeSeriesEmbedding(cfg.ts, w, dtype=DT)
    from chatts_b200.processor import sp_encoding
    rng = np.random.default_rng(0)
    x = torch.from_numpy(np.stack([sp_encoding(np.cumsum(rng.normal(size=256)))[0] for _ in range(8)])).to(DT)
    feats, pc = enc(x.cuda())
    assert pc.tolist() == [16] * 8 and feats.shape == (128, 5120)
    ref, _ = ote.forward(x, cfg.ts, {k[len("ts_encoder."):]: v for k, v in w.items()})
    e = rel_err(feats, ref)
    record("full_size_ts_encoder", err=e)
    assert e < 6e-3


def test_full_size_decoder_layer_vs_oracle():
    """One decoder layer at the real ChatTS-14B shapes (hidden 5120, 40/8 heads x 128, inter 13824), small vocab:
    prefill of 40 positions + 3 cached decode steps against the CPU oracle (bf16)."""
    from chatts_b200 import ChatTSConfig
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig(num_hidden_layers=1, vocab_size=512, ts_token_start_index=500, eos_token_id=510, pad_token_id=511,
                       max_position_embeddings=1024)
    sd = synthetic_state_dict(cfg, seed=9, device="cpu", dtype=DT)
    model = ChatTSForCausalLM(cfg, sd, dtype=DT, max_batch=2, max_seq_len=256, page_size=64)
    ids = torch.randint(0, 480, (1, 40), generator=torch.Generator().manual_seed(1))
    out = model.generate(input_ids=ids, max_new_tokens=4, ignore_eos=True)
    lg = model.forward(ids).logits[0, 0]
    st = od.State(1)
    e0 = sd["model.embed_tokens.weight"][ids[0]]
    ref = od.logits(od.forward_hidden(e0, sd, cfg.to_dict(), st)[-1:], sd)[0]
    err = rel_err(lg, ref)
    worst = 0.0
    lgf = ref.float()
    for tok in out[0, 40:].tolist():
        worst = max(worst, float((lgf.max() - lgf[tok]) / lgf.abs().max()))
        lgf = od.logits(od.forward_hidden(sd["model.embed_tokens.weight"][tok][None], sd, cfg.to_dict(), st), sd)[0].float()
    record("full_size_decoder_layer", err=err, worst_gap_rel=worst)
    assert err < 1.4e-2 and worst < 1e-2


@BOTH
def test_chatts_8b_qwen3_variant_matches_oracle(dt):
    """ChatTS-8B decoder family (Qwen3: per-head q/k RMSNorm before RoPE, no qkv bias; chatts_vllm.py:633-668)."""
    cfg, sd, model, proc = _mk(seed=6, max_batch=2, max_seq_len=512, dt=dt, qk_norm=True, attention_bias=False)
    assert "model.layers.0.self_attn.q_norm.weight" in sd and "model.layers.0.self_attn.q_proj.bias" not in sd
    x = np.arange(200)
    enc = proc(text=["Q3 <ts><ts/> end", "no ts"], timeseries=[np.cos(x / 7) * 3], padding=True, return_tensors="pt")
    lg = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0]
    _gate("chatts_8b_qwen3_variant", lg, cfg, sd, enc, [0, 1], dt, 1.8e-2 if dt == torch.bfloat16 else 2.2e-3)      # measured: 1.18e-2 (bf16), 1.45e-3 (fp16)
    ids = model.generate(**enc, max_new_tokens=10, ignore_eos=True)
    assert ids.shape[1] == enc["input_ids"].shape[1] + 10


def test_lora_merge_and_unload_matches_oracle(tmp_path):
    """demo/demo_lora.ipynb cells 3-4: PeftModel.from_pretrained(...).merge_and_unload() -> adapters folded into the weights."""
    import json
    from safetensors.torch import save_file
    cfg, sd, model, proc = _mk(seed=8, max_batch=2, max_seq_len=512)
    g = torch.Generator().manual_seed(4)
    r, alpha = 8, 16
    ad, sd2 = {}, {k: v.clone() for k, v in sd.items()}
    for l in range(cfg.num_hidden_layers):
        for blk, proj in (("self_attn", "q_proj"), ("self_attn", "k_proj"), ("self_attn", "v_proj"), ("self_attn", "o_proj"),
                          ("mlp", "gate_proj"), ("mlp", "up_proj"), ("mlp", "down_proj")):
            w = sd[f"model.layers.{l}.{blk}.{proj}.weight"]
            A = torch.randn(r, w.shape[1], generator=g) * 0.05
            B = torch.randn(w.shape[0], r, generator=g) * 0.05
            ad[f"base_model.model.model.layers.{l}.{blk}.{proj}.lora_A.weight"] = A
            ad[f"base_model.model.model.layers.{l}.{blk}.{proj}.lora_B.weight"] = B
            sd2[f"model.layers.{l}.{blk}.{proj}.weight"] = (w.float() + (alpha / r) * (B @ A)).to(DT)
    d = tmp_path / "adapter"
    d.mkdir()
    save_file(ad, str(d / "adapter_model.safetensors"))
    json.dump({"r": r, "lora_alpha": alpha, "target_modules": ["q_proj"]}, open(d / "adapter_config.json", "w"))
    x = np.arange(128)
    enc = proc(text=["lora <ts><ts/> ?"], timeseries=[np.sin(x / 9.0)], return_tensors="pt")
    before = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0].clone()
    assert model.merge_lora(str(d)) == 7 * cfg.num_hidden_layers
    lg = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0]
    ref, _ = _oracle_last_logits(cfg, sd2, enc, samples=[0])
    e = rel_err(lg[0], ref[0][0])
    record("lora_merge", err=e, moved=rel_err(lg[0], before[0]))
    assert e < 1.3e-2 and rel_err(lg[0], before[0]) > 5e-2          # matches the merged oracle (measured 8.7e-3), and really changed
