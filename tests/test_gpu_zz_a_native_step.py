"""cts_decoder_step / cts_rmsnorm / cts_lm_head (csrc/decoder_step.cu: host-side executors over the validated kernels) against
the per-kernel Python orchestration: the same launches in the same order must give bit-identical tokens and logits.
Plain tests (no xfail markers)."""
import numpy as np
import pytest
import torch

from tests.gpu_util import ctx

pytestmark = pytest.mark.gpu
DT = torch.bfloat16


def _models(qwen3, graph):
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig.tiny()
    if qwen3:
        cfg.qk_norm, cfg.attention_bias = True, False
    sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=DT, std=0.05)
    kw = dict(dtype=DT, max_batch=4, max_seq_len=256, page_size=16, use_cuda_graph=graph)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    return ChatTSForCausalLM(cfg, sd, **kw), ChatTSForCausalLM(cfg, sd, use_native_step=True, **kw), proc


@pytest.mark.parametrize("qwen3,graph", [(False, False), (True, True)])
def test_native_step_is_bit_identical(qwen3, graph):
    ref, native, proc = _models(qwen3, graph)
    x = np.arange(256)
    enc = proc(text=["A <ts><ts/> ?", "text only, longer prompt to pad the first"], timeseries=[np.sin(x / 9) * 4], return_tensors="pt")
    a = ref.generate(**enc, max_new_tokens=24, ignore_eos=True)
    b = native.generate(**enc, max_new_tokens=24, ignore_eos=True)
    assert torch.equal(a, b)


def test_rmsnorm_and_lm_head_aliases():
    c = ctx()
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(9, 256, generator=g)).to(DT).cuda()
    w = (torch.rand(256, generator=g) + 0.5).to(DT).cuda()
    a, b = torch.empty_like(x), torch.empty_like(x)
    c.rmsnorm(x, w, 1e-6, a)
    c.reduce_residual_rmsnorm(None, 0, x, None, w, 1e-6, b)
    wl = (torch.randn(1000, 256, generator=g) * 0.05).to(DT).cuda()
    la, lb = torch.empty(9, 1000, device="cuda", dtype=DT), torch.empty(9, 1000, device="cuda", dtype=DT)
    c.lm_head(x, wl, la)
    c.gemm(x, wl, lb)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(la, lb)


@pytest.mark.parametrize("n_series,lens", [(3, [256, 100, 37]), (16, [256] * 16)])
def test_ts_encode_executor_matches_python_orchestration(n_series, lens):
    """cts_ts_encode (counts + patchify + MLP from one C call) == TimeSeriesEmbedding.encode (the same launches from Python)."""
    from chatts_b200 import ChatTSConfig
    from chatts_b200.processor import sp_encoding
    from chatts_b200.ts_encoder import TimeSeriesEmbedding
    from chatts_b200.weights import synthetic_state_dict
    c = ctx()
    cfg = ChatTSConfig.tiny()
    sd = synthetic_state_dict(cfg, seed=4, device="cpu", dtype=DT, std=0.05)
    ts_w = {k: v for k, v in sd.items() if k.startswith("ts_encoder.")}
    enc = TimeSeriesEmbedding(cfg.ts, ts_w, dtype=DT)
    series = [sp_encoding(np.sin(np.arange(L) / 7.0) * (i + 1))[0] for i, L in enumerate(lens)]
    Lmax = max(e.shape[0] for e in series)
    x = np.zeros((n_series, Lmax, 1))
    for i, e in enumerate(series):
        x[i, : e.shape[0]] = e
    xt = torch.from_numpy(x).to(torch.float32)
    feats, cnt = enc.encode(xt)
    total = int(cnt.sum())
    out = torch.full((total, enc.hidden_size), float("nan"), device="cuda", dtype=DT)
    valid, pc, off = c.ts_encode(xt.cuda().to(DT), enc.num_features, enc.patch_size, enc.mode, enc.pos_table, enc.embedding_dim,
                                 enc.max_sequence_length, enc.w, enc.b, total, out)
    torch.cuda.synchronize()
    assert pc.cpu().tolist() == cnt.tolist() and torch.equal(out, feats)
    # scattered variant: rows land at row_map positions of a bigger buffer
    perm = torch.randperm(total + 5, generator=torch.Generator().manual_seed(1))[:total].to(torch.int32)
    big = torch.zeros(total + 5, enc.hidden_size, device="cuda", dtype=DT)
    c.ts_encode(xt.cuda().to(DT), enc.num_features, enc.patch_size, enc.mode, enc.pos_table, enc.embedding_dim, enc.max_sequence_length,
                enc.w, enc.b, total, big, row_map=perm.cuda())
    torch.cuda.synchronize()
    assert torch.equal(big[perm.long().cuda()], feats)


def test_continuous_engine_on_the_captured_decode_graph():
    """engine.ContinuousEngine on the GPU: requests join / leave the static slots between CUDA-graph replays; every request
    reproduces the tokens it gets when it is served alone at the same decode width (same kernels, same split factors, rows
    independent), and its first token is generate()'s."""
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.engine import ContinuousEngine
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig.tiny()
    sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=DT, std=0.05)
    model = ChatTSForCausalLM(cfg, sd, dtype=DT, max_batch=4, max_seq_len=256, page_size=16, use_cuda_graph=True)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    x = np.arange(200)
    specs = [("A <ts><ts/> ?", [np.sin(x / 9) * 4], 9), ("plain text", [], 5), ("B <ts><ts/> and <ts><ts/>", [x * 0.05, np.cos(x / 5)[:77]], 12),
             ("short", [], 2), ("one more plain prompt", [], 7), ("C <ts><ts/>", [np.sin(x / 3)], 6)]
    encs = [(proc(text=[t], timeseries=s, return_tensors="pt"), n) for t, s, n in specs]
    # reference: the same engine serving ONE request at a time (prefill alone, decode width 4 with three dummy slots) -- identical
    # kernel shapes and split factors, so row independence makes the crowded run reproduce it exactly
    ref = []
    for enc, n in encs:
        solo = ContinuousEngine(model, slots=4, steps_per_round=3, max_prefill_batch=1)
        solo.add_request(enc["input_ids"][0], enc["timeseries"], max_new_tokens=n, ignore_eos=True)
        ref.append(solo.run()[0].tokens)
        solo.close()
    one = model.generate(**encs[0][0], max_new_tokens=1, ignore_eos=True)[0, -1].item()
    assert ref[0][0] == one                                                   # same first token as generate() (same prefill shape)
    pages0 = len(model.pool.free)
    eng = ContinuousEngine(model, slots=4, steps_per_round=3, max_prefill_batch=1)
    for enc, n in encs:
        eng.add_request(enc["input_ids"][0], enc["timeseries"], max_new_tokens=n, ignore_eos=True)
    done = eng.run()
    eng.close()
    assert [r.tokens for r in done] == ref
    assert len(model.pool.free) == pages0 and max(eng.occupancy) <= 4
