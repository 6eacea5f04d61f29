"""cts_gemm_w4 (csrc/gemm_w4.cu: W4A16 decode GEMM, the 4-bit codes dequantised inside the TMA -> shared memory -> wgmma operand
path) against cts_gemm on the dequantised weight -- the same values through the same MMA order, so the fp32 split-K partials must be
BIT-IDENTICAL -- and the whole model decoding through the packed weights against decoding through the dense copy."""
import numpy as np
import pytest
import torch

from tests.gpu_util import ctx, decode_run, record

pytestmark = pytest.mark.gpu
EPI_PARTIAL = 3


def _rand_w4(n, k, gs, dtype, seed):
    from chatts_b200.weights import dequantize_w4
    g = torch.Generator().manual_seed(seed)
    qw = torch.randint(0, 256, (n, k // 2), generator=g, dtype=torch.uint8)
    sc = ((torch.rand(n, k // gs, generator=g) + 0.5) * 0.01).to(dtype)
    zp = torch.randint(1, 17, (n, k // gs), generator=g, dtype=torch.uint8)
    return qw, sc, zp, dequantize_w4(qw, sc, zp, gs)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n,k,gs,t,split", [(256, 512, 128, 1, 1), (256, 512, 128, 5, 2), (384, 1024, 128, 17, 3), (128, 256, 64, 32, 4),
                                            (200, 768, 128, 8, 2), (1024, 2560, 128, 32, 7), (7168, 5120, 128, 32, 7), (5120, 13824, 128, 1, 11),
                                            (256, 5120, 128, 8, 1), (27648, 5120, 128, 32, 1)])          # unsplit K: every staging slot reused 6 times
def test_w4_partials_bit_identical_to_the_dense_gemm(n, k, gs, t, split, dtype):
    c = ctx()
    qw, sc, zp, w = _rand_w4(n, k, gs, dtype, seed=n + k + t)
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(t, k, generator=g) * 0.5).to(dtype).cuda()
    ref = torch.full((split, t, n), float("nan"), device="cuda")
    got = torch.full((split, t, n), float("nan"), device="cuda")
    c.gemm(x, w.cuda(), ref, epilogue=EPI_PARTIAL, split_k=split, t=t)
    c.gemm_w4(x, qw.cuda(), sc.cuda(), zp.cuda(), gs, got, split, t=t)
    torch.cuda.synchronize()
    same = torch.equal(got, ref)
    record("gemm_w4", n=n, k=k, t=t, split=split, dtype=str(dtype), bit_identical=int(same),
           max_abs_diff=float((got - ref).abs().max()) if not same else 0.0)
    assert same


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n,k,gs,t,split", [(256, 512, 128, 1, 1), (256, 512, 128, 5, 2), (384, 1024, 128, 17, 3), (128, 256, 64, 32, 2),
                                            (200, 768, 128, 8, 2), (1024, 2560, 128, 32, 7), (7168, 5120, 128, 32, 5), (5120, 13824, 128, 1, 11),
                                            (256, 5120, 128, 9, 1), (27648, 5120, 128, 32, 2), (27648, 5120, 128, 3, 8), (5120, 13824, 256, 16, 7),
                                            (528, 1536, 64, 24, 3)])
def test_w4_mma_partials_match_the_dense_gemm(n, k, gs, t, split, dtype):
    """cts_gemm_w4_mma (registers + mma.sync, persistent CTAs over (tile, split) units, every ring slot reused many times at the big
    shapes): the same 16-bit operand values as the dense copy, so a result may differ from the dense path only by the fp32 summation order.
    Its K ranges are cut at multiples of 128 (a pipeline stage), cts_gemm's at multiples of 64, so (a) each partial is checked against an
    fp32 matmul of the dequantised weight over ITS range and (b) the sum of the partials against the sum of cts_gemm's -- bound 2e-5 of
    the largest magnitude (measured: a few 1e-7)."""
    from chatts_b200.weights import repack_w4_mma
    c = ctx()
    qw, sc, zp, w = _rand_w4(n, k, gs, dtype, seed=n + k + t)
    qwf, szp = repack_w4_mma(qw, sc, zp, gs)
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(t, k, generator=g) * 0.5).to(dtype).cuda()
    ref = torch.full((split, t, n), float("nan"), device="cuda")
    got = torch.full((split, t, n), float("nan"), device="cuda")
    c.gemm(x, w.cuda(), ref, epilogue=EPI_PARTIAL, split_k=split, t=t)
    c.gemm_w4_mma(x, qwf.cuda(), szp.cuda(), n, gs, got, split, t=t)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(got).all())
    ks = k // 128
    w32, x32 = w.float().cuda(), x.float()
    want = torch.stack([x32[:, (ks * s_) // split * 128:(ks * (s_ + 1)) // split * 128] @ w32[:, (ks * s_) // split * 128:(ks * (s_ + 1)) // split * 128].t()
                        for s_ in range(split)])
    err = float((got - want).abs().max() / want.abs().max())
    err_sum = float((got.sum(0) - ref.sum(0)).abs().max() / ref.sum(0).abs().max())
    record("gemm_w4_mma", n=n, k=k, t=t, split=split, dtype=str(dtype), rel_err=err, rel_err_sum_vs_dense_gemm=err_sum)
    assert err <= 2e-5 and err_sum <= 2e-5


def test_w4_suggested_split_keeps_the_group_table_in_range():
    c = ctx()
    for n, k in ((7168, 5120), (5120, 5120), (27648, 5120), (5120, 13824), (256, 256)):
        s = c.gemm_w4_suggest_split(n, k)
        blocks = -(-(-(-k // 64)) // s) + 1
        assert 1 <= s <= 16 and blocks * 64 // 128 + 2 <= 44


@pytest.mark.parametrize("kernel", ["mma", "tc5"])
@pytest.mark.parametrize("qwen3", [False, True])
def test_model_decodes_through_the_packed_weights(qwen3, kernel, monkeypatch):
    """quantize_w4_synthetic: dense weights = the dequantised values, packed copy attached; the decode step through cts_gemm_w4 (its own
    split factors) must pick the tokens the dense decode picks (same weights; fp32 summation order differs with the split)."""
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    monkeypatch.setenv("CTS_W4_KERNEL", kernel)
    cfg = ChatTSConfig.tiny(intermediate_size=768)
    if qwen3:
        cfg.qk_norm, cfg.attention_bias = True, False
    sd = synthetic_state_dict(cfg, seed=5, device="cpu", dtype=torch.bfloat16, std=0.05)
    model = ChatTSForCausalLM(cfg, sd, dtype=torch.bfloat16, max_batch=4, max_seq_len=256, page_size=16)
    model.quantize_w4_synthetic(group_size=64)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    x = np.arange(200)
    enc = proc(text=["A <ts><ts/> ?", "text only, a longer prompt"], timeseries=[np.sin(x / 9) * 4], padding=True, return_tensors="pt")
    l0 = model.ctx.launches
    a = model.generate(**enc, max_new_tokens=16, ignore_eos=True)
    assert model.w4 is not None and model.w4["kernel"] == kernel and model.ctx.launches > l0
    lg4 = decode_run(model, enc, 1).logits[0]
    w4, model.w4, model._steps = model.w4, None, {}
    b = model.generate(**enc, max_new_tokens=16, ignore_eos=True)
    lgd = decode_run(model, enc, 1).logits[0]
    S = enc["input_ids"].shape[1]
    agree = [int(next((i for i in range(16) if a[r, S + i] != b[r, S + i]), 16)) for r in range(2)]
    err = float((lg4 - lgd).abs().max() / lgd.abs().max())
    record("w4_model_decode", qwen3=int(qwen3), kernel=kernel, greedy_agreement=str(agree), first_step_logits_rel_err=err)
    assert min(agree) >= 12          # same weights; only the K partition of the fp32 sums differs
    assert err <= 1e-2               # ... which moves a few activations by one 16-bit ulp


def test_gptq_checkpoint_directory_decodes_through_the_packed_weights(tmp_path):
    """The load path a user takes (README.md:52,262-263): a GPTQ-Int4 checkpoint DIRECTORY (qweight / qzeros / scales / g_idx per
    projection + quantization_config) through from_pretrained -> packed decode weights attached (mma kernel), prefill on the dequantised
    copy; the greedy continuation equals the one through the model's own dense copy; CTS_W4=0 loads the dequantised weights only."""
    import json
    import os
    from safetensors.torch import save_file
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import pack_gptq_linear, synthetic_state_dict
    cfg = ChatTSConfig.tiny(intermediate_size=768)
    sd = synthetic_state_dict(cfg, seed=9, device="cpu", dtype=torch.bfloat16, std=0.05)
    out = {}
    for k, v in sd.items():
        if ".layers." in k and k.endswith("_proj.weight"):
            qw, qz, sc, gi = pack_gptq_linear(v.float(), 128, 1)
            base = k[: -len(".weight")]
            out.update({base + ".qweight": qw, base + ".qzeros": qz, base + ".scales": sc, base + ".g_idx": gi})
        else:
            out[k] = v.contiguous()
    d = tmp_path / "ckpt"
    d.mkdir()
    conf = cfg.to_dict()
    conf["quantization_config"] = {"bits": 4, "group_size": 128, "quant_method": "gptq"}
    json.dump(conf, open(d / "config.json", "w"))
    save_file(out, str(d / "model.safetensors"))
    kw = dict(torch_dtype="bfloat16", max_batch=4, max_seq_len=256, page_size=16)
    m4 = ChatTSForCausalLM.from_pretrained(str(d), **kw)
    assert m4.w4 is not None and m4.w4["kernel"] == "mma" and m4.w4["group_size"] == 128
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    x = np.arange(200)
    enc = proc(text=["A <ts><ts/> ?", "text only, a longer prompt"], timeseries=[np.cos(x / 7) * 3], padding=True, return_tensors="pt")
    a = m4.generate(**enc, max_new_tokens=12, ignore_eos=True)
    # the same weights through the dequantised dense copy the prefill uses (a CTS_W4=0 load would keep the fp16 scales un-rounded:
    # other weights, not a comparison of kernels)
    m4.w4, m4._steps = None, {}
    b = m4.generate(**enc, max_new_tokens=12, ignore_eos=True)
    S = enc["input_ids"].shape[1]
    agree = [int(next((i for i in range(12) if a[r, S + i] != b[r, S + i]), 12)) for r in range(2)]
    record("w4_gptq_checkpoint_dir", greedy_agreement=str(agree))
    assert min(agree) >= 9
    os.environ["CTS_W4"] = "0"
    try:
        md = ChatTSForCausalLM.from_pretrained(str(d), **kw)
    finally:
        del os.environ["CTS_W4"]
    assert md.w4 is None and md.generate(**enc, max_new_tokens=4, ignore_eos=True).shape[1] == S + 4
