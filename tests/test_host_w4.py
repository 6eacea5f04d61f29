"""W4A16 (GPTQ-Int4, README.md:52,262-263) host logic on CPU: the repacked layout round-trips the checkpoint tensors, the model's
decode step through the packed weights equals the decode step through the dequantised dense weights (C-ABI double), a GPTQ
checkpoint directory loads with the packed copy attached, act-order checkpoints fall back to the dense weights."""
import json

import numpy as np
import pytest
import torch

from tests.test_host_model import _build, _series


def test_repack_round_trip_and_scale_rounding():
    from chatts_b200.weights import dequantize_gptq_linear, dequantize_w4, pack_gptq_linear, repack_gptq_w4
    g = torch.Generator().manual_seed(1)
    w = torch.randn(192, 384, generator=g) * 0.05
    for zo in (0, 1):
        qw, qz, sc, gi = pack_gptq_linear(w, 128, zo)
        for dt in (torch.float16, torch.bfloat16):
            a, b, c = repack_gptq_w4(qw, qz, sc, 128, zo, dt)
            assert a.dtype == torch.uint8 and a.shape == (192, 192) and b.shape == c.shape == (192, 3)
            want = dequantize_gptq_linear(qw, qz, sc, None, 128, zo, dt, scale_dtype=dt)
            assert torch.equal(dequantize_w4(a, b, c, 128), want)
        # fp16: rounding the scale to the model dtype changes nothing (the checkpoint stores fp16 scales)
        assert torch.equal(dequantize_gptq_linear(qw, qz, sc, None, 128, zo, torch.float16, scale_dtype=torch.float16),
                           dequantize_gptq_linear(qw, qz, sc, None, 128, zo, torch.float16))


def _gptq_checkpoint(tmp_path, cfg, sd, act_order=False):
    from safetensors.torch import save_file
    from chatts_b200.weights import pack_gptq_linear
    out = {}
    for k, v in sd.items():
        if ".layers." in k and k.endswith("_proj.weight"):
            qw, qz, sc, gi = pack_gptq_linear(v.float(), 64, 1)
            if act_order:
                gi = gi.flip(0).contiguous()
            base = k[: -len(".weight")]
            out.update({base + ".qweight": qw, base + ".qzeros": qz, base + ".scales": sc, base + ".g_idx": gi})
        else:
            out[k] = v.contiguous()
    d = tmp_path / ("ckpt_ao" if act_order else "ckpt")
    d.mkdir()
    conf = cfg.to_dict()
    conf["quantization_config"] = {"bits": 4, "group_size": 64, "quant_method": "gptq"}
    json.dump(conf, open(d / "config.json", "w"))
    save_file(out, str(d / "model.safetensors"))
    return str(d)


@pytest.mark.parametrize("kernel", ["mma", "tc5"])
def test_gptq_checkpoint_decodes_through_the_packed_weights(cabi_double, tmp_path, monkeypatch, kernel):
    from chatts_b200.model import ChatTSForCausalLM
    monkeypatch.setenv("CTS_W4_KERNEL", kernel)
    cfg, sd, _, proc = _build(cabi_double)
    if kernel == "mma":          # the mma kernel's pipeline stage is 128 K wide: the tiny config's 704-wide MLP (5.5 x 128) is for the wgmma kernel
        from chatts_b200.weights import synthetic_state_dict
        cfg.intermediate_size = 768
        sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=torch.bfloat16, std=0.05)
    path = _gptq_checkpoint(tmp_path, cfg, sd)
    kw = dict(device="cpu", torch_dtype="bfloat16", max_batch=4, max_seq_len=512, page_size=16, use_cuda_graph=False)
    m4 = ChatTSForCausalLM.from_pretrained(path, **kw)
    assert m4.w4 is not None and m4.w4["group_size"] == 64 and len(m4.w4["gu"]) == cfg.num_hidden_layers
    monkeypatch.setenv("CTS_W4", "0")
    md = ChatTSForCausalLM.from_pretrained(path, **kw)
    assert md.w4 is None
    enc = proc(text=["A <ts><ts/> and B <ts><ts/> ?", "text only"], timeseries=list(_series()), padding=True, return_tensors="pt")
    calls = []
    entry = "gemm_w4_mma" if kernel == "mma" else "gemm_w4"
    orig = getattr(cabi_double, entry)
    monkeypatch.setattr(cabi_double, entry, lambda *a, **k: (calls.append(1), orig(*a, **k))[1])
    a = m4.generate(**enc, max_new_tokens=10, ignore_eos=True)
    assert len(calls) == 4 * cfg.num_hidden_layers * 9          # every projection of every decode step (9 steps after the prefill token)
    # the dense weights of the W4 model are the dequantised values the kernel uses: decoding through them gives the same tokens
    m4.w4, m4._steps = None, {}
    b = m4.generate(**enc, max_new_tokens=10, ignore_eos=True)
    assert torch.equal(a, b)


def test_act_order_checkpoint_keeps_the_dense_weights(cabi_double, tmp_path):
    from chatts_b200.model import ChatTSForCausalLM
    cfg, sd, _, proc = _build(cabi_double)
    path = _gptq_checkpoint(tmp_path, cfg, sd, act_order=True)
    m = ChatTSForCausalLM.from_pretrained(path, device="cpu", torch_dtype="bfloat16", max_batch=2, max_seq_len=256, page_size=16, use_cuda_graph=False)
    assert m.w4 is None


def test_attach_w4_rejects_tensor_parallel_models(cabi_double):
    cfg, sd, model, proc = _build(cabi_double)
    model.tp_size = 2
    with pytest.raises(ValueError):
        model.attach_w4({}, 128)


def test_fragment_major_repack_round_trips(cabi_double):
    """weights.py:repack_w4_mma against the independent inverse of tests/cabi_double.py (the layout include/chatts_b200.h states for
    cts_gemm_w4f_args): the decoded dense weight equals dequantize_w4 of the row layout, for a feature count that needs padding."""
    from chatts_b200.weights import dequantize_w4, repack_w4_mma
    g = torch.Generator().manual_seed(11)
    for dt in (torch.bfloat16, torch.float16):
        for n, k, gs in ((200, 256, 64), (512, 384, 128)):
            qw = torch.randint(0, 256, (n, k // 2), generator=g, dtype=torch.uint8)
            sc = ((torch.rand(n, k // gs, generator=g) + 0.5) * 0.01).to(dt)
            zp = torch.randint(0, 17, (n, k // gs), generator=g, dtype=torch.uint8)
            qwf, szp = repack_w4_mma(qw, sc, zp, gs)
            tiles = -(-n // 256)
            assert qwf.shape == (tiles * (k // 64) * 8192,) and szp.shape == (tiles, k // gs, 256) and szp.dtype == torch.int32
            x = torch.eye(k, dtype=dt)[:32]                               # the first 32 unit vectors: out[t] = column t of W
            out = torch.zeros(1, 32, n)
            cabi_double.gemm_w4_mma(x, qwf, szp, n, gs, out, 1, t=32)
            want = dequantize_w4(qw, sc, zp, gs).float()[:, :32].t()
            assert torch.equal(out[0], want)


def test_shapes_the_mma_kernel_cannot_take_fall_back_to_the_tcgen05_kernel(cabi_double, tmp_path, monkeypatch):
    """cts_gemm_w4_mma streams 128-K stages: a down_proj with 704 inputs (not a multiple of 128) makes attach_w4 choose cts_gemm_w4."""
    from chatts_b200.model import ChatTSForCausalLM
    monkeypatch.setenv("CTS_W4_KERNEL", "mma")
    cfg, sd, _, proc = _build(cabi_double)
    assert cfg.intermediate_size % 128 != 0
    path = _gptq_checkpoint(tmp_path, cfg, sd)
    m = ChatTSForCausalLM.from_pretrained(path, device="cpu", torch_dtype="bfloat16", max_batch=2, max_seq_len=256, page_size=16, use_cuda_graph=False)
    assert m.w4 is not None and m.w4["kernel"] == "tc5"
