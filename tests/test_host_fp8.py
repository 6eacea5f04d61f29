"""FP8 weights (ChatTSForCausalLM.quantize_fp8) on CPU: the quantizer (per-row scale, round-to-nearest-even codes, zero rows, non-finite
weights, fusing commutes with quantising), the fragment-major layout, the model's routing through the C-ABI double (decode-sized steps
stream the codes through gemm_fp8, every other step dequantises each projection just before its gemm), the refusals, the vLLM / server
surfaces, and the tensor-parallel scales over two gloo ranks."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from chatts_b200 import ChatTSConfig
from chatts_b200.weights import dequantize_fp8, pack_fp8_mma, quantize_fp8_rows, synthetic_state_dict, unpack_fp8_mma
from tests.fp8_double import Fp8Double
from tests.test_host_model import _build, _series

PROMPTS = ["A <ts><ts/> and B <ts><ts/> ?", "Only text, no series, but a longer prompt to left-pad the other one"]


@pytest.fixture
def cabi_double(cabi_double, monkeypatch):
    """The C-ABI double of tests/conftest.py with the FP8 entry points (tests/fp8_double.py)."""
    from chatts_b200 import _cabi
    dbl = Fp8Double()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: dbl)
    return dbl


def _e4m3_values():
    """Value of each of the 256 e4m3fn codes from the format's definition (1 sign, 4 exponent bits with bias 7, 3 mantissa bits; no
    infinities, S.1111.111 = NaN), independent of torch's float8 type."""
    v = np.full(256, np.nan)
    for c in range(256):
        s, e, m = c >> 7, (c >> 3) & 15, c & 7
        if e == 15 and m == 7:
            continue
        mag = (m / 8.0) * 2.0 ** -6 if e == 0 else (1 + m / 8.0) * 2.0 ** (e - 7)
        v[c] = -mag if s else mag
    return v


def _rne_codes(x):
    """Round-to-nearest-even onto the e4m3 grid (ties to the code with an even mantissa), by exhaustive search."""
    vals = _e4m3_values()
    fin = np.array([c for c in range(256) if np.isfinite(vals[c]) and c != 0x80])        # +0 stands for both zeros
    out = np.empty(x.shape, dtype=np.uint8)
    for i, xv in np.ndenumerate(x):
        d = np.abs(vals[fin] - xv)
        best = fin[d == d.min()]
        if len(best) > 1:
            best = best[(best & 1) == 0]
        c = int(best[0])
        out[i] = 0x80 if (c == 0 and np.signbit(xv)) else c
    return out


def test_quantizer_scale_codes_and_special_rows():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(6, 96, generator=g) * 0.05).to(torch.bfloat16)
    w[2] = 0                                                   # an all-zero row
    w[4, 7] = -0.3                                             # the row maximum is a negative entry
    q, s = quantize_fp8_rows(w)
    assert q.dtype == torch.uint8 and s.dtype == torch.float32 and q.shape == w.shape
    amax = w.float().abs().amax(1)
    assert torch.equal(s[[0, 1, 3, 4, 5]], amax[[0, 1, 3, 4, 5]] / 448.0)
    assert torch.isfinite(s).all() and s[2] > 0 and bool((q[2] == 0).all())
    assert int(q[4, 7]) == 0xFE                                 # -448: the row maximum maps onto the largest code
    want = _rne_codes((w.float() / s[:, None]).numpy().astype(np.float64))
    assert np.array_equal(q.numpy(), want)
    w16 = dequantize_fp8(q, s, torch.float32)
    assert not torch.isnan(w16).any() and float((w16 - w.float()).abs().max()) <= float(s.max()) * 16   # half an ulp of 448 is 16
    # ties go to even: 1.0625 lies halfway between the codes of 1.0 (0x38) and 1.125 (0x39)
    t = torch.tensor([[448.0, 1.0625, -1.0625, 0.0]])
    assert quantize_fp8_rows(t)[0].tolist() == [[0x7E, 0x38, 0xB8, 0x00]]


def test_quantizer_rejects_non_finite_weights_naming_the_tensor():
    w = torch.ones(4, 64)
    w[1, 3] = float("inf")
    with pytest.raises(ValueError, match="layers.3.mlp.up_proj"):
        quantize_fp8_rows(w, name="model.layers.3.mlp.up_proj.weight")


def test_quantising_then_fusing_equals_fusing_then_quantising():
    g = torch.Generator().manual_seed(1)
    q_, k_, v_ = (torch.randn(n, 128, generator=g).to(torch.bfloat16) for n in (256, 128, 128))
    gate, up = (torch.randn(192, 128, generator=g).to(torch.bfloat16) for _ in range(2))
    il = lambda a, b: torch.stack([a.view(-1, 64, a.shape[1]), b.view(-1, 64, b.shape[1])], 1).reshape(2 * a.shape[0], a.shape[1])
    fq, fs = quantize_fp8_rows(torch.cat([q_, k_, v_]))
    parts = [quantize_fp8_rows(t) for t in (q_, k_, v_)]
    assert torch.equal(fq, torch.cat([p[0] for p in parts])) and torch.equal(fs, torch.cat([p[1] for p in parts]))
    gq, gs = quantize_fp8_rows(il(gate, up))
    (aq, as_), (bq, bs) = quantize_fp8_rows(gate), quantize_fp8_rows(up)
    assert torch.equal(gq, il(aq, bq)) and torch.equal(gs, il(as_[:, None], bs[:, None])[:, 0])


def test_fragment_major_pack_round_trips(cabi_double):
    """pack_fp8_mma against its inverse AND against the independent decoding of the double (the layout include/chatts_b200.h states
    for cts_gemm_fp8_args), for a feature count that needs padding."""
    g = torch.Generator().manual_seed(2)
    for n, k in ((200, 128), (512, 704), (300, 64)):
        codes = torch.randint(0, 256, (n, k), generator=g, dtype=torch.uint8)
        codes[(codes == 0x7F) | (codes == 0xFF)] = 1
        s = torch.rand(n, generator=g) + 0.5
        packed = pack_fp8_mma(codes)
        assert packed.shape == (-(-n // 256) * (k // 64) * 16384,)
        assert torch.equal(unpack_fp8_mma(packed, n, k), codes)
        out = torch.zeros(n, k, dtype=torch.bfloat16)
        cabi_double.fp8_dequant(packed, s, k, out)
        assert torch.equal(out, dequantize_fp8(codes, s, torch.bfloat16))


def _w_prime_state_dict(sd, dtype):
    out = dict(sd)
    for name, w in sd.items():
        if ".layers." in name and name.endswith("_proj.weight"):
            out[name] = dequantize_fp8(*quantize_fp8_rows(w), dtype)
    return out


def _log_calls(monkeypatch, dbl, names):
    log = []
    for nm in names:
        orig = getattr(dbl, nm)

        def wrap(*a, _o=orig, _n=nm, **k):
            log.append((_n, a, k))
            return _o(*a, **k)
        monkeypatch.setattr(dbl, nm, wrap)
    return log


@pytest.mark.parametrize("qwen3", [False, True])
def test_model_routes_decode_through_gemm_fp8_and_prefill_through_dequant(cabi_double, monkeypatch, qwen3):
    from chatts_b200.model import ChatTSForCausalLM
    cfg, sd, model, proc = _build(cabi_double, qwen3=qwen3)
    model.next_prefetch_bytes = 1 << 20                        # an L2 hint must not name a freed weight
    assert model.quantize_fp8() is model
    assert all(w is None for ws in (model.wqkv, model.wo, model.wgu, model.wd) for w in ws)
    assert model.embed.dtype == model.lm_head.dtype == model.ln1[0].dtype == model.kv.dtype == torch.bfloat16
    assert model.fp8["scratch"].numel() == 2 * model.I * model.H
    enc = proc(text=PROMPTS, timeseries=list(_series()), padding=True, return_tensors="pt")
    log = _log_calls(monkeypatch, cabi_double, ("gemm", "gemm_fp8", "fp8_dequant"))
    # prefill (forward): every projection dequantised into the scratch matrix right before the gemm that reads it
    lg = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits
    deq = [i for i, e in enumerate(log) if e[0] == "fp8_dequant"]
    assert len(deq) == 4 * cfg.num_hidden_layers and not any(e[0] == "gemm_fp8" for e in log)
    scratch = model.fp8["scratch"].data_ptr()
    for i in deq:
        assert log[i + 1][0] == "gemm" and log[i + 1][1][1].data_ptr() == scratch
    # the prefill computes exactly what the 16-bit model computes on the dequantised weights W'
    ref = ChatTSForCausalLM(cfg, _w_prime_state_dict(sd, torch.bfloat16), device="cpu", dtype=torch.bfloat16, max_batch=8, max_seq_len=512,
                            page_size=16, use_cuda_graph=False)
    assert torch.equal(lg, ref.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits)
    # generate: one prefill (dequant + gemm) and 9 decode steps through gemm_fp8 for all four projections
    log.clear()
    a = model.generate(**enc, max_new_tokens=10, ignore_eos=True)
    assert sum(e[0] == "gemm_fp8" for e in log) == 4 * cfg.num_hidden_layers * 9
    assert sum(e[0] == "fp8_dequant" for e in log) == 4 * cfg.num_hidden_layers
    assert all(e[2].get("next_w") is None for e in log if e[0] == "gemm")
    b = ref.generate(**enc, max_new_tokens=10, ignore_eos=True)
    S = enc["input_ids"].shape[1]
    assert torch.equal(a[:, :S + 1], b[:, :S + 1])           # the prefill's token; decode sums in another order (fp32 W' vs 16-bit W')


def test_fused_chain_and_native_decode_variants_do_not_engage(cabi_double, monkeypatch):
    cfg, sd, model, proc = _build(cabi_double, use_fused_decode=1, use_chain=True, use_native_step=True)
    model.quantize_fp8()
    assert not model._chain_ok(2) and not model._native_ok(2)
    for nm in ("gemm_decode_fused", "decoder_step"):
        monkeypatch.setattr(cabi_double, nm, lambda *a, **k: pytest.fail("a 16-bit decode variant ran on an FP8 model"))
    log = _log_calls(monkeypatch, cabi_double, ("gemm_fp8",))
    enc = proc(text=PROMPTS, timeseries=list(_series()), padding=True, return_tensors="pt")
    model.generate(**enc, max_new_tokens=4, ignore_eos=True)
    assert len(log) == 4 * cfg.num_hidden_layers * 3


def test_refusals(cabi_double, tmp_path):
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.train import LoraTrainer
    cfg, sd, model, proc = _build(cabi_double)
    # shapes the kernels cannot take, and non-finite weights: refused before anything is freed
    wo = model.wo
    model.wo = [w[:, :200].contiguous() for w in wo]
    with pytest.raises(ValueError, match="multiple of 64"):
        model.quantize_fp8()
    model.wo = wo
    model.wd[1][3, 5] = float("nan")
    with pytest.raises(ValueError, match=r"model\.layers\.1\.mlp\.down_proj\.weight"):
        model.quantize_fp8()
    assert model.fp8 is None and all(w is not None for w in model.wqkv + model.wo + model.wgu + model.wd)
    model.wd[1][3, 5] = 0
    model.quantize_fp8()
    with pytest.raises(ValueError, match="already"):
        model.quantize_fp8()
    with pytest.raises(ValueError):
        model.attach_w4({}, 128)
    with pytest.raises(ValueError):
        model.quantize_w4_synthetic()
    with pytest.raises(ValueError, match="quantize_fp8"):
        model.merge_lora({"model.layers.0.self_attn.q_proj.lora_A.weight": torch.zeros(2, cfg.hidden_size),
                          "model.layers.0.self_attn.q_proj.lora_B.weight": torch.zeros(cfg.hidden_size, 2)})
    with pytest.raises(ValueError, match="FP8"):
        LoraTrainer(model)
    with pytest.raises(ValueError, match="int3"):
        ChatTSForCausalLM.from_synthetic(cfg, device="cpu", quantization="int3")
    # a GPTQ checkpoint is already quantised
    from tests.test_host_w4 import _gptq_checkpoint
    path = _gptq_checkpoint(tmp_path, cfg, sd)
    with pytest.raises(ValueError, match="GPTQ"):
        ChatTSForCausalLM.from_pretrained(path, device="cpu", torch_dtype="bfloat16", max_batch=2, max_seq_len=256, page_size=16,
                                          use_cuda_graph=False, quantization="fp8")


def test_from_pretrained_and_the_vllm_and_server_surfaces(cabi_double, tmp_path):
    import json
    from safetensors.torch import save_file
    from chatts_b200 import server, vllm_compat
    from chatts_b200.model import ChatTSForCausalLM
    cfg, sd, model, proc = _build(cabi_double)
    d = tmp_path / "ckpt"
    d.mkdir()
    json.dump(cfg.to_dict(), open(d / "config.json", "w"))
    save_file({k: v.contiguous() for k, v in sd.items()}, str(d / "model.safetensors"))
    kw = dict(device="cpu", torch_dtype="bfloat16", max_batch=4, max_seq_len=256, page_size=16, use_cuda_graph=False)
    m = ChatTSForCausalLM.from_pretrained(str(d), quantization="fp8", **kw)
    assert m.fp8 is not None and m.wqkv[0] is None
    assert ChatTSForCausalLM.from_pretrained(str(d), **kw).fp8 is None
    llm = vllm_compat.LLM(model=model, quantization="fp8")
    assert llm.model is model and model.fp8 is not None and len(model.fp8["d"]) == cfg.num_hidden_layers
    out = llm.generate({"prompt": "A <ts><ts/> ?", "multi_modal_data": {"timeseries": [_series()[0]]}},
                       vllm_compat.SamplingParams(max_tokens=3, temperature=0.0))
    assert len(out) == 1
    with pytest.raises(ValueError, match="int3"):
        vllm_compat.LLM(model=model, quantization="int3")
    assert server.parse_args(["--quantization", "fp8"]).quantization == "fp8"
    assert server.parse_args([]).quantization is None
    with pytest.raises(SystemExit):
        server.parse_args(["--quantization", "int3"])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _tp_worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from chatts_b200 import _cabi
    from chatts_b200.model import ChatTSForCausalLM
    dbl = Fp8Double()
    _cabi.get_context = lambda device=None: dbl
    torch.cuda.is_available = lambda: True
    torch.cuda.current_device = lambda: 0
    cfg = ChatTSConfig.tiny(num_attention_heads=8, num_key_value_heads=4, hidden_size=256, intermediate_size=1024)
    sd = synthetic_state_dict(cfg, seed=4, device="cpu", dtype=torch.bfloat16, std=0.05)
    sd["model.layers.1.mlp.down_proj.weight"][7, 900] = 0.9          # the row maximum of rank 1's slice: rank 0 must take it too
    kw = dict(device="cpu", dtype=torch.bfloat16, max_batch=2, max_seq_len=128, page_size=16, use_cuda_graph=False, use_peer_allreduce=False)
    one = ChatTSForCausalLM(cfg, sd, **kw).quantize_fp8()
    tp = ChatTSForCausalLM(cfg, sd, tp_rank=rank, tp_size=world, **kw).quantize_fp8()
    H, I, d = cfg.hidden_size, cfg.intermediate_size, cfg.head_dim
    nh, nkv = cfg.num_attention_heads // world, cfg.num_key_value_heads // world
    for l in range(cfg.num_hidden_layers):
        for kind, n, k in (("qkv", (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * d, H), ("o", H, cfg.num_attention_heads * d),
                           ("gu", 2 * I, H), ("d", H, I)):
            full_q, full_s, _ = one.fp8[kind][l]
            loc_q, loc_s, loc_k = tp.fp8[kind][l]
            fq, lq = unpack_fp8_mma(full_q, n, k), unpack_fp8_mma(loc_q, loc_s.shape[0], loc_k)
            if kind == "qkv":
                rows = torch.cat([torch.arange(rank * nh * d, (rank + 1) * nh * d)] +
                                 [off + torch.arange(rank * nkv * d, (rank + 1) * nkv * d) for off in
                                  (cfg.num_attention_heads * d, (cfg.num_attention_heads + cfg.num_key_value_heads) * d)])
                assert torch.equal(lq, fq[rows]) and torch.equal(loc_s, full_s[rows])
            elif kind == "gu":                                  # interleaved per 64 rows: rank r owns a contiguous block of 128-row tiles
                per = 2 * I // world
                assert torch.equal(lq, fq[rank * per:(rank + 1) * per]) and torch.equal(loc_s, full_s[rank * per:(rank + 1) * per])
            else:                                               # row-parallel: a K-slice of every row, the scale of the full row
                per = k // world
                assert torch.equal(lq, fq[:, rank * per:(rank + 1) * per]) and torch.equal(loc_s, full_s)
    ret[rank] = True
    dist.destroy_process_group()


def test_tensor_parallel_codes_and_scales_are_slices_of_the_single_gpu_result():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_tp_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert all(ret.get(r) for r in range(world))
