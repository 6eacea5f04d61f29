"""cts_gemm_decode_fused (csrc/gemm_decode_fused.cu: the K splits of a tile reduce over distributed shared memory inside one
cluster and apply the projection's tail) against the two-launch path it replaces -- cts_gemm(CTS_EPI_PARTIAL_F32) + cts_reduce_* /
cts_qkv_rope_cache -- which must be reproduced BIT FOR BIT (same summation order), and through generate().
Plain tests (no xfail markers)."""
import numpy as np
import pytest
import torch

from tests.gpu_util import ctx, record

pytestmark = pytest.mark.gpu
DT = torch.bfloat16
EPI_PARTIAL = 3


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rn(g, *shape, std=1.0, dtype=DT):
    return (torch.randn(*shape, generator=g) * std).to(dtype).cuda()


@pytest.mark.parametrize("t,n,k,s", [(1, 256, 512, 2), (8, 5120, 5120, 7), (32, 5120, 13824, 7), (17, 384, 1024, 8), (32, 200, 640, 3)])
def test_fused_residual(t, n, k, s):
    c = ctx()
    g = _g(t + n + k)
    x, w, h0 = _rn(g, t, k, std=0.5), _rn(g, n, k, std=0.05), _rn(g, t, n, std=0.5)
    ws = torch.empty(s * t * n, device="cuda", dtype=torch.float32)
    c.gemm(x, w, ws, epilogue=EPI_PARTIAL, split_k=s, t=t)
    ref = h0.clone()
    c.reduce_residual_rmsnorm(ws, s, ref, ref, None, 1e-6, None, t=t)
    out = h0.clone()
    c.gemm_decode_fused(x, w, 0, s, t, h=out)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("t,inter,k,s", [(1, 128, 256, 1), (8, 13824, 5120, 2), (32, 704, 512, 4)])
def test_fused_swiglu(t, inter, k, s):
    c = ctx()
    g = _g(t + inter)
    x, w = _rn(g, t, k, std=0.5), _rn(g, 2 * inter, k, std=0.05)
    ws = torch.empty(s * t * 2 * inter, device="cuda", dtype=torch.float32)
    c.gemm(x, w, ws, epilogue=EPI_PARTIAL, split_k=s, t=t)
    ref = torch.empty(t, inter, device="cuda", dtype=DT)
    c.reduce_swiglu(ws, s, t, inter, ref, interleaved=True)
    out = torch.full((t, inter), float("nan"), device="cuda", dtype=DT)
    c.gemm_decode_fused(x, w, 1, s, t, act=out)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("d,nh,nkv,qk,bias", [(128, 40, 8, False, True), (128, 8, 2, True, False), (64, 4, 2, False, True), (64, 5, 1, True, False)])
@pytest.mark.parametrize("t,s", [(1, 5), (32, 3)])
def test_fused_qkv_rope(d, nh, nkv, qk, bias, t, s):
    c = ctx()
    g = _g(d + nh + t)
    H, page, pages = 1024, 16, 8
    N = (nh + 2 * nkv) * d
    x, w = _rn(g, t, H, std=0.5), _rn(g, N, H, std=0.05)
    b = _rn(g, N, std=0.2) if bias else None
    qn = (torch.rand(d, generator=g) + 0.5).to(DT).cuda() if qk else None
    kn = (torch.rand(d, generator=g) + 0.5).to(DT).cuda() if qk else None
    pos = torch.randint(0, 100, (t,), generator=g).to(torch.int32).cuda()
    ang = torch.rand(128, d // 2, generator=g) * 6.28
    cos, sin = ang.cos().to(DT).cuda(), ang.sin().to(DT).cuda()
    slot = torch.randperm(pages * page, generator=g)[:t].to(torch.int32)
    if t > 2:
        slot[1] = -1
    slot = slot.cuda()
    outs = []
    for fused in (False, True):
        q = torch.full((t, nh * d), float("nan"), device="cuda", dtype=DT)
        kc = torch.zeros(pages, nkv, page, d, device="cuda", dtype=DT)
        vc = torch.zeros(pages, nkv, page, d, device="cuda", dtype=DT)
        if fused:
            c.gemm_decode_fused(x, w, 2, s, t, bias=b, positions=pos, cos=cos, sin=sin, slot_map=slot, q_out=q, k_cache=kc, v_cache=vc,
                                q_norm=qn, k_norm=kn, eps=1e-6, nh=nh, nkv=nkv, head_dim=d, page_size=page)
        else:
            ws = torch.empty(s * t * N, device="cuda", dtype=torch.float32)
            c.gemm(x, w, ws, epilogue=EPI_PARTIAL, split_k=s, t=t)
            c.qkv_rope_cache(ws, True, s, b, pos, cos, sin, slot, q, kc, vc, None, None, t, nh, nkv, d, page, qn, kn, 1e-6)
        torch.cuda.synchronize()
        outs.append((q, kc, vc))
    if qk:      # the per-head statistic is summed in a different (still fixed) order: one bf16 ulp at most
        for a, r in zip(outs[1], outs[0]):
            assert float((a.float() - r.float()).abs().max()) <= 2 ** -7 * float(r.float().abs().max()) + 1e-6
    else:
        assert all(torch.equal(a, r) for a, r in zip(outs[1], outs[0]))


@pytest.mark.parametrize("qwen3,graph", [(False, True), (True, False)])
def test_generate_with_fused_decode_gemms(qwen3, graph):
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig.tiny()
    if qwen3:
        cfg.qk_norm, cfg.attention_bias = True, False
    sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=DT, std=0.05)
    kw = dict(dtype=DT, max_batch=4, max_seq_len=256, page_size=16, use_cuda_graph=graph)
    ref, fused = ChatTSForCausalLM(cfg, sd, **kw), ChatTSForCausalLM(cfg, sd, use_fused_decode=True, **kw)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    x = np.arange(256)
    enc = proc(text=["A <ts><ts/> ?", "text only, a longer prompt to pad the first one"], timeseries=[np.sin(x / 9) * 4], return_tensors="pt")
    a = ref.generate(**enc, max_new_tokens=24, ignore_eos=True)
    b = fused.generate(**enc, max_new_tokens=24, ignore_eos=True)
    record("fused_decode_generate", qwen3=qwen3, equal=bool(torch.equal(a, b)))
    if not qwen3:
        assert torch.equal(a, b)
    else:       # q/k-norm statistic order differs by an ulp: identical prefix expected, full equality not guaranteed
        assert torch.equal(a[:, : enc["input_ids"].shape[1] + 4], b[:, : enc["input_ids"].shape[1] + 4])


@pytest.mark.parametrize("t,n,k,s", [(8, 5120, 5120, 7), (32, 640, 1024, 3)])
def test_residual_emits_per_tile_sums_of_squares(t, n, k, s):
    c = ctx()
    g = _g(t + n)
    x, w, h0 = _rn(g, t, k, std=0.5), _rn(g, n, k, std=0.05), _rn(g, t, n, std=0.5)
    tiles = (n + 127) // 128
    out, ssq = h0.clone(), torch.full((t, tiles), float("nan"), device="cuda")
    c.gemm_decode_fused(x, w, 0, s, t, h=out, ssq_out=ssq)
    ref = h0.clone()
    c.gemm_decode_fused(x, w, 0, s, t, h=ref)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    want = torch.nn.functional.pad(out.float(), (0, tiles * 128 - n)).view(t, tiles, 128).pow(2).sum(-1)
    assert torch.allclose(ssq, want, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("mode,t,s", [(1, 8, 2), (2, 32, 5), (1, 32, 3)])
def test_rmsnorm_fused_into_the_token_operand(mode, t, s):
    """norm_h / norm_w / ssq_in: the kernel builds xn = w * dtype(h * rstd) itself -- against the RMSNorm launch + the same fused GEMM."""
    c = ctx()
    g = _g(mode * 100 + t)
    H, inter, d, nh, nkv, page = 1024, 704, 128, 4, 2, 16
    h = _rn(g, t, H, std=1.5)
    nw = (torch.rand(H, generator=g) + 0.5).to(DT).cuda()
    tiles = H // 128
    ssq = h.float().view(t, tiles, 128).pow(2).sum(-1).contiguous()
    xn = torch.empty_like(h)
    c.reduce_residual_rmsnorm(None, 0, h, None, nw, 1e-6, xn, t=t)
    if mode == 1:
        w = _rn(g, 2 * inter, H, std=0.05)
        a, b = torch.empty(t, inter, device="cuda", dtype=DT), torch.empty(t, inter, device="cuda", dtype=DT)
        c.gemm_decode_fused(xn, w, 1, s, t, act=a)
        c.gemm_decode_fused(None, w, 1, s, t, act=b, norm_h=h, norm_w=nw, ssq_in=ssq, norm_eps=1e-6)
        pairs = [(a, b)]
    else:
        N = (nh + 2 * nkv) * d
        w, bias = _rn(g, N, H, std=0.05), _rn(g, N, std=0.2)
        pos = torch.arange(t, dtype=torch.int32).cuda()
        ang = torch.rand(64, d // 2, generator=g) * 6.28
        cos, sin = ang.cos().to(DT).cuda(), ang.sin().to(DT).cuda()
        slot = torch.arange(t, dtype=torch.int32).cuda()
        outs = []
        for fused_norm in (False, True):
            q = torch.empty(t, nh * d, device="cuda", dtype=DT)
            kc, vc = torch.zeros(4, nkv, page, d, device="cuda", dtype=DT), torch.zeros(4, nkv, page, d, device="cuda", dtype=DT)
            kw = dict(bias=bias, positions=pos, cos=cos, sin=sin, slot_map=slot, q_out=q, k_cache=kc, v_cache=vc, eps=1e-6, nh=nh, nkv=nkv,
                      head_dim=d, page_size=page)
            if fused_norm:
                c.gemm_decode_fused(None, w, 2, s, t, norm_h=h, norm_w=nw, ssq_in=ssq, norm_eps=1e-6, **kw)
            else:
                c.gemm_decode_fused(xn, w, 2, s, t, **kw)
            outs.append((q, kc, vc))
        pairs = list(zip(outs[0], outs[1]))
    torch.cuda.synchronize()
    for a, b in pairs:      # the row statistic is summed tile by tile: rstd may move by an fp32 ulp -> at most one bf16 ulp in the output
        assert torch.isfinite(b.float()).all()
        assert float((a.float() - b.float()).abs().max()) <= 2 ** -7 * float(a.float().abs().max()) + 1e-6


def test_generate_with_five_stage_layers():
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig.tiny()
    sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=DT, std=0.05)
    kw = dict(dtype=DT, max_batch=4, max_seq_len=256, page_size=16, use_cuda_graph=True)
    ref, deep = ChatTSForCausalLM(cfg, sd, **kw), ChatTSForCausalLM(cfg, sd, use_fused_decode=2, **kw)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    x = np.arange(256)
    enc = proc(text=["A <ts><ts/> ?", "text only, a longer prompt to pad the first one"], timeseries=[np.sin(x / 9) * 4], return_tensors="pt")
    a = ref.generate(**enc, max_new_tokens=16, ignore_eos=True)
    b = deep.generate(**enc, max_new_tokens=16, ignore_eos=True)
    S = enc["input_ids"].shape[1]
    record("fused_decode_5stage_generate", equal=bool(torch.equal(a, b)), first_diff=int((a != b).float().argmax()) if not torch.equal(a, b) else -1)
    assert torch.equal(a[:, : S + 3], b[:, : S + 3])           # an ulp in a statistic may flip a near-tie later on; the start must agree
