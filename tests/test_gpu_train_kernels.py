"""Kernels of the LoRA fine-tune step (row A9): the small-N / small-K LoRA GEMM shapes, SwiGLU forward/backward, RMSNorm backward,
RoPE(+q/k-norm) backward, fused cross entropy, row gather and the LoRA weight-gradient kernel -- through the C-ABI against
the torch restatement of every entry point (tests/cabi_double.py, fp32 on the CPU, itself checked against oracle/lora.py by
tests/test_host_train.py).  The parts of the training path still waiting for their first GPU run live in
tests/test_gpu_zz_c_train.py."""
import math

import numpy as np
import pytest
import torch

from tests.cabi_double import TorchDouble
from tests.gpu_util import ctx, record, rel_err

DT = torch.bfloat16
DBL = TorchDouble()


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rn(g, *shape, std=1.0, dtype=DT):
    return (torch.randn(*shape, generator=g) * std).to(dtype)


pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ small-N / small-K GEMMs
@pytest.mark.parametrize("t,n,k", [(300, 24, 256), (300, 256, 24), (64, 8, 704), (513, 16, 136), (40, 48, 512), (1000, 704, 8),
                                   (129, 1408, 16), (7, 24, 256)])
def test_gemm_lora_shapes(t, n, k):
    """The LoRA down/up products: N = fused rank (8..48) and K = fused rank -- box larger than the tensor on one side."""
    c = ctx()
    g = _g(t + n + k)
    x, w = _rn(g, t, k, std=0.5), _rn(g, n, k, std=0.1)
    res = _rn(g, t, n, std=0.3)
    out = torch.full((t, n), float("nan"), device="cuda", dtype=DT)
    c.gemm(x.cuda(), w.cuda(), out)
    ref = (x.float() @ w.float().T).to(DT)
    e0 = rel_err(out, ref)
    h = res.cuda().clone()
    c.gemm(x.cuda(), w.cuda(), h, residual=h, epilogue=4)
    torch.cuda.synchronize()
    ref2 = (res.float() + ref.float()).to(DT)
    e1 = rel_err(h, ref2)
    record("gemm_lora_shape", t=t, n=n, k=k, err=e0, err_residual=e1)
    assert torch.isfinite(out.float()).all() and e0 < 8e-3 and e1 <= 2 ** -7 + 1e-6


# ------------------------------------------------------------------------------------------------ elementwise backward
@pytest.mark.parametrize("t,inter,il", [(5, 704, True), (300, 128, True), (33, 704, False), (2, 8, False)])
def test_swiglu_fwd_bwd(t, inter, il):
    c = ctx()
    g = _g(t + inter)
    gu, dact = _rn(g, t, 2 * inter), _rn(g, t, inter)
    out, dgu = torch.empty(t, inter, device="cuda", dtype=DT), torch.empty(t, 2 * inter, device="cuda", dtype=DT)
    c.swiglu(gu.cuda(), t, inter, out, interleaved=il)
    c.swiglu_bwd(gu.cuda(), dact.cuda(), t, inter, dgu, interleaved=il)
    torch.cuda.synchronize()
    ro, rd = torch.empty(t, inter, dtype=DT), torch.empty(t, 2 * inter, dtype=DT)
    DBL.swiglu(gu, t, inter, ro, interleaved=il)
    DBL.swiglu_bwd(gu, dact, t, inter, rd, interleaved=il)
    assert rel_err(out, ro) <= 2 ** -7 + 1e-6 and rel_err(dgu, rd) < 1e-2


@pytest.mark.parametrize("t,h", [(3, 256), (70, 4096), (5, 5120)])
def test_rmsnorm_bwd(t, h):
    c = ctx()
    g = _g(t + h)
    dy, x, w, dres = _rn(g, t, h), _rn(g, t, h, std=2.0), (torch.rand(h, generator=g) + 0.5).to(DT), _rn(g, t, h)
    ref = torch.empty(t, h, dtype=DT)
    DBL.rmsnorm_bwd(dy, x, w, 1e-6, dres, ref)
    out = torch.empty(t, h, device="cuda", dtype=DT)
    c.rmsnorm_bwd(dy.cuda(), x.cuda(), w.cuda(), 1e-6, dres.cuda(), out)
    e = rel_err(out, ref)
    ref0 = torch.empty(t, h, dtype=DT)
    DBL.rmsnorm_bwd(dy, x, w, 1e-6, None, ref0)
    inpl = dy.cuda().clone()
    c.rmsnorm_bwd(inpl, x.cuda(), w.cuda(), 1e-6, None, inpl)            # dx_out aliases dy
    acc = dres.cuda().clone()
    c.rmsnorm_bwd(dy.cuda(), x.cuda(), w.cuda(), 1e-6, acc, acc)          # dx_out aliases dres_in (the trainer's use)
    torch.cuda.synchronize()
    record("rmsnorm_bwd", t=t, h=h, err=e)
    assert e < 1e-2 and rel_err(inpl, ref0) < 1e-2 and torch.equal(acc, out)


@pytest.mark.parametrize("d,nh,nkv,qk", [(64, 4, 2, False), (64, 4, 2, True), (128, 8, 2, True), (128, 5, 1, False)])
def test_qkv_rope_bwd(d, nh, nkv, qk):
    c = ctx()
    t = 37
    g = _g(d + nh)
    W = (nh + 2 * nkv) * d
    qkv, dq, dk, dv = _rn(g, t, W), _rn(g, t, nh * d), _rn(g, t, nkv * d), _rn(g, t, nkv * d)
    pos = torch.randint(0, 200, (t,), generator=g).to(torch.int32)
    ang = torch.rand(256, d // 2, generator=g) * 6.28
    cos, sin = ang.cos().to(DT), ang.sin().to(DT)
    qn = (torch.rand(d, generator=g) + 0.5).to(DT) if qk else None
    kn = (torch.rand(d, generator=g) + 0.5).to(DT) if qk else None
    ref = torch.empty(t, W, dtype=DT)
    DBL.qkv_rope_bwd(dq, dk, dv, qkv, pos, cos, sin, qn, kn, 1e-6, ref, t, nh, nkv, d)
    out = torch.full((t, W), float("nan"), device="cuda", dtype=DT)
    cu = lambda a: None if a is None else a.cuda()
    c.qkv_rope_bwd(dq.cuda(), dk.cuda(), dv.cuda(), qkv.cuda(), pos.cuda(), cos.cuda(), sin.cuda(), cu(qn), cu(kn), 1e-6, out, t, nh, nkv, d)
    torch.cuda.synchronize()
    e = rel_err(out, ref)
    record("qkv_rope_bwd", d=d, qk=qk, err=e)
    assert torch.isfinite(out.float()).all() and e < 1e-2


@pytest.mark.parametrize("n,vocab", [(1, 1000), (9, 1000), (3, 151936)])
def test_cross_entropy_fwd_bwd(n, vocab):
    c = ctx()
    g = _g(n + vocab)
    logits = _rn(g, n, vocab, std=3.0)
    tgt = torch.randint(0, vocab, (n,), generator=g).to(torch.int32)
    ref_l, ref_rows, ref_out = logits.clone(), torch.zeros(n), torch.full((1,), 0.25)
    DBL.ce_loss_grad(ref_l, tgt, n, 1.0 / 7, ref_rows, ref_out, accumulate=True)
    lg = logits.clone().cuda()
    rows, out = torch.zeros(n, device="cuda"), torch.full((1,), 0.25, device="cuda")
    c.ce_loss_grad(lg, tgt.cuda(), n, 1.0 / 7, rows, out, accumulate=True)
    torch.cuda.synchronize()
    e = rel_err(lg, ref_l)
    record("ce_loss_grad", n=n, vocab=vocab, err=e, loss=float(out[0]))
    assert torch.allclose(rows.cpu(), ref_rows, atol=1e-4, rtol=1e-5) and abs(float(out[0]) - float(ref_out[0])) < 1e-4 * abs(float(ref_out[0]))
    assert e < 1e-2
    out2 = torch.full((1,), 5.0, device="cuda")
    c.ce_loss_grad(logits.clone().cuda(), tgt.cuda(), n, 1.0 / 7, rows, out2, accumulate=False)
    assert abs(float(out2[0]) - (float(ref_out[0]) - 0.25)) < 1e-4 * abs(float(ref_out[0]))


def test_gather_rows_and_zero_fill():
    c = ctx()
    g = _g(0)
    src = _rn(g, 50, 256)
    idx = torch.tensor([3, -1, 49, 0, -1, 7], dtype=torch.int32)
    out = torch.full((6, 256), float("nan"), device="cuda", dtype=DT)
    c.gather_rows(src.cuda(), idx.cuda(), 6, out)
    ref = torch.empty(6, 256, dtype=DT)
    DBL.gather_rows(src, idx, 6, ref)
    assert torch.equal(out.cpu(), ref)


# ------------------------------------------------------------------------------------------------ LoRA weight gradient
@pytest.mark.parametrize("t,m,r,il", [(37, 256, 8, 0), (5000, 704, 16, 0), (300, 128, 4, 1), (300, 128, 16, 2), (9000, 64, 16, 0),
                                      (100, 4096, 16, 0)])
def test_lora_wgrad(t, m, r, il):
    c = ctx()
    g = _g(t + m + r)
    ld = 2 * m if il else m + 64
    col0 = 0 if il else 32
    p, q = _rn(g, t, ld, std=0.5), _rn(g, t, 3 * r + 8, std=0.5)
    # dB layout [m, r] and dA layout [r, m], each accumulated on top of existing content
    for so_m, so_r, name in ((r, 1, "dB"), (1, m, "dA")):
        base = torch.randn(m * r, generator=g)
        ref = base.clone()
        DBL.lora_wgrad(p, col0, il, m, q, r, r, t, 0.5, ref, so_m, so_r)
        out = base.cuda()
        c.lora_wgrad(p.cuda(), col0, il, m, q.cuda(), r, r, t, 0.5, out, so_m, so_r)
        torch.cuda.synchronize()
        e = rel_err(out, ref)
        record("lora_wgrad", t=t, m=m, r=r, il=il, layout=name, err=e)
        assert e < 2e-4, (name, e)                  # fp32 accumulation of exact bf16 products: only the summation order differs
