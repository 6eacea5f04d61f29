"""wgmma GEMM through the C-ABI against fp32 torch on the CPU (same bf16/fp16 inputs)."""
import pytest
import torch

from tests.gpu_util import ctx, record, rel_err

pytestmark = pytest.mark.gpu
EPI_NONE, EPI_GELU, EPI_SWIGLU, EPI_PARTIAL, EPI_RESIDUAL = 0, 1, 2, 3, 4


def _mk(t, n, k, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(t, k, generator=g) * 0.5).to(dtype)
    w = (torch.randn(n, k, generator=g) * 0.1).to(dtype)
    b = (torch.randn(n, generator=g) * 0.2).to(dtype)
    return x, w, b


SHAPES = [(1, 128, 64), (1, 384, 512), (8, 384, 512), (32, 256, 1024), (5, 200, 272), (17, 130, 72),
          (64, 128, 128), (100, 384, 256), (128, 256, 512), (300, 256, 512), (513, 200, 136)]


@pytest.mark.parametrize("t,n,k", SHAPES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_gemm_bias(t, n, k, dtype):
    c = ctx()
    x, w, b = _mk(t, n, k, dtype, 1)
    ref = (x.float() @ w.float().T + b.float())
    out = torch.full((t, n), float("nan"), device="cuda", dtype=dtype)
    c.gemm(x.cuda(), w.cuda(), out, bias=b.cuda(), epilogue=EPI_NONE)
    torch.cuda.synchronize()
    e = rel_err(out, ref.to(dtype))
    record("gemm_bias", t=t, n=n, k=k, dtype=str(dtype), err=e)
    assert torch.isfinite(out.float()).all()
    assert e < 8e-3


@pytest.mark.parametrize("t,n,k,s", [(1, 384, 512, 4), (8, 256, 1024, 16), (32, 200, 2048, 5), (4, 130, 272, 3)])
def test_gemm_split_k_partial_and_reduce(t, n, k, s):
    c = ctx()
    dtype = torch.bfloat16
    x, w, b = _mk(t, n, k, dtype, 2)
    part = torch.full((s, t, n), float("nan"), device="cuda", dtype=torch.float32)
    c.gemm(x.cuda(), w.cuda(), part, epilogue=EPI_PARTIAL, split_k=s)
    torch.cuda.synchronize()
    ref = x.float() @ w.float().T
    got = part.sum(0).cpu()
    assert torch.isfinite(part).all()
    assert (got - ref).abs().max() / ref.abs().max() < 1e-5          # fp32 partials: only summation order differs
    out = torch.empty(t, n, device="cuda", dtype=dtype)
    c.reduce_bias_act(part, s, t, n, b.cuda(), EPI_GELU, out)
    torch.cuda.synchronize()
    ref2 = torch.nn.functional.gelu((ref + b.float()).to(dtype).float()).to(dtype)
    assert rel_err(out, ref2) < 8e-3


@pytest.mark.parametrize("t,n,k,s", [(1, 384, 512, 4), (8, 256, 1024, 16), (32, 200, 2048, 5), (4, 130, 272, 3), (32, 5120, 640, 3)])
def test_gemm_split_k_reduced_in_kernel(t, n, k, s):
    """CTS_EPI_SPLITK_F32: the last split of each tile sums the partials; twice, to check the counters reset; bit-identical runs."""
    c = ctx()
    x, w, _ = _mk(t, n, k, torch.bfloat16, 5)
    xd, wd = x.cuda(), w.cuda()
    ws = torch.empty(s * t * n, device="cuda", dtype=torch.float32)
    cnt = torch.zeros(1024, device="cuda", dtype=torch.int32)
    ref = x.float() @ w.float().T
    outs = []
    for _ in range(3):
        out = torch.full((t, n), float("nan"), device="cuda", dtype=torch.float32)
        c.gemm(xd, wd, out, epilogue=5, split_k=s, splitk_ws=ws, tile_counters=cnt)
        torch.cuda.synchronize()
        outs.append(out.cpu())
        assert (out.cpu() - ref).abs().max() / ref.abs().max() < 1e-5
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])       # deterministic summation order
    assert int(cnt.abs().sum()) == 0


@pytest.mark.parametrize("t", [1, 8, 40, 200])
def test_gemm_gelu_swiglu_residual_rowmap(t):
    c = ctx()
    dtype = torch.bfloat16
    n, k = 256, 384
    x, w, b = _mk(t, n, k, dtype, 3)
    _, w2, _ = _mk(t, n, k, dtype, 4)
    xd, wd, w2d, bd = x.cuda(), w.cuda(), w2.cuda(), b.cuda()
    # GELU
    out = torch.empty(t, n, device="cuda", dtype=dtype)
    c.gemm(xd, wd, out, bias=bd, epilogue=EPI_GELU)
    ref = torch.nn.functional.gelu((x.float() @ w.float().T + b.float()).to(dtype).float()).to(dtype)
    assert rel_err(out, ref) < 8e-3
    # SwiGLU (dual accumulators)
    out = torch.empty(t, n, device="cuda", dtype=dtype)
    c.gemm(xd, wd, out, w2=w2d, epilogue=EPI_SWIGLU)
    g = (x.float() @ w.float().T).to(dtype)
    u = (x.float() @ w2.float().T).to(dtype)
    ref = (torch.nn.functional.silu(g.float()).to(dtype).float() * u.float()).to(dtype)
    e = rel_err(out, ref)
    record("gemm_swiglu", t=t, err=e)
    assert e < 8e-3
    # residual, in place
    res = (torch.randn(t, n, generator=torch.Generator().manual_seed(12)) * 0.3).to(dtype)
    h = res.cuda().clone()
    c.gemm(xd, wd, h, bias=bd, residual=h, epilogue=EPI_RESIDUAL)
    ref = (res.float() + (x.float() @ w.float().T + b.float()).to(dtype).float()).to(dtype)
    assert rel_err(h, ref) <= 2 ** -7 + 1e-6
    # row scatter: token i -> row perm[i] of a bigger buffer, -1 dropped
    big = torch.zeros(2 * t + 3, n, device="cuda", dtype=dtype)
    perm = torch.randperm(2 * t + 3, generator=torch.Generator().manual_seed(13))[:t].to(torch.int32)
    if t > 2:
        perm[1] = -1
    c.gemm(xd, wd, big, bias=bd, row_map=perm.cuda(), epilogue=EPI_NONE)
    torch.cuda.synchronize()
    full = (x.float() @ w.float().T + b.float()).to(dtype)
    exp = torch.zeros(2 * t + 3, n, dtype=dtype)
    for i in range(t):
        if perm[i] >= 0:
            exp[perm[i]] = full[i]
    assert rel_err(big, exp) < 8e-3
    assert (big.cpu()[exp.abs().sum(1) == 0] == 0).all()


def test_gemm_bad_args_report_errors():
    from chatts_b200._cabi import CtsError
    c = ctx()
    x = torch.zeros(4, 60, device="cuda", dtype=torch.bfloat16)      # pitch 120 B: not a multiple of 16
    w = torch.zeros(128, 60, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(4, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(CtsError):
        c.gemm(x, w, out)
    with pytest.raises(CtsError):
        c.gemm(torch.zeros(4, 64, device="cuda", dtype=torch.bfloat16), torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16),
               out, split_k=2)            # split-K without the partial epilogue


@pytest.mark.parametrize("t,inter,k", [(129, 128, 128), (300, 704, 256), (1000, 1408, 512), (2048, 256, 1024)])
def test_persistent_swiglu_interleaved(t, inter, k):
    """Persistent double-buffered kernel + tile-local SwiGLU on interleaved gate/up weights (CTS_EPI_SWIGLU_IL), and the
    decode-side cts_reduce_swiglu(interleaved) on the same weights."""
    c = ctx()
    dtype = torch.bfloat16
    g = torch.Generator().manual_seed(t + inter)
    x = (torch.randn(t, k, generator=g) * 0.5).to(dtype)
    wg = (torch.randn(inter, k, generator=g) * 0.1).to(dtype)
    wu = (torch.randn(inter, k, generator=g) * 0.1).to(dtype)
    wil = torch.stack([wg.view(-1, 64, k), wu.view(-1, 64, k)], 1).reshape(2 * inter, k).contiguous()
    gg = (x.float() @ wg.float().T).to(dtype)
    uu = (x.float() @ wu.float().T).to(dtype)
    ref = (torch.nn.functional.silu(gg.float()).to(dtype).float() * uu.float()).to(dtype)
    out = torch.full((t, inter), float("nan"), device="cuda", dtype=dtype)
    c.gemm(x.cuda(), wil.cuda(), out, epilogue=6)
    torch.cuda.synchronize()
    e = rel_err(out, ref)
    record("gemm_persistent_swiglu_il", t=t, inter=inter, k=k, err=e)
    assert torch.isfinite(out.float()).all() and e < 8e-3
    # decode-style: split-K partials + interleaved reduce on a few rows
    tt, s = min(t, 8), 2
    part = torch.empty(s, tt, 2 * inter, device="cuda", dtype=torch.float32)
    c.gemm(x[:tt].cuda().contiguous(), wil.cuda(), part, epilogue=EPI_PARTIAL, split_k=s)
    out2 = torch.empty(tt, inter, device="cuda", dtype=dtype)
    c.reduce_swiglu(part, s, tt, inter, out2, interleaved=True)
    torch.cuda.synchronize()
    assert rel_err(out2, ref[:tt]) < 8e-3


@pytest.mark.parametrize("t,n,k", [(257, 384, 640), (1024, 5120, 512), (700, 200, 136)])
def test_persistent_bias_gelu_residual(t, n, k):
    c = ctx()
    dtype = torch.bfloat16
    x, w, b = _mk(t, n, k, dtype, 7)
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    lin = x.float() @ w.float().T + b.float()
    out = torch.full((t, n), float("nan"), device="cuda", dtype=dtype)
    c.gemm(xd, wd, out, bias=bd, epilogue=EPI_GELU)
    eg = rel_err(out, torch.nn.functional.gelu(lin.to(dtype).float()).to(dtype))
    assert eg <= 2 ** -7 + 1e-6, eg
    res = (torch.randn(t, n, generator=torch.Generator().manual_seed(11)) * 0.3).to(dtype)
    h = res.cuda().clone()
    c.gemm(xd, wd, h, bias=bd, residual=h, epilogue=EPI_RESIDUAL)          # in place
    torch.cuda.synchronize()
    ref = (res.float() + lin.to(dtype).float()).to(dtype)
    e = rel_err(h, ref)
    # at most one bf16 ulp (2^-7 of the largest magnitude) anywhere: accumulation order only
    n_off = int(((h.float().cpu() - ref.float()).abs() > 0).sum())
    record("gemm_persistent_residual", t=t, n=n, k=k, err=e, elements_differing=n_off)
    assert e <= 2 ** -7 + 1e-6, (e, n_off)


def test_persistent_kernel_is_deterministic_under_repetition():
    """Race detector: the persistent double-buffered kernel must give bit-identical results on 12 repetitions
    (RESIDUAL with a separate residual buffer, and interleaved SwiGLU)."""
    c = ctx()
    dtype = torch.bfloat16
    t, n, k = 1536, 5120, 1024
    x, w, b = _mk(t, n, k, dtype, 21)
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    res = (torch.randn(t, n, generator=torch.Generator().manual_seed(3)) * 0.3).to(dtype).cuda()
    first = None
    for _ in range(12):
        out = torch.empty(t, n, device="cuda", dtype=dtype)
        c.gemm(xd, wd, out, bias=bd, residual=res, epilogue=EPI_RESIDUAL)
        out2 = torch.empty(t, n // 2, device="cuda", dtype=dtype)
        c.gemm(xd, wd, out2, epilogue=6)
        torch.cuda.synchronize()
        if first is None:
            first = (out.clone(), out2.clone())
            ref = (res.float().cpu() + (x.float() @ w.float().T + b.float()).to(dtype).float()).to(dtype)
            assert rel_err(out, ref) <= 2 ** -7 + 1e-6
        else:
            assert torch.equal(out, first[0]) and torch.equal(out2, first[1])
