"""Decode-sized cts_gemm (t <= 32): the persistent streaming kernel against gemm_tn_kernel (CTS_NO_STREAM_GEMM=1), BIT FOR BIT.

Both kernels accumulate every output with the same m64nBNk16 wgmma sequence over the same K range of its split, so the fp32 partials and
the split-1 outputs must be identical, whatever ring depth, tile height or K blocks per ring slot the streaming kernel runs with."""
import contextlib
import copy
import ctypes as C
import os

import pytest
import torch

from tests.gpu_util import ctx

pytestmark = pytest.mark.gpu
EPI_NONE, EPI_PARTIAL = 0, 3
_ctxs = {}


@contextlib.contextmanager
def _env(env):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


class _EnvCtx:
    """A second context of the same library, created with the given CTS_* variables set: the library reads them at context creation.
    They also stay set around every call made through this object, because the CPU shim's stand-in context reads them at each launch."""

    def __init__(self, env):
        base = ctx()
        self.env = env
        with _env(env):
            h = C.c_void_p()
            assert base.lib.cts_ctx_create(base.device, C.byref(h)) == 0
        self.c = copy.copy(base)
        self.c.h = h

    def gemm(self, *a, **k):
        with _env(self.env):
            return self.c.gemm(*a, **k)


def _ctx_env(**env):
    key = tuple(sorted(env.items()))
    if key not in _ctxs:
        _ctxs[key] = _EnvCtx(env)
    return _ctxs[key]


def _legacy():
    return _ctx_env(CTS_NO_STREAM_GEMM=1)


def _mk(t, n, k, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(t, k, generator=g) * 0.5).to(dtype)
    w = (torch.randn(n, k, generator=g) * 0.1).to(dtype)
    b = (torch.randn(n, generator=g) * 0.2).to(dtype)
    return x.cuda(), w.cuda(), b.cuda()


def _partials(c, x, w, s):
    out = torch.full((s, x.shape[0], w.shape[0]), float("nan"), device="cuda", dtype=torch.float32)
    c.gemm(x, w, out, epilogue=EPI_PARTIAL, split_k=s)
    torch.cuda.synchronize()
    return out


def _check_partials(x, w, s, c=None):
    new = _partials(c or ctx(), x, w, s)
    old = _partials(_legacy(), x, w, s)
    assert torch.isfinite(new).all()
    assert torch.equal(new, old)
    ref = x.float().cpu() @ w.float().cpu().T
    assert (new.sum(0).cpu() - ref).abs().max() / ref.abs().max() < 1e-5


@pytest.mark.parametrize("t", [1, 3, 8, 16, 17, 32])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_partials_bitwise_against_gemm_tn(t, dtype):
    x, w, _ = _mk(t, 1000, 1600, dtype, t)          # n not a multiple of 128; 25 K blocks in splits of 8 / 8 / 9
    _check_partials(x, w, 3)


@pytest.mark.parametrize("rows,kblocks,ctas", [(64, 1, 2), (64, 2, 3), (64, 4, 1), (128, 1, 1), (128, 2, 2), (128, 4, 1)])
def test_every_stream_shape_is_bitwise(rows, kblocks, ctas):
    """The tile height, the K blocks per ring slot and the ring depth move bytes, not arithmetic."""
    c = _ctx_env(CTS_STREAM_ROWS=rows, CTS_STREAM_KBLOCKS=kblocks, CTS_STREAM_CTAS=ctas)
    for t, n, k, s in [(1, 704, 1600, 3), (32, 200, 1088, 2), (9, 384, 512, 1)]:
        x, w, _ = _mk(t, n, k, torch.bfloat16, n + t)
        _check_partials(x, w, s, c)


# (n, k, dual): ChatTS-14B (hidden 5120, intermediate 13824, 40 + 2 x 8 heads of 128), ChatTS-8B (4096 / 12288, 32 + 2 x 8 heads),
# and the tensor-parallel shards of the 14B projections at TP2 and TP8 (column-split qkv / gate_up, row-split o / down)
PROJ = {
    "14b_qkv": (7168, 5120, False), "14b_o": (5120, 5120, False), "14b_gate_up": (13824, 5120, True), "14b_down": (5120, 13824, False),
    "8b_qkv": (6144, 4096, False), "8b_o": (4096, 4096, False), "8b_gate_up": (12288, 4096, True), "8b_down": (4096, 12288, False),
    "tp2_qkv": (3584, 5120, False), "tp2_o": (5120, 2560, False), "tp2_gate_up": (6912, 5120, True), "tp2_down": (5120, 6912, False),
    "tp8_qkv": (896, 5120, False), "tp8_o": (5120, 640, False), "tp8_gate_up": (1728, 5120, True), "tp8_down": (5120, 1728, False),
}


@pytest.mark.parametrize("t", [1, 32])
@pytest.mark.parametrize("name", sorted(PROJ))
def test_projection_shapes_bitwise(name, t):
    n, k, dual = PROJ[name]
    c = ctx()
    s = c.suggest_split(n, k, t, dual)
    x, w, _ = _mk(t, 2 * n if dual else n, k, torch.bfloat16, 7)
    _check_partials(x, w, s)


def _none(c, x, w, b):
    out = torch.full((x.shape[0], w.shape[0]), float("nan"), device="cuda", dtype=x.dtype)
    c.gemm(x, w, out, bias=b, epilogue=EPI_NONE)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("t,n,k", [(1, 1000, 512), (32, 1000, 512), (5, 130, 272), (1, 152064, 5120), (32, 152064, 5120)])
@pytest.mark.parametrize("bias", [False, True])
def test_split1_output_bitwise(t, n, k, bias):
    """CTS_EPI_NONE at split 1 (the lm_head at ChatTS-14B's vocabulary, and split-1 QKV with its bias)."""
    for dtype in ([torch.bfloat16, torch.float16] if n < 10000 else [torch.bfloat16]):
        x, w, b = _mk(t, n, k, dtype, n + t)
        b = b if bias else None
        new, old = _none(ctx(), x, w, b), _none(_legacy(), x, w, b)
        assert torch.isfinite(new.float()).all()
        assert torch.equal(new, old)


def test_repeatable():
    c = ctx()
    x, w, _ = _mk(17, 3000, 2048, torch.bfloat16, 3)
    first = _partials(c, x, w, 5)
    for _ in range(4):
        assert torch.equal(_partials(c, x, w, 5), first)


def test_argument_errors():
    from chatts_b200._cabi import CtsError
    x, w, _ = _mk(4, 256, 512, torch.bfloat16, 1)
    out = torch.empty(2, 4, 256, device="cuda", dtype=torch.float32)
    with pytest.raises(CtsError):
        ctx().gemm(x, w, torch.empty(9, 4, 256, device="cuda", dtype=torch.float32), epilogue=EPI_PARTIAL, split_k=9)   # 8 K blocks
    with pytest.raises(CtsError, match="CTS_STREAM_ROWS"):
        _ctx_env(CTS_STREAM_ROWS=96).gemm(x, w, out, epilogue=EPI_PARTIAL, split_k=2)
    with pytest.raises(CtsError, match="fewer than two"):
        _ctx_env(CTS_STREAM_CTAS=4, CTS_STREAM_KBLOCKS=4).gemm(x, w, out, epilogue=EPI_PARTIAL, split_k=2)
