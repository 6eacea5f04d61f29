"""attention_bwd_wgmma.cu (wgmma attention backward, head_dim 128, the default; CTS_ATTN_BWD_WGMMA=0 selects the HMMA kernels)
against autograd and against the HMMA kernels.  It drives an mbarrier pipeline with bounded waits and lives late in the suite so
that a trapped wait cannot cost any other result."""
import math

import numpy as np
import pytest
import torch

from tests.cabi_double import TorchDouble
from tests.gpu_util import ctx, record

DT = torch.bfloat16
DBL = TorchDouble()


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rn(g, *shape, std=1.0, dtype=DT):
    return (torch.randn(*shape, generator=g) * std).to(dtype)


pytestmark = pytest.mark.gpu


def _attn_inputs(d, lens, nh=4, nkv=2, dtype=DT):
    T = sum(lens)
    g = _g(T + d)
    q, k, v, do = _rn(g, T, nh * d, dtype=dtype), _rn(g, T, nkv * d, dtype=dtype), _rn(g, T, nkv * d, dtype=dtype), _rn(g, T, nh * d, dtype=dtype)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)
    return T, q, k, v, do, cu


@pytest.mark.parametrize("lens,nh,nkv,dtype", [([1], 4, 2, DT), ([5, 64, 65], 4, 2, DT), ([130, 17, 200, 1], 4, 2, DT), ([577], 4, 2, DT),
                                               ([128, 256], 8, 1, DT), ([300, 129], 4, 4, torch.float16)])
def test_attention_backward_wgmma(lens, nh, nkv, dtype, monkeypatch):
    """attention_bwd_wgmma.cu (head_dim 128): wgmma dQ and dK/dV kernels against autograd AND against the HMMA kernels of
    attention_bwd.cu (CTS_ATTN_BWD_WGMMA=0) on the same inputs."""
    c = ctx()
    d = 128
    T, q, k, v, do, cu = _attn_inputs(d, lens, nh, nkv, dtype)
    sc = 1.0 / math.sqrt(d)
    qd, kd, vd, dod, cud = q.cuda(), k.cuda(), v.cuda(), do.cuda(), cu.cuda()
    o, lse = torch.empty(T, nh * d, device="cuda", dtype=dtype), torch.empty(T, nh, device="cuda")
    c.attn_prefill_lse(qd, kd, vd, cud, len(lens), max(lens), nh, nkv, d, sc, o, lse)
    ws = torch.empty(T, nh, device="cuda")
    outs = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("CTS_ATTN_BWD_WGMMA", flag)
        dq, dk, dv = (torch.full((T, n_ * d), float("nan"), device="cuda", dtype=dtype) for n_ in (nh, nkv, nkv))
        c.attn_bwd(qd, kd, vd, o, dod, lse, cud, len(lens), max(lens), nh, nkv, d, sc, ws, dq, dk, dv)
        torch.cuda.synchronize()
        outs[flag] = (dq, dk, dv)
    rq, rk, rv = torch.empty(T, nh * d, dtype=dtype), torch.empty(T, nkv * d, dtype=dtype), torch.empty(T, nkv * d, dtype=dtype)
    DBL.attn_bwd(q, k, v, None, do, None, cu, len(lens), max(lens), nh, nkv, d, sc, None, rq, rk, rv)
    # absolute floor in the denominator: a length-1 sequence has dQ = dK = 0 exactly and the kernels leave ~1e-7 of rounding noise there
    err = lambda a, r_: float((a.float().cpu() - r_.float().cpu()).abs().max() / r_.float().abs().max().clamp_min(1e-4))
    errs = [err(a, r_) for a, r_ in zip(outs["1"], (rq, rk, rv))]
    cross = [err(a, b_) for a, b_ in zip(outs["1"], outs["0"])]
    record("attn_bwd_wgmma", lens=str(lens), nh=nh, nkv=nkv, dq=errs[0], dk=errs[1], dv=errs[2], vs_hmma=max(cross))
    for t_ in outs["1"]:
        assert torch.isfinite(t_.float()).all()
    assert max(errs) < 2e-2 and max(cross) < 2e-2, (errs, cross)
    # deterministic
    dq2, dk2, dv2 = (torch.empty_like(t_) for t_ in outs["1"])
    c.attn_bwd(qd, kd, vd, o, dod, lse, cud, len(lens), max(lens), nh, nkv, d, sc, ws, dq2, dk2, dv2)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b_) for a, b_ in zip(outs["1"], (dq2, dk2, dv2)))
