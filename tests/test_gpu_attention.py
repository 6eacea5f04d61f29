"""Attention kernels against the oracle's eager GQA attention (modeling_qwen2.py:161-184)."""
import math

import pytest
import torch

from oracle import decoder as od
from tests.gpu_util import ctx, record, rel_err

pytestmark = pytest.mark.gpu
DT = torch.bfloat16


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("lens", [[1], [5, 64, 65], [130, 17, 200, 1], [577]])
def test_prefill_varlen_causal_gqa(d, lens):
    _prefill_case(d, lens, torch.bfloat16)


@pytest.mark.parametrize("d", [64, 128])
def test_prefill_fp16(d):
    _prefill_case(d, [129, 64, 300], torch.float16)


@pytest.mark.parametrize("DT", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("lens", [[577], [300, 129, 64]])
def test_prefill_growing_scores_force_the_lazy_rescale(lens, DT):
    """The wgmma kernel rescales l and the O accumulator registers whenever a tile raises a row's running maximum.  Random data
    rarely moves the maximum after the first tile; here the scores grow along the sequence (keys scaled by their position), so every
    64-key tile raises the maximum for most rows -- the rescale runs in nearly every tile, with large correction factors."""
    _prefill_case(128, lens, DT, ramp=True)


@pytest.mark.parametrize("DT", [torch.bfloat16, torch.float16])
def test_prefill_many_items_per_persistent_cta(DT):
    """40 sequences x 8 heads x 3 query tiles = 960 (query tile, head, sequence) items, many of them dead (sequences shorter than the
    longest): the wgmma kernel's grid covers every item, and the CTAs of dead items must leave before issuing anything."""
    lens = [300, 17, 129, 256, 1, 64, 200, 299, 128, 65] * 4
    _prefill_case(128, lens, DT, nh=8)


def _prefill_case(d, lens, DT, ramp=False, nh=4):
    c = ctx()
    nkv = 2
    T = sum(lens)
    g = torch.Generator().manual_seed(T + d)
    q = torch.randn(T, nh, d, generator=g).to(DT)
    k = torch.randn(T, nkv, d, generator=g).to(DT)
    v = torch.randn(T, nkv, d, generator=g).to(DT)
    if ramp:
        # q = |q| and k = position-dependent positive multiple of |k|: q.k grows roughly linearly with the key position (~ +0.6 per key
        # after the 1/sqrt(d) scale, i.e. ~ +55 log2 units per 64-key tile), rows with a small |q| grow slower than the threshold
        pos = torch.cat([torch.arange(n) for n in lens]).float()
        q = (q.float().abs() * torch.linspace(0.02, 1.0, nh * d).view(1, nh, d)).to(DT)
        k = (k.float().abs() * (0.05 + pos / 64.0).view(-1, 1, 1)).to(DT)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)
    out = torch.full((T, nh * d), float("nan"), device="cuda", dtype=DT)
    c.attn_prefill(q.cuda().contiguous(), k.cuda().contiguous(), v.cuda().contiguous(), cu.cuda(), len(lens), max(lens), nh, nkv, d,
                   1.0 / math.sqrt(d), out)
    torch.cuda.synchronize()
    ref = torch.cat([od.attention(q[a:b].float(), k[a:b].float(), v[a:b].float(), nh // nkv, 0)
                     for a, b in zip(cu[:-1].tolist(), cu[1:].tolist())])
    e = rel_err(out, ref)
    record("attn_prefill", d=d, lens=str(lens), err=e, dtype=str(DT))
    assert torch.isfinite(out.float()).all()
    assert e < 1.5e-2


@pytest.mark.parametrize("d,nh,nkv,page", [(128, 40, 8, 64), (128, 10, 2, 64), (64, 4, 2, 16), (128, 8, 1, 32), (64, 8, 8, 64),
                                            (128, 14, 2, 16), (128, 5, 1, 64)])
@pytest.mark.parametrize("splits", [1, 3, 16])
def test_decode_paged(d, nh, nkv, page, splits):
    _decode_case(d, nh, nkv, page, splits, torch.bfloat16)


@pytest.mark.parametrize("d,nh,nkv,page", [(128, 40, 8, 64), (64, 4, 2, 16)])
def test_decode_paged_fp16(d, nh, nkv, page):
    _decode_case(d, nh, nkv, page, 3, torch.float16)


def _decode_case(d, nh, nkv, page, splits, DT):
    c = ctx()
    seq_lens = [1, page, page + 1, 5 * page - 3, 333][: 4 if nh == 40 else 5]
    B = len(seq_lens)
    max_pages = (max(seq_lens) + page - 1) // page + 1
    n_pages = B * max_pages + 3
    g = torch.Generator().manual_seed(d + nh + page)
    kc = torch.randn(n_pages, nkv, page, d, generator=g).to(DT)
    vc = torch.randn(n_pages, nkv, page, d, generator=g).to(DT)
    perm = torch.randperm(n_pages, generator=g)[: B * max_pages].view(B, max_pages).to(torch.int32)   # scattered pages
    q = torch.randn(B, nh, d, generator=g).to(DT)
    ws = torch.zeros(c.attn_decode_workspace_floats(B, nh, d, splits), device="cuda", dtype=torch.float32)
    out = torch.full((B, nh * d), float("nan"), device="cuda", dtype=DT)
    for _ in range(2):          # twice: the arrival counters must reset themselves
        out.fill_(float("nan"))
        c.attn_decode(q.cuda(), kc.cuda(), vc.cuda(), perm.cuda(), torch.tensor(seq_lens, dtype=torch.int32).cuda(), B, nh, nkv, d, page,
                      1.0 / math.sqrt(d), splits, ws, out)
        torch.cuda.synchronize()
    refs = []
    for b, sl in enumerate(seq_lens):
        pages = perm[b, : (sl + page - 1) // page].long()
        kk = kc[pages].permute(0, 2, 1, 3).reshape(-1, nkv, d)[:sl]      # [tokens, nkv, d]
        vv = vc[pages].permute(0, 2, 1, 3).reshape(-1, nkv, d)[:sl]
        refs.append(od.attention(q[b:b + 1].float(), kk.float(), vv.float(), nh // nkv, sl - 1))
    ref = torch.cat(refs)
    e = rel_err(out, ref)
    record("attn_decode", d=d, nh=nh, nkv=nkv, page=page, splits=splits, err=e)
    assert torch.isfinite(out.float()).all()
    assert e < 1e-2
