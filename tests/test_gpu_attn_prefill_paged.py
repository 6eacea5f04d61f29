"""cts_attn_prefill_paged (csrc/attention.cu): causal GQA of new query rows over the keys of the paged KV cache -- a cached prompt
prefix plus the new rows -- against an fp32 torch statement of paged attention, and bit for bit against cts_attn_prefill and against
itself (suffix rows of a full prefill, repetition, foreign cache rows)."""
import math

import pytest
import torch

from oracle import decoder as od
from tests.gpu_util import ctx, record, rel_err

pytestmark = pytest.mark.gpu
DTS = [pytest.param(torch.bfloat16, id="bf16"), pytest.param(torch.float16, id="fp16")]
GQA = [(4, 4), (4, 2), (10, 2), (16, 2)]                       # 1:1, 2:1, 5:1, 8:1
# (prefix, q_len) of the sequences of one batch: every batch mixes sequences with and without a prefix
SHORT = [(p, n) for p in (0, 1, 63, 64, 65) for n in (1, 7, 64)]
LONG = [(p, n) for p in (576, 2464) for n in (1, 7, 64, 200)] + [(p, 200) for p in (0, 1, 63, 64, 65)]


def _fill_cache(seqs, nkv, d, page, DT, g, foreign="random"):
    """Random K/V for every position of every sequence, scattered over the pages of a cache whose other rows hold ``foreign``
    ("random", "zero", "nan" or "max": NaN / +-max of the dtype).  Returns (k_cache, v_cache, page_table, k_seq, v_seq)."""
    kv_lens = [p + n for p, n in seqs]
    max_pages = max((L + page - 1) // page for L in kv_lens) + 1
    n_pages = len(seqs) * max_pages + 3
    shape = (n_pages, nkv, page, d)
    if foreign == "random":
        kc, vc = torch.randn(shape, generator=g).to(DT), torch.randn(shape, generator=g).to(DT)
    elif foreign == "zero":
        kc, vc = torch.zeros(shape, dtype=DT), torch.zeros(shape, dtype=DT)
    elif foreign == "nan":
        kc, vc = torch.full(shape, float("nan"), dtype=DT), torch.full(shape, float("nan"), dtype=DT)
    else:
        mx = torch.finfo(DT).max
        sign = torch.where(torch.rand(shape, generator=torch.Generator().manual_seed(99)) < 0.5, -1.0, 1.0)   # g's stream untouched
        kc, vc = (sign * mx).to(DT), (-sign * mx).to(DT)
    pt = torch.randperm(n_pages, generator=g)[: len(seqs) * max_pages].view(len(seqs), max_pages).to(torch.int32)
    ks, vs = [], []
    for b, L in enumerate(kv_lens):
        k = torch.randn(L, nkv, d, generator=g).to(DT)
        v = torch.randn(L, nkv, d, generator=g).to(DT)
        pos = torch.arange(L)
        pg = pt[b, pos // page].long()
        kc[pg, :, pos % page] = k
        vc[pg, :, pos % page] = v
        ks.append(k)
        vs.append(v)
    return kc, vc, pt, ks, vs


def _run(c, q, seqs, kc, vc, pt, nh, nkv, d, page):
    qlens = [n for _, n in seqs]
    cu = torch.tensor([0] + torch.tensor(qlens).cumsum(0).tolist(), dtype=torch.int32)
    kv_lens = torch.tensor([p + n for p, n in seqs], dtype=torch.int32)
    out = torch.full((q.shape[0], nh * d), float("nan"), device="cuda", dtype=q.dtype)
    c.attn_prefill_paged(q.cuda(), cu.cuda(), kv_lens.cuda(), kc.cuda(), vc.cuda(), pt.cuda(), len(seqs), max(qlens), nh, nkv, d, page,
                         1.0 / math.sqrt(d), out)
    torch.cuda.synchronize()
    return out.cpu()


def _case(d, nh, nkv, page, seqs, DT):
    c = ctx()
    g = torch.Generator().manual_seed(d * 1000 + nh * 10 + nkv + page)
    kc, vc, pt, ks, vs = _fill_cache(seqs, nkv, d, page, DT, g)
    T = sum(n for _, n in seqs)
    q = torch.randn(T, nh * d, generator=g).to(DT)
    out = _run(c, q, seqs, kc, vc, pt, nh, nkv, d, page)
    again = _run(c, q, seqs, kc, vc, pt, nh, nkv, d, page)
    assert torch.equal(out, again), "two runs on the same inputs differ"
    refs, o = [], 0
    for (p, n), k, v in zip(seqs, ks, vs):
        refs.append(od.attention(q[o:o + n].view(n, nh, d).float(), k.float(), v.float(), nh // nkv, p))
        o += n
    ref = torch.cat(refs)
    e = rel_err(out, ref)
    record("attn_prefill_paged", d=d, nh=nh, nkv=nkv, page=page, seqs=str(seqs), dtype=str(DT), err=e)
    assert torch.isfinite(out.float()).all()
    assert e < 1.5e-2, e


@pytest.mark.parametrize("DT", DTS)
@pytest.mark.parametrize("page", [16, 32, 64])
@pytest.mark.parametrize("nh,nkv", GQA)
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("seqs", [pytest.param(SHORT, id="short"), pytest.param(LONG, id="long")])
def test_matches_fp32_paged_attention(seqs, d, nh, nkv, page, DT):
    _case(d, nh, nkv, page, seqs, DT)


@pytest.mark.parametrize("DT", DTS)
@pytest.mark.parametrize("d,nh,nkv,page,lens", [(128, 10, 2, 16, [1, 64, 65, 300]), (128, 16, 2, 64, [577, 7]),
                                                (64, 4, 2, 32, [5, 64, 129, 200]), (64, 4, 4, 16, [63, 1, 130])])
def test_no_prefix_is_cts_attn_prefill_bit_for_bit(d, nh, nkv, page, lens, DT):
    """kv_lens == q lens: the paged kernel gives the bits of the linear one on the same keys."""
    c = ctx()
    g = torch.Generator().manual_seed(sum(lens) + d)
    seqs = [(0, n) for n in lens]
    kc, vc, pt, ks, vs = _fill_cache(seqs, nkv, d, page, DT, g)
    T = sum(lens)
    q = torch.randn(T, nh * d, generator=g).to(DT)
    paged = _run(c, q, seqs, kc, vc, pt, nh, nkv, d, page)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32)
    lin = torch.full((T, nh * d), float("nan"), device="cuda", dtype=DT)
    c.attn_prefill(q.cuda(), torch.cat(ks).reshape(T, -1).cuda(), torch.cat(vs).reshape(T, -1).cuda(), cu.cuda(), len(lens), max(lens),
                   nh, nkv, d, 1.0 / math.sqrt(d), lin)
    torch.cuda.synchronize()
    assert torch.equal(paged, lin.cpu())


@pytest.mark.parametrize("DT", DTS)
@pytest.mark.parametrize("d,nh,nkv,page", [(128, 10, 2, 16), (128, 40, 8, 64), (64, 4, 2, 32)])
@pytest.mark.parametrize("full,split", [(200, 64), (700, 576), (130, 1), (2600, 2464), (64, 63)])
def test_suffix_rows_equal_the_full_prefill(d, nh, nkv, page, full, split, DT):
    """A query row gives the same bits whether it is computed in a full prefill or in a suffix call over the same cache."""
    c = ctx()
    g = torch.Generator().manual_seed(full + split + d)
    kc, vc, pt, _, _ = _fill_cache([(0, full)], nkv, d, page, DT, g)
    q = torch.randn(full, nh * d, generator=g).to(DT)
    whole = _run(c, q, [(0, full)], kc, vc, pt, nh, nkv, d, page)
    suffix = _run(c, q[split:], [(split, full - split)], kc, vc, pt, nh, nkv, d, page)
    assert torch.equal(suffix, whole[split:])


@pytest.mark.parametrize("DT", DTS)
@pytest.mark.parametrize("foreign", ["nan", "max"])
@pytest.mark.parametrize("d,nh,nkv,page", [(128, 10, 2, 16), (128, 8, 1, 32), (64, 4, 2, 64), (64, 8, 8, 16)])
def test_foreign_cache_rows_do_not_leak(d, nh, nkv, page, foreign, DT):
    """Every cache row that is not a live key of some sequence holds NaN or +-max: the output is the bits of a zero-filled cache."""
    c = ctx()
    seqs = [(0, 5), (63, 2), (64, 1), (100, 29), (17, 64)]
    outs = []
    for fill in ("zero", foreign):
        g = torch.Generator().manual_seed(7 + d + page)
        kc, vc, pt, _, _ = _fill_cache(seqs, nkv, d, page, DT, g, foreign=fill)
        q = torch.randn(sum(n for _, n in seqs), nh * d, generator=g).to(DT)
        outs.append(_run(c, q, seqs, kc, vc, pt, nh, nkv, d, page))
    assert torch.isfinite(outs[0].float()).all()
    assert torch.equal(outs[0], outs[1])


def test_argument_errors():
    from chatts_b200._cabi import CtsError
    c = ctx()
    DT = torch.bfloat16
    q = torch.zeros(4, 8 * 64, device="cuda", dtype=DT)
    kc = torch.zeros(4, 2, 16, 64, device="cuda", dtype=DT)
    cu = torch.tensor([0, 4], dtype=torch.int32, device="cuda")
    kvl = torch.tensor([4], dtype=torch.int32, device="cuda")
    pt = torch.zeros(1, 4, dtype=torch.int32, device="cuda")
    out = torch.zeros_like(q)
    ok = dict(nh=8, nkv=2, head_dim=64, page_size=16)
    c.attn_prefill_paged(q, cu, kvl, kc, kc, pt, 1, 4, ok["nh"], ok["nkv"], ok["head_dim"], ok["page_size"], 0.125, out)
    torch.cuda.synchronize()
    for bad, msg in ((dict(page_size=8), "page_size"), (dict(nh=18), "nh/nkv"), (dict(nh=7), "nh/nkv"), (dict(nh=32), "nh/nkv"),
                     (dict(head_dim=96), "head_dim")):
        a = dict(ok, **bad)
        with pytest.raises(CtsError, match=msg):
            c.attn_prefill_paged(q, cu, kvl, kc, kc, pt, 1, 4, a["nh"], a["nkv"], a["head_dim"], a["page_size"], 0.125, out)
