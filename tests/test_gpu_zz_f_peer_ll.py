"""cts_peer_allreduce_ll (csrc/allreduce_ll.cu: two-shot all-reduce with the flags inside the data) on ONE GPU: the W "ranks" are W
streams of this process, their symmetric regions W plain allocations -- to the kernel a peer is only a pointer, so the whole
protocol (scatter, owner reduction in rank order, gather, statistic, epochs, buffer reuse over consecutive calls) runs exactly as it
does over NVLink, minus the link.  The W kernels of a call spin on each other and therefore must be co-resident: sizes here keep
W x C x T <= 128 CTAs of 256 threads (one per SM suffices), and the kernel's bounded polls turn a scheduling surprise into a trap
instead of a hang.  Expected values: the rank-ordered fp32 sum formed step by step (bit-exact h), RMSNorm from h (tolerance: the
statistic's summation order differs from torch's), bit-identical results on all ranks.
The protocol
itself is model-checked on CPU in tests/test_peer_ll_protocol.py."""
import pytest
import torch

from tests.gpu_util import ctx, record

pytestmark = pytest.mark.gpu


class _Ranks:
    """W simulated ranks on one device: regions (2 buffer sets), states, streams."""

    def __init__(self, c, W, max_tokens, h):
        self.c, self.W, self.max_tokens, self.h = c, W, max_tokens, h
        self.bytes = c.peer_ll_region_bytes(W, max_tokens, h)
        self.regions = [[torch.zeros((self.bytes + 3) // 4, dtype=torch.int32, device="cuda") for _ in range(W)] for _ in range(2)]
        self.ptrs = [torch.tensor([r.data_ptr() for r in self.regions[b]], dtype=torch.int64, device="cuda") for b in range(2)]
        self.state = [torch.zeros(2, dtype=torch.int32, device="cuda") for _ in range(W)]
        self.streams = [torch.cuda.Stream() for _ in range(W)]

    def call(self, which, parts, split, resid, norm_w, eps, xn, T):
        """parts[r]: fp32 [split, T, h] of rank r; resid[r] is updated in place (as st.h is), xn[r] receives the norm."""
        torch.cuda.synchronize()
        for r in range(self.W):
            with torch.cuda.stream(self.streams[r]):
                self.c.peer_allreduce_ll(parts[r], split, self.ptrs[which], self.bytes, self.state[r], r, self.W, self.max_tokens,
                                         resid[r], resid[r], norm_w, eps, xn[r], T)
        torch.cuda.synchronize()


def _expected(parts, split, resid, dt):
    acc = torch.zeros_like(parts[0][0])
    for p in parts:
        loc = p[0].clone()
        for s in range(1, split):
            loc = loc + p[s]
        acc = acc + loc
    return (resid.float() + acc.to(dt).float()).to(dt)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("W,T,h,split", [(2, 1, 256, 1), (2, 5, 5120, 3), (4, 4, 5120, 2), (8, 1, 5120, 1), (8, 4, 5120, 2), (4, 3, 1024, 4), (8, 4, 4096, 1)])
def test_ll_allreduce_matches_rank_ordered_sum(W, T, h, split, dt):
    c = ctx()
    g = torch.Generator().manual_seed(W * 1000 + T + h)
    R = _Ranks(c, W, max(T, 16), h)
    h0 = (torch.randn(T, h, generator=g) * 0.5).to(dt).cuda()
    nw = (1.0 + 0.1 * torch.randn(h, generator=g)).to(dt).cuda()
    resid = [h0.clone() for _ in range(W)]
    xn = [torch.full((T, h), float("nan"), dtype=dt, device="cuda") for _ in range(W)]
    cur = h0.clone()
    worst = 0.0
    for n, which in enumerate([0, 1, 0, 1, 1, 0]):                       # alternating as the model does, plus one repeated set
        parts = [(torch.randn(split, T, h, generator=g) * 0.3).cuda() for _ in range(W)]
        R.call(which, parts, split, resid, nw, 1e-6, xn, T)
        cur = _expected(parts, split, cur, dt)
        for r in range(W):
            assert torch.equal(resid[r], cur), f"call {n}: h differs from the rank-ordered sum on rank {r}"
            assert torch.equal(xn[r], xn[0]), f"call {n}: norm_out differs between ranks 0 and {r}"
        x = cur.float()
        want = nw.float() * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)).to(dt).float()
        err = float((xn[0].float() - want).abs().max() / want.abs().max())
        worst = max(worst, err)
        assert err < 1.2e-2, f"call {n}: RMSNorm off by {err}"
    record("peer_ll_allreduce", W=W, T=T, h=h, split=split, dtype=str(dt), norm_rel=worst, bit_exact_h=True)


def test_ll_allreduce_without_norm_and_epoch_shared_with_other_sizes():
    """norm_w = None (residual only) and a T that changes from call to call over the same regions (prefill-sized, then decode-sized)."""
    c = ctx()
    dt, W, h = torch.bfloat16, 4, 2048
    g = torch.Generator().manual_seed(7)
    R = _Ranks(c, W, 8, h)
    for n, T in enumerate([8, 1, 5, 8, 2]):                                # W x C x T <= 128 CTAs: all co-resident
        h0 = (torch.randn(T, h, generator=g) * 0.5).to(dt).cuda()
        resid = [h0.clone() for _ in range(W)]
        parts = [(torch.randn(1, T, h, generator=g) * 0.3).cuda() for _ in range(W)]
        R.call(n % 2, parts, 1, resid, None, 1e-6, [None] * W, T)
        want = _expected(parts, 1, h0, dt)
        for r in range(W):
            assert torch.equal(resid[r], want)


def test_ll_rejects_bad_arguments():
    from chatts_b200._cabi import CtsError
    c = ctx()
    R = _Ranks(c, 2, 16, 256)
    h0 = torch.zeros(1, 256, dtype=torch.bfloat16, device="cuda")
    part = torch.zeros(1, 1, 256, device="cuda")
    with pytest.raises(CtsError):                                        # 3 ranks: not built
        c.peer_allreduce_ll(part, 1, R.ptrs[0], R.bytes, R.state[0], 0, 3, 16, h0, h0, None, 1e-6, None, 1)
    with pytest.raises(CtsError):                                        # region too small
        c.peer_allreduce_ll(part, 1, R.ptrs[0], R.bytes - 16, R.state[0], 0, 2, 16, h0, h0, None, 1e-6, None, 1)
    with pytest.raises(CtsError):                                        # more tokens than the region holds
        c.peer_allreduce_ll(torch.zeros(1, 17, 256, device="cuda"), 1, R.ptrs[0], R.bytes, R.state[0], 0, 2, 16,
                            torch.zeros(17, 256, dtype=torch.bfloat16, device="cuda"), torch.zeros(17, 256, dtype=torch.bfloat16, device="cuda"),
                            None, 1e-6, None, 17)


@pytest.mark.parametrize("W,T,N,Kr,S", [(2, 1, 256, 128, 1), (2, 7, 512, 320, 2), (4, 16, 512, 256, 3), (8, 32, 1024, 640, 2), (4, 32, 1024, 1728, 4)])
def test_fused_gemm_allreduce_tail(W, T, N, Kr, S):
    """gemm_decode_fused(CTS_FUSED_RESIDUAL, peer=...): row-parallel projection + all-reduce + residual (+ per-tile sums of squares) in
    ONE launch per rank, W ranks as W streams.  Expected h: each rank's partial from the validated split-K GEMM (splits added in
    order), ranks added in order, rounded, added to the residual -- bit for bit; ssq_out = per-tile sums of squares of that h."""
    c = ctx()
    dt = torch.bfloat16
    g = torch.Generator().manual_seed(W * 100 + T + N)
    tmax = 32
    R = _Ranks(c, W, tmax, N)
    need = tmax * N * 12 + tmax * (N // 128) * 8
    assert R.bytes >= need
    h0 = (torch.randn(T, N, generator=g) * 0.5).to(dt).cuda()
    hs = [h0.clone() for _ in range(W)]
    ssq = [torch.full((T, N // 128), float("nan"), device="cuda") for _ in range(W)]
    cur = h0.clone()
    for n, which in enumerate([0, 1, 0]):
        xs = [(torch.randn(T, Kr, generator=g) * 0.5).to(dt).cuda() for _ in range(W)]
        ws_ = [(torch.randn(N, Kr, generator=g) * 0.05).to(dt).cuda() for _ in range(W)]
        acc = torch.zeros(T, N, device="cuda")
        for r in range(W):
            buf = torch.empty(S * T * N, device="cuda", dtype=torch.float32)
            c.gemm(xs[r], ws_[r], buf, epilogue=3, split_k=S, t=T)
            part = buf.view(S, T, N)
            loc = part[0].clone()
            for s in range(1, S):
                loc = loc + part[s]
            acc = acc + loc
        torch.cuda.synchronize()
        for r in range(W):
            with torch.cuda.stream(R.streams[r]):
                c.gemm_decode_fused(xs[r], ws_[r], 0, S, T, h=hs[r], ssq_out=ssq[r], peer=(R.ptrs[which], R.bytes, R.state[r], r, W, tmax))
        torch.cuda.synchronize()
        cur = (cur.float() + acc.to(dt).float()).to(dt)
        want_ssq = cur.float().pow(2).view(T, N // 128, 128).sum(-1)
        for r in range(W):
            assert torch.equal(hs[r], cur), f"call {n}: h differs from the rank-ordered sum on rank {r}"
            assert torch.equal(ssq[r], ssq[0]), f"call {n}: statistic differs between ranks 0 and {r}"
        assert torch.allclose(ssq[0], want_ssq, rtol=1e-4), f"call {n}: per-tile sums of squares"
    record("fused_gemm_allreduce_tail", W=W, T=T, N=N, K_per_rank=Kr, split=S, bit_exact_h=True)
