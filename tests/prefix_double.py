"""TEST INFRASTRUCTURE ONLY: cts_attn_prefill_paged restated with plain torch ops on top of the torch/CPU test double of
tests/cabi_double.py, for the host-logic tests of prefix caching."""
from tests.cabi_double import TorchDouble


class PrefixDouble(TorchDouble):
    def attn_prefill_paged(self, q, cu_q, kv_lens, kc, vc, pt, B, max_q, nh, nkv, d, page, scale, out):
        for b in range(B):
            a, e, n = int(cu_q[b]), int(cu_q[b + 1]), int(kv_lens[b])
            pages = pt[b, : (n + page - 1) // page].long()
            kk = kc[pages].permute(0, 2, 1, 3).reshape(-1, nkv, d)[:n]
            vv = vc[pages].permute(0, 2, 1, 3).reshape(-1, nkv, d)[:n]
            out[a:e] = self._attn(q[a:e].view(-1, nh, d), kk, vv, nh // nkv, n - (e - a)).to(out.dtype)
