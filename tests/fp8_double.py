"""TEST INFRASTRUCTURE ONLY: the FP8 entry points of the C-ABI binding (cts_gemm_fp8, cts_gemm_fp8_suggest_split, cts_fp8_dequant) restated
with plain torch ops on top of the torch/CPU test double of tests/cabi_double.py, for the host-logic tests of FP8 models."""
import torch

from tests.cabi_double import TorchDouble


class Fp8Double(TorchDouble):
    def gemm_fp8_suggest_split(self, n, k, t=1): return self.split if k >= 128 * self.split else 1

    def _fp8_weight(self, qw, scales, k):
        """The fragment-major layout decoded back to e4m3 values times the row scale, in fp32 (the formula include/chatts_b200.h states
        for cts_gemm_fp8_args, written independently of weights.py:pack_fp8_mma)."""
        n = scales.shape[0]
        key = (qw.data_ptr(), scales.data_ptr(), int(k))
        cache = self.__dict__.setdefault("_fp8_cache", {})
        if key not in cache:
            tiles = -(-n // 256)
            b = qw.view(tiles, k // 64, 16, 2, 32, 2, 2, 4)                  # [tile, kb, m, ks // 2, lane, ks % 2, j, byte]
            q = torch.zeros(tiles * 256, k, dtype=torch.uint8)
            for lane in range(32):
                g, tq = lane >> 2, lane & 3
                for ks in range(4):
                    for j in range(2):
                        for byte in range(4):
                            rows = torch.arange(16) * 16 + g + 8 * (byte >> 1)                               # feature row of m-tile m
                            col = 16 * ks + 2 * tq + 8 * j + (byte & 1)
                            v = b[:, :, :, ks >> 1, lane, ks & 1, j, byte]                                   # [tile, kb, m]
                            q.view(tiles, 256, k // 64, 64)[:, rows, :, col] = v.permute(0, 2, 1)
            cache[key] = q[:n].view(torch.float8_e4m3fn).float() * scales.float()[:, None]
        return cache[key]

    def gemm_fp8(self, x, qw, scales, k, out, split_k, t=None):
        t = x.shape[0] if t is None else t
        assert int(k) % 64 == 0 and 1 <= split_k <= int(k) // 64 and t <= 32                  # cts_gemm_fp8_args
        w = self._fp8_weight(qw, scales, int(k))
        xx, kb = x[:t].float(), int(k) // 64
        o = out.view(-1)[: split_k * t * w.shape[0]].view(split_k, t, w.shape[0])
        for s in range(split_k):
            a, e = kb * s // split_k * 64, kb * (s + 1) // split_k * 64
            o[s] = xx[:, a:e] @ w[:, a:e].T

    def fp8_dequant(self, qw, scales, k, out):
        out[: scales.shape[0], : int(k)] = self._fp8_weight(qw, scales, int(k)).to(out.dtype)
