#!/usr/bin/env python
"""The two W4A16 decode GEMMs alone at the ChatTS-14B projection shapes: packed GB/s per launch (distinct weights per launch, >> L2)
for several split factors and token counts, next to the bf16 decode GEMM on the dequantised weight.
   cts_gemm_w4      (wgmma operand path, csrc/gemm_w4.cu)        -- T = 32 only
   cts_gemm_w4_mma  (registers + mma.sync, csrc/gemm_w4_mma.cu) -- T = 1 / 8 / 16 / 32
`--once` runs a few launches of the mma kernel only (for ncu); W4_TC5=0 skips the wgmma kernel."""
import json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from chatts_b200 import _cabi  # noqa: E402
from chatts_b200.weights import repack_w4_mma  # noqa: E402


def main():
    once = "--once" in sys.argv
    tc5 = os.environ.get("W4_TC5", "1") != "0" and not once
    c = _cabi.get_context()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(1)
    res = {}
    shapes = {"gate_up": (27648, 5120), "down": (5120, 13824), "qkv": (7168, 5120), "o": (5120, 5120)}
    for name, (n, k) in shapes.items():
        L = 2 if once else max(2, int(600e6 // (n * k // 2)))          # enough distinct weights to defeat the L2
        qw = [torch.randint(0, 256, (n, k // 2), generator=g, device=dev, dtype=torch.uint8) for _ in range(L)]
        sc = (torch.rand(n, k // 128, generator=g, device=dev) * 0.01 + 0.005).to(torch.bfloat16)
        zp = torch.randint(1, 17, (n, k // 128), generator=g, device=dev, dtype=torch.uint8)
        frag = [repack_w4_mma(q, sc, zp, 128) for q in qw]
        wd = [torch.randn(n, k, generator=g, device=dev).to(torch.bfloat16) for _ in range(min(L, 4))]
        byts = n * k / 2 + n * (k // 128) * 4
        out = {}
        for T in ((int(os.environ.get('W4_ONCE_T', '32')),) if once else (1, 8, 16, 32)):
            x = (torch.randn(T, k, generator=g, device=dev) * 0.5).to(torch.bfloat16)
            sug = c.gemm_w4_mma_suggest_split(n, k, T)
            row = {}
            for split in ([sug] if once else sorted({1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, sug})):
                if split * 4 > k // 64:
                    continue
                ws = torch.empty(split * T * n, device=dev, dtype=torch.float32)
                us = bench._event_timer(lambda i: c.gemm_w4_mma(x, frag[i % L][0], frag[i % L][1], n, 128, ws, split, t=T), 2 * L if not once else 2)
                row[f"split{split}"] = {"us": round(us, 2), "packed_gbs": round(byts / (us * 1e-6) / 1e9, 1)}
            best = min(row, key=lambda kk: row[kk]["us"])
            out[f"mma_T{T}"] = {"suggested": f"split{sug}", "best": best, "best_us": row[best]["us"], "suggested_us": row[f"split{sug}"]["us"],
                                "best_packed_gbs": row[best]["packed_gbs"], "all": row}
            if not once:
                sp = c.suggest_split(n if name != "gate_up" else n // 2, k, T, name == "gate_up")
                ws = torch.empty(sp * T * n, device=dev, dtype=torch.float32)
                us = bench._event_timer(lambda i: c.gemm(x, wd[i % len(wd)], ws, epilogue=3, split_k=sp, t=T), 8)
                out[f"bf16_T{T}"] = {"split": sp, "us": round(us, 2), "gbs": round(n * k * 2 / (us * 1e-6) / 1e9, 1)}
                out[f"mma_T{T}"]["speedup_vs_bf16"] = round(us / row[best]["us"], 2)
        if tc5:
            T = 32
            x = (torch.randn(T, k, generator=g, device=dev) * 0.5).to(torch.bfloat16)
            split = c.gemm_w4_suggest_split(n, k)
            ws = torch.empty(split * T * n, device=dev, dtype=torch.float32)
            us = bench._event_timer(lambda i: c.gemm_w4(x, qw[i % L], sc, zp, 128, ws, split, t=T), 2 * L)
            out["tc5_T32"] = {"split": split, "us": round(us, 2), "packed_gbs": round(byts / (us * 1e-6) / 1e9, 1)}
        res[name] = out
        del qw, wd, frag
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
