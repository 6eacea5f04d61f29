#!/usr/bin/env python
"""The wgmma prefill attention kernel ALONE (no model): causal-useful TFLOP/s at the benchmark shape (32 x 576, 40 / 8 heads of 128)
and at two longer ones, next to the attention kernels installed on the box (library code, a stated comparison only).  One JSON line.
`--once` runs the benchmark shape a few times only (for ncu)."""
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from chatts_b200 import _cabi  # noqa: E402


def main():
    once = "--once" in sys.argv
    c = _cabi.get_context()
    nh, nkv, d = 40, 8, 128
    scale = 1.0 / math.sqrt(d)
    dev = "cuda"
    peak, src = bench.tensor_peak()
    out = {"peak_tflops": peak, "peak_source": src, "shapes": {}}
    for dt in ((torch.bfloat16,) if once else (torch.bfloat16, torch.float16)):
        for batch, seqlen in (((32, 576),) if once else ((32, 576), (8, 2464), (4, 4096))):
            T = batch * seqlen
            g = torch.Generator(device=dev).manual_seed(7)
            q = (torch.randn(T, nh * d, device=dev, generator=g) * 0.5).to(dt)
            k = (torch.randn(T, nkv * d, device=dev, generator=g) * 0.5).to(dt)
            v = (torch.randn(T, nkv * d, device=dev, generator=g) * 0.5).to(dt)
            o = torch.empty(T, nh * d, device=dev, dtype=dt)
            cu = torch.arange(0, T + 1, seqlen, dtype=torch.int32, device=dev)
            us = bench._event_timer(lambda i: c.attn_prefill(q, k, v, cu, batch, seqlen, nh, nkv, d, scale, o), 3 if once else 10)
            flops = batch * 4.0 * (seqlen * seqlen / 2.0) * d * nh
            row = {"us": round(us, 1), "causal_useful_tflops": round(flops / (us * 1e-6) / 1e12, 1), "frac_of_tensor_peak": round(flops / (us * 1e-6) / 1e12 / peak, 3)}
            if not once and dt == torch.bfloat16:
                row["vs_installed"] = {kk: ({"us": round(vv["us"], 1), "tflops": round(vv["tflops"], 1)} if "us" in vv else vv)
                                       for kk, vv in bench.installed_attention(q, k, v, batch, seqlen, nh, nkv, d, scale, flops, bench._event_timer).items()}
            out["shapes"][f"{str(dt).split('.')[-1]}_{batch}x{seqlen}"] = row
    print(json.dumps(out))


if __name__ == "__main__":
    main()
