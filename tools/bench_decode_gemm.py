#!/usr/bin/env python
"""Decode GEMM microbenchmark: the 16-bit projections of ChatTS-14B (qkv / o / gate_up / down of one layer, and the lm_head) at
t = 1 / 8 / 32, gemm_stream_kernel (the default) against gemm_tn_kernel (a context created with CTS_NO_STREAM_GEMM=1), alternating in one
process, with the FP8 decode GEMM on the same projections as the rate weight streaming reaches on this card.
  * every projection is timed over all layers in turn (one weight per layer, 48 x 550 MB, far beyond the 50 MB L2), as a CUDA graph of
    one launch per layer: microseconds per launch from CUDA events over graph replays
  * GB/s from shape-computed bytes (weights + activations + the fp32 partials or the 16-bit output), as a fraction of the 3.35 TB/s
    HBM3 data-sheet figure and of a read ceiling measured in the same run (a bf16 sum over 2 GiB)
  * --sweep: the streaming kernel at every resident CTAs per SM x tile height x K blocks per ring slot, and gemm_tn_kernel at
    CTS_DECODE_SMEM_KB = 75 / 110 / 150
The split factors are cts_gemm_suggest_split's (cts_gemm_fp8_suggest_split's for FP8).  The GPU name, power limit and clocks are read
by a query in the same run (nothing is set).  Writes DIR/bench_decode_gemm.json and prints a table.

    python tools/bench_decode_gemm.py --out DIR [--sweep] [--layers 48] [--reps 5] [--rounds 3]
"""
import argparse
import copy
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
H, I, NQKV, VOCAB = 5120, 13824, 7168, 152064
# name -> (n, k, dual for the split factor); gate_up is the interleaved [2 I, H] weight the decode step streams
PROJ = {"qkv": (NQKV, H, False), "o": (H, H, False), "gate_up": (2 * I, H, True), "down": (H, I, False), "lm_head": (VOCAB, H, False)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def ctx_env(**env):
    """A context of the loaded library created with the given CTS_* variables set (they are read at context creation)."""
    from chatts_b200 import _cabi
    base = _cabi.get_context()
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        h = C.c_void_p()
        if base.lib.cts_ctx_create(base.device, C.byref(h)) != 0:
            raise RuntimeError(f"cts_ctx_create with {env} failed")
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    c = copy.copy(base)
    c.h = h
    return c


def graph_us(launch, count, reps):
    """Microseconds per launch of `launch(i)` for i < count, captured as one CUDA graph and replayed `reps` times."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(min(count, 2)):
            launch(i)                                   # kernel attributes set before the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(count):
            launch(i)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    del g
    return e0.elapsed_time(e1) * 1e3 / (reps * count)


def read_ceiling(gib=2, reps=10):
    x = torch.ones(gib << 29, dtype=torch.bfloat16, device="cuda")
    x.sum()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        x.sum()
    e1.record()
    torch.cuda.synchronize()
    bps = x.numel() * 2 * reps / (e0.elapsed_time(e1) * 1e-3)
    del x
    return bps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--layers", type=int, default=48)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of the default-against-old comparison")
    args = ap.parse_args()
    from chatts_b200 import _cabi
    from chatts_b200._cabi import EPI_NONE, EPI_PARTIAL_F32
    os.makedirs(args.out, exist_ok=True)
    dt = torch.bfloat16
    L = args.layers
    c0 = _cabi.get_context()
    ceiling = read_ceiling()
    res = {"card": card(), "layers": L, "reps": args.reps, "hbm_peak": HBM_PEAK, "read_ceiling_gbs": ceiling / 1e9, "rows": [], "sweep": []}
    print(f"card: {res['card']}   read ceiling (bf16 sum over 2 GiB): {ceiling / 1e9:.0f} GB/s = {ceiling / HBM_PEAK:.3f} of the data sheet", flush=True)

    g = torch.Generator(device="cuda").manual_seed(0)
    W, Q = {}, {}
    for name, (n, k, _) in PROJ.items():
        cnt = 1 if name == "lm_head" else L             # the lm_head alone is 1.56 GB
        W[name] = [torch.empty(n, k, dtype=dt, device="cuda").normal_(0, 0.02, generator=g) for _ in range(cnt)]
        if name != "lm_head":                          # FP8 codes in the fragment-major layout (values do not matter for timing)
            nbytes = -(-n // 256) * (k // 64) * 16384
            Q[name] = [torch.randint(0, 0x7E, (nbytes,), dtype=torch.uint8, device="cuda", generator=g) for _ in range(L)]
    X = {k: torch.randn(32, k, device="cuda", generator=g).to(dt) for k in (H, I)}
    scales = {name: torch.full((n,), 1e-3, device="cuda") for name, (n, _, _) in PROJ.items()}

    def bf16_launcher(c, name, t):
        n, k, dual = PROJ[name]
        x = X[k][:t]
        if name == "lm_head":
            out = torch.empty(t, n, dtype=dt, device="cuda")
            return (lambda i: c.gemm(x, W[name][0], out, epilogue=EPI_NONE)), 8, n * k * 2 + t * k * 2 + t * n * 2, 1
        s = c0.suggest_split(n // 2 if dual else n, k, t, dual)
        out = torch.empty(s, t, n, dtype=torch.float32, device="cuda")
        return (lambda i: c.gemm(x, W[name][i], out, epilogue=EPI_PARTIAL_F32, split_k=s)), L, n * k * 2 + t * k * 2 + s * t * n * 4, s

    def fp8_launcher(name, t):
        n, k, _ = PROJ[name]
        x = X[k][:t]
        s = c0.gemm_fp8_suggest_split(n, k, t)
        out = torch.empty(s, t, n, dtype=torch.float32, device="cuda")
        return (lambda i: c0.gemm_fp8(x, Q[name][i], scales[name], k, out, s)), L, n * k + n * 4 + t * k * 2 + s * t * n * 4, s

    def timed(variant, name, t, launcher):
        fn, count, nbytes, s = launcher
        us = graph_us(fn, count, args.reps)
        return {"variant": variant, "proj": name, "t": t, "split": s, "us": us, "gbs": nbytes / (us * 1e-6) / 1e9,
                "frac_datasheet": nbytes / (us * 1e-6) / HBM_PEAK, "frac_ceiling": nbytes / (us * 1e-6) / ceiling}

    old = ctx_env(CTS_NO_STREAM_GEMM=1)
    ts = (1, 8, 32)
    # ---- the default streaming kernel against gemm_tn_kernel, alternating; the FP8 kernel once per round
    per = {}
    for r in range(args.rounds):
        for t in ts:
            for name in PROJ:
                for variant, launcher in (("stream", lambda: bf16_launcher(c0, name, t)), ("gemm_tn", lambda: bf16_launcher(old, name, t)),
                                          ("fp8", lambda: fp8_launcher(name, t) if name != "lm_head" else None)):
                    la = launcher()
                    if la is None:
                        continue
                    per.setdefault((variant, name, t), []).append(timed(variant, name, t, la))
    print(f"\n{'proj':>8} {'t':>3} {'variant':>8} {'split':>5} {'us (median)':>12} {'min-max':>14} {'GB/s':>7} {'/sheet':>7} {'/ceil':>6}")
    for (variant, name, t), rows in per.items():
        us = [x["us"] for x in rows]
        med = sorted(rows, key=lambda x: x["us"])[len(rows) // 2]
        row = dict(med, us_all=us, us_median=statistics.median(us))
        res["rows"].append(row)
        print(f"{name:>8} {t:>3} {variant:>8} {row['split']:>5} {row['us_median']:>12.1f} {min(us):>6.1f}-{max(us):<7.1f} {row['gbs']:>7.0f} "
              f"{row['frac_datasheet']:>7.3f} {row['frac_ceiling']:>6.3f}", flush=True)

    # ---- whole-step GEMM time at each t: 48 layers x the four projections + the lm_head
    def step_us(variant, t):
        get = {(x["variant"], x["proj"], x["t"]): x["us_median"] for x in res["rows"]}
        return sum(get[(variant, p, t)] * (1 if p == "lm_head" else L) for p in PROJ)
    res["step_gemm_us"] = {v: {t: step_us(v, t) for t in ts} for v in ("stream", "gemm_tn")}
    print("\nGEMM time of one decode step (us):", json.dumps(res["step_gemm_us"]))

    if args.sweep:
        configs = [("gemm_tn", {"CTS_NO_STREAM_GEMM": 1, "CTS_DECODE_SMEM_KB": kb}) for kb in (75, 110, 150)]
        configs += [("stream", {"CTS_STREAM_CTAS": cpsm, "CTS_STREAM_ROWS": rows, "CTS_STREAM_KBLOCKS": kbl})
                    for cpsm in (1, 2, 3) for rows in (64, 128) for kbl in (1, 2, 4)]
        print(f"\n{'kernel':>8} {'setting':>48} " + " ".join(f"{'t=' + str(t) + ' step us':>14}" for t in ts))
        for variant, env in configs:
            try:
                c = ctx_env(**env)
            except RuntimeError as e:
                print(variant, env, e)
                continue
            entry = {"variant": variant, "env": env, "us": {}, "step_us": {}}
            try:
                for t in ts:
                    tot = 0.0
                    for name in PROJ:
                        row = timed(variant, name, t, bf16_launcher(c, name, t))
                        entry["us"][f"{name}@{t}"] = row["us"]
                        tot += row["us"] * (1 if name == "lm_head" else L)
                    entry["step_us"][t] = tot
            except _cabi.CtsError as e:                 # a ring of fewer than two slots: not a valid setting
                entry["error"] = str(e)
            res["sweep"].append(entry)
            print(f"{variant:>8} {json.dumps(env):>48} " + " ".join(f"{entry['step_us'].get(t, float('nan')):>14.0f}" for t in ts)
                  + (f"  ({entry['error'][:60]})" if "error" in entry else ""), flush=True)
    with open(os.path.join(args.out, "bench_decode_gemm.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
