"""cts_sample_advance alone on ChatTS-14B's vocabulary (V = 152 064, bf16 logits): a CUDA graph of --reps launches at batch 1 / 8 / 32,
one step each, for the sampling settings the reference uses (temperature 0.2, top_p 1.0 and 0.9) and a top-k one.  Prints one JSON
object (and writes it to DIR/bench_sampling.json with --out DIR), with the card's name and power limit read in the same call.

    python tools/bench_sampling.py [--reps 200] [--baseline LIB] [--out DIR]

--baseline LIB: another build of libchatts_b200.so (for instance the parent commit's) timed in the same process, alternating with the
in-tree library round by round; the tokens both libraries draw over the timed steps are compared as well.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
V = 152064
SETTINGS = {"t0.2": (0.2, 0, 1.0), "t0.2_p0.9": (0.2, 0, 0.9), "t1_k50": (1.0, 50, 1.0)}


def _gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi failed: {e}"


class Sampler:
    """cts_sample_advance of one library through its own context."""

    def __init__(self, path):
        vp, i, ll, f = C.c_void_p, C.c_int, C.c_longlong, C.c_float
        self.lib = C.CDLL(path)
        self.lib.cts_ctx_create.argtypes = [i, C.POINTER(vp)]
        self.lib.cts_ctx_create.restype = i
        self.lib.cts_last_error.argtypes = [vp]
        self.lib.cts_last_error.restype = C.c_char_p
        self.lib.cts_sample_advance.argtypes = [vp, vp, ll, i, f, i, f, C.c_ulonglong, vp, i, vp, vp, vp, vp, vp, vp, i, i, i, vp]
        self.lib.cts_sample_advance.restype = i
        self.h = vp()
        if self.lib.cts_ctx_create(torch.cuda.current_device(), C.byref(self.h)) != 0:
            raise RuntimeError(f"cts_ctx_create failed for {path}")

    def __call__(self, logits, B, temp, top_k, top_p, out, step_ptr, cur):
        rc = self.lib.cts_sample_advance(self.h, logits.data_ptr(), V, B, temp, top_k, top_p, 1234, out.data_ptr(), out.stride(0),
                                         step_ptr.data_ptr(), cur.data_ptr(), None, None, None, None, 0, 16, 0,
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError(self.lib.cts_last_error(self.h).decode())


def _graph(sampler, logits, B, setting, reps):
    temp, top_k, top_p = SETTINGS[setting]
    out = torch.full((B, reps), -1, dtype=torch.int32, device="cuda")
    sp = torch.zeros(2, dtype=torch.int32, device="cuda")
    cur = torch.zeros(B, dtype=torch.int32, device="cuda")
    sampler(logits, B, temp, top_k, top_p, out, sp, cur)                  # warm-up, outside the graph
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            sampler(logits, B, temp, top_k, top_p, out, sp, cur)

    def run():
        sp.zero_()
        g.replay()
    return run, out


def _time_us(run, reps, n=5):
    ts = []
    for _ in range(n + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / reps)
    return ts[1:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--baseline", default=None, help="another libchatts_b200.so to time against the in-tree one")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling needs an H100")
    from chatts_b200 import _cabi
    libs = {"new": Sampler(_cabi.LIB_PATH)}
    if args.baseline:
        libs["old"] = Sampler(os.path.abspath(args.baseline))
    res = dict(gpu=_gpu_info(), vocab=V, reps=args.reps, us_per_launch={})
    g = torch.Generator().manual_seed(0)
    row = torch.randn(V, generator=g) * 3
    for B in (1, 8, 32):
        logits = row[None].repeat(B, 1).to(torch.bfloat16).cuda()
        for setting in SETTINGS:
            runs = {name: _graph(s, logits, B, setting, args.reps) for name, s in libs.items()}
            times = {name: [] for name in libs}
            for r in range(args.rounds):                                   # alternate the libraries round by round
                for name in (list(libs) if r % 2 == 0 else list(libs)[::-1]):
                    times[name] += _time_us(runs[name][0], args.reps)
            entry = {name: round(float(np.median(t)), 2) for name, t in times.items()}
            if "old" in runs:
                a, b = runs["new"][1].cpu(), runs["old"][1].cpu()
                entry["same_tokens"] = round(float((a == b).float().mean()), 5)
                entry["new_over_old"] = round(entry["new"] / entry["old"], 3)
            res["us_per_launch"][f"b{B}_{setting}"] = entry
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sampling.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
