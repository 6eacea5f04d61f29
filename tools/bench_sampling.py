"""cts_sample_advance alone on ChatTS-14B's vocabulary (V = 152 064, bf16 logits): a CUDA graph of --reps launches at batch 1 / 8 / 32,
one step each, for the sampling settings the reference uses (temperature 0.2, top_p 1.0 and 0.9) and a top-k one.  Prints one JSON
object (and writes it to DIR/bench_sampling.json with --out DIR), with the card's name and power limit read in the same call.

    python tools/bench_sampling.py [--reps 200] [--baseline LIB] [--engine] [--out DIR]

--baseline LIB: another build of libchatts_b200.so (for instance the parent commit's) timed in the same process, alternating with the
in-tree library round by round; the tokens both libraries draw over the timed steps are compared as well.

The same call times cts_sample_advance_rows against cts_sample_advance with uniform parameters (draw_key = row, draw_step = step, so
both draw the same tokens), alternating round by round, and one mixed launch: half the rows greedy, half at temperature 0.7 with
top_p 0.9.  --engine adds continuous-engine rounds (8 slots, 4 steps per round, ChatTS-14B with synthetic bf16 weights, bench.py's
prompts) with 0, 1 and 8 slots sampling at temperature 0.7 / top_p 0.9.
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


def _rows_graph(logits, B, temps, top_ks, top_ps, reps):
    """cts_sample_advance_rows of the in-tree library (seed 1234 on every row, draw_key = row, draw_step = step_ptr[0]), as _graph."""
    from chatts_b200 import _cabi
    c = _cabi.get_context()
    dev = dict(device="cuda")
    prm = [torch.tensor(temps, dtype=torch.float32, **dev), torch.tensor(top_ks, dtype=torch.int32, **dev),
           torch.tensor(top_ps, dtype=torch.float32, **dev), torch.full((B,), 1234, dtype=torch.int64, **dev),
           torch.arange(B, dtype=torch.int32, **dev)]
    step = torch.zeros(B, dtype=torch.int32, **dev)
    out = torch.full((B, reps), -1, dtype=torch.int32, **dev)
    sp = torch.zeros(2, dtype=torch.int32, **dev)
    cur = torch.zeros(B, dtype=torch.int32, **dev)
    launch = lambda: c.sample_advance_rows(logits, B, *prm, step, out, sp, cur, None, None, None, None, 16)
    launch()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            launch()

    def run():
        sp.zero_()
        step.zero_()
        g.replay()
    return run, out


def _engine_rounds(rounds=10, cycles=2):
    """ms per continuous-engine round (4 decode steps of 8 slots) with 0, 1 and 8 slots sampling, the configurations alternated."""
    import time
    sys.path.insert(0, ROOT)
    from bench import make_batch
    from chatts_b200.config import ChatTSConfig
    from chatts_b200.engine import ContinuousEngine
    from chatts_b200.model import ChatTSForCausalLM
    cfg = ChatTSConfig.chatts_14b()
    model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, max_batch=8, max_seq_len=1024, page_size=64)
    enc = make_batch(cfg, 8)
    per = enc["timeseries"].shape[0] // 8
    out = {n: [] for n in (0, 1, 8)}
    for _ in range(cycles):
        for n in out:
            eng = ContinuousEngine(model, slots=8, steps_per_round=4, max_prefill_batch=8)
            for b in range(8):
                kw = dict(temperature=0.7, top_p=0.9, seed=b) if b < n else {}
                eng.add_request(enc["input_ids"][b], enc["timeseries"][b * per:(b + 1) * per], max_new_tokens=4 * (rounds + 3),
                                ignore_eos=True, **kw)
            eng.step()                                                     # admission + one round
            eng.step()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(rounds):
                eng.step()                                                 # ends in the round's device->host read of the tokens
            out[n].append((time.perf_counter() - t0) * 1e3 / rounds)
            assert len(eng.active) == 8
            eng.close()
    return {f"{n}_sampling": dict(ms_per_round=round(float(np.median(t)), 3), ms_per_step=round(float(np.median(t)) / 4, 3),
                                  all_cycles=[round(x, 3) for x in t]) for n, t in out.items()}


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
    ap.add_argument("--engine", action="store_true", help="also time continuous-engine rounds on ChatTS-14B")
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
            # the per-row kernel with the same parameters on every row, alternating with the scalar entry
            temp, top_k, top_p = SETTINGS[setting]
            rows = _rows_graph(logits, B, [temp] * B, [top_k] * B, [top_p] * B, args.reps)
            rt = {"scalar": [], "rows": []}
            for r in range(args.rounds):
                for name in (("scalar", "rows") if r % 2 == 0 else ("rows", "scalar")):
                    rt[name] += _time_us(runs["new"][0] if name == "scalar" else rows[0], args.reps)
            ent = {k: round(float(np.median(v)), 2) for k, v in rt.items()}
            ent["same_tokens"] = round(float((rows[1].cpu() == runs["new"][1].cpu()).float().mean()), 5)
            ent["rows_over_scalar"] = round(ent["rows"] / ent["scalar"], 3)
            res.setdefault("rows_vs_scalar_us", {})[f"b{B}_{setting}"] = ent
        if B > 1:
            h = B // 2
            mixed = _rows_graph(logits, B, [0.0] * h + [0.7] * (B - h), [0] * B, [1.0] * h + [0.9] * (B - h), args.reps)
            mt = []
            for _ in range(args.rounds):
                mt += _time_us(mixed[0], args.reps)
            res.setdefault("mixed_half_greedy_half_t0.7_p0.9_us", {})[f"b{B}"] = round(float(np.median(mt)), 2)
    if args.engine:
        res["engine_round"] = _engine_rounds()
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sampling.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
