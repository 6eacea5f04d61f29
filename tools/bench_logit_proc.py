"""Logits processors on ChatTS-14B shapes (V = 152 064, synthetic bf16 weights): the two kernels alone, the decode step with processors
off and on, and a continuous-engine round.  Prints one JSON object (and writes it to DIR/bench_logit_proc.json with --out DIR).

    python tools/bench_logit_proc.py [--reps 200] [--skip-model] [--out DIR]

  * kernels: a CUDA graph of --reps cts_logit_proc_apply + cts_logit_proc_update pairs with every processor on in every row (a per-row
    bias row with an allowed-id mask, counts, seen bits, min_tokens stop ids) at batch 1 / 8 / 32; bytes from the shapes (logits read
    and written, bias and counts read) over the measured time;
  * decode step: generate() of bench.py's prompts at batch 1 / 8 / 32, step time = (t(72 tokens) - t(8 tokens)) / 64, processors off
    against presence + frequency + logit_bias + repetition penalty on, alternately, two runs each;
  * engine: one ContinuousEngine round (4 steps) of 8 slots, bench.py's prompt text without its series, with 0, 1 and all 8
    requests penalised, median of 5 rounds.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
V = 152064
PEN = dict(presence_penalty=0.5, frequency_penalty=0.3, repetition_penalty=1.1, logit_bias={100: 2.0, 200: -3.0})


def _gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi failed: {e}"


def _events_ms(fn, n=5):
    ts = []
    for _ in range(n + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts[1:]))


def bench_kernels(reps):
    from chatts_b200 import _cabi
    from chatts_b200.logit_proc import LogitProcState, Processors
    c = _cabi.get_context()
    out = {}
    for B in (1, 8, 32):
        st = LogitProcState(c, B, V, 32768, "cuda")
        p = Processors(presence_penalty=0.5, frequency_penalty=0.3, repetition_penalty=1.1, logit_bias={5: 1.0},
                       allowed_token_ids=list(range(0, V, 2)), min_tokens=10 ** 6)
        for b in range(B):
            st.set_rows([b], p, [151643, 151645], shared_bias=False)
        logits = torch.randn(B, V, device="cuda").bfloat16()
        cur = torch.randint(0, V, (B,), dtype=torch.int32, device="cuda")

        def pair():
            st.apply(logits, B)
            st.update(cur, B)
        pair()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(reps):
                pair()
        g.replay()
        torch.cuda.synchronize()
        us = _events_ms(g.replay, 3) * 1e3 / reps
        nbytes = B * V * (2 + 2 + 4 + 2) + B * ((V + 31) // 32) * 4       # logits read + written, bias, counts, seen
        out[f"b{B}"] = dict(us_per_pair=round(us, 2), mbytes=round(nbytes / 1e6, 2), gbps=round(nbytes / us / 1e3, 1))
    return out


def _gen_ms(model, enc, n, on):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ids = model.generate(**enc, max_new_tokens=n, sync_every=16, ignore_eos=True, **(PEN if on else {}))
    torch.cuda.synchronize()
    assert ids.shape[1] == enc["input_ids"].shape[1] + n
    return (time.perf_counter() - t0) * 1e3


def bench_decode(model, bench, cfg):
    out = {}
    for B in (1, 8, 32):
        enc = bench.make_batch(cfg, B, seed=0)
        for on in (False, True):
            _gen_ms(model, enc, 8, on)
        runs = {"off": [], "on": []}
        for _ in range(2):
            for on in (False, True):
                long_, short = _gen_ms(model, enc, 72, on), _gen_ms(model, enc, 8, on)
                runs["on" if on else "off"].append(round((long_ - short) / 64, 4))
        off = float(np.mean(runs["off"]))
        out[f"b{B}"] = dict(step_ms=runs, overhead_pct=round((np.mean(runs["on"]) / off - 1) * 100, 2),
                            overhead_us=round((np.mean(runs["on"]) - off) * 1e3, 1))
    return out


def bench_engine(model, bench, cfg, slots=8, k=4):
    from chatts_b200.engine import ContinuousEngine
    ids = bench.make_batch(cfg, 1, seed=0)["input_ids"][0]
    ids = ids[(ids < cfg.ts_token_start_index)]                   # the prompt's text ids: one request without series
    out = {}
    for n_pen in (0, 1, slots):
        eng = ContinuousEngine(model, slots=slots, steps_per_round=k)
        for i in range(slots):
            eng.add_request(ids, None, max_new_tokens=200, ignore_eos=True, **(PEN if i < n_pen else {}))
        eng.step()                                           # admission + first round
        times = []
        for _ in range(6):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.step()
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        eng.close()
        out[f"penalised_{n_pen}"] = dict(round_ms=round(float(np.median(times[1:])), 3), steps_per_round=k)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_logit_proc needs an H100")
    res = dict(gpu=_gpu_info(), kernels=bench_kernels(args.reps))
    if not args.skip_model:
        import bench
        from chatts_b200 import ChatTSConfig
        from chatts_b200.model import ChatTSForCausalLM
        cfg = ChatTSConfig.chatts_14b()
        model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, max_batch=32, max_seq_len=1024, page_size=64)
        res["decode"] = bench_decode(model, bench, cfg)
        res["engine"] = bench_engine(model, bench, cfg)
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_logit_proc.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
