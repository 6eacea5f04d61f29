"""Log probabilities on ChatTS-14B (synthetic bf16 weights): cts_logprobs alone, the decode step with logprobs off / 0 / 20, and the
prefill of bench.py's prompt with and without prompt logprobs.  Prints one JSON object (and writes it to DIR/bench_logprobs.json with
--out DIR).

    python tools/bench_logprobs.py [--reps 200] [--skip-model] [--out DIR]

  * kernel: CUDA events around a CUDA graph of --reps launches at rows = 1 / 8 / 32, V = 152 064, k = 0 and 20, bf16; the rate is the logits bytes read
    over the time (the logits of one launch are a few MB, so after the first launch they are likely in L2);
  * decode step: generate() of bench.py's prompts at batch 1 / 8 / 32, step time = (t(72 tokens) - t(8 tokens)) / 64, logprobs off / 0 /
    20 run alternately in one process, two runs each;
  * prompt logprobs: the prefill of the 576-position prompt at batch 1 and 8, with prompt logprobs (k = 20) against without.
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


def _gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi failed: {e}"


def bench_kernel(reps):
    from chatts_b200 import _cabi
    from chatts_b200.logprobs import LogprobBuffers
    c = _cabi.get_context()
    V, out = 152064, {}
    for rows in (1, 8, 32):
        logits = (torch.randn(rows, V, device="cuda") * 4).bfloat16()
        chosen = torch.randint(0, V, (rows, 1), device="cuda", dtype=torch.int32)
        for k in (0, 20):
            buf = LogprobBuffers(c, rows, 1, k, V, "cuda")
            buf.launch(logits, rows, chosen)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()                            # replayed, so the host's launch rate does not bound the time
            with torch.cuda.graph(graph):
                for _ in range(reps):
                    buf.launch(logits, rows, chosen)
            graph.replay()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graph.replay()
            b.record()
            torch.cuda.synchronize()
            us = a.elapsed_time(b) * 1e3 / reps
            out[f"rows{rows}_k{k}"] = dict(us=round(us, 2), logits_GBps=round(rows * V * 2 / (us * 1e-6) / 1e9, 1))
    return out


def _gen_ms(model, enc, n, lp):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model.generate(**enc, max_new_tokens=n, ignore_eos=True, logprobs=lp, sync_every=16)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def bench_decode(model, bench, cfg):
    out = {}
    for B in (1, 8, 32):
        enc = bench.make_batch(cfg, B, seed=0)
        for lp in (None, 0, 20):                                      # warm-up: graph capture, buffers
            _gen_ms(model, enc, 8, lp)
        runs = {str(lp): [] for lp in (None, 0, 20)}
        for _ in range(2):
            for lp in (None, 0, 20):
                long_, short = _gen_ms(model, enc, 72, lp), _gen_ms(model, enc, 8, lp)
                runs[str(lp)].append(round((long_ - short) / 64, 4))
        off = float(np.mean(runs["None"]))
        out[f"b{B}"] = dict(step_ms=runs, overhead_k0_pct=round((np.mean(runs["0"]) / off - 1) * 100, 2),
                            overhead_k20_pct=round((np.mean(runs["20"]) / off - 1) * 100, 2),
                            overhead_k20_us=round((np.mean(runs["20"]) - off) * 1e3, 1))
    return out


def bench_prompt(model, bench, cfg, reps):
    out = {}
    for B in (1, 8):
        enc = bench.make_batch(cfg, B, seed=0)
        _, _, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
        pts, held = model._alloc_pages(lay.lens, 1)
        try:
            res = {}
            for _ in range(2):
                for k in (None, 20):
                    ts = []
                    for _ in range(reps + 1):
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        model._prefill(lay, counts, enc["timeseries"], pts, prompt_lp=k)
                        b.record()
                        torch.cuda.synchronize()
                        ts.append(a.elapsed_time(b))
                    res.setdefault(str(k), []).append(round(float(np.median(ts[1:])), 3))
            out[f"b{B}"] = dict(prefill_ms=res, positions=int(lay.lens.sum()))
        finally:
            model.pool.release(held)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_logprobs needs an H100")
    res = dict(gpu=_gpu_info(), kernel=bench_kernel(args.reps))
    if not args.skip_model:
        import bench
        from chatts_b200 import ChatTSConfig
        from chatts_b200.model import ChatTSForCausalLM
        cfg = ChatTSConfig.chatts_14b()
        model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, max_batch=32, max_seq_len=1024, page_size=64)
        res["decode"] = bench_decode(model, bench, cfg)
        res["prompt_logprobs"] = bench_prompt(model, bench, cfg, 5)
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_logprobs.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
