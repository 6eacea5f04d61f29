"""Prefix caching on ChatTS-14B (synthetic bf16 weights): prefill and time to first token cold against warm, a three-turn chat through
generate(), and cts_attn_prefill_paged alone against cts_attn_prefill.  Prints one JSON object (and writes it to DIR/bench_prefix_cache.json
with --out DIR).

    python tools/bench_prefix_cache.py [--reps 5] [--skip-model] [--out DIR]

Workloads (bench.py's make_batch series):
  * batch 1, 8 and 32 of the benchmark prompt (8 series + a 64-id question, 576 merged positions): cold = nothing cached; warm = the
    same series with another 64-id question after a call that cached them;
  * config-4-sized prompts (30 series x 512 points) at batch 8, cold and warm;
  * a three-turn chat through generate() (every turn resends the history): prefix caching on against the same calls with the cache
    cleared before each;
  * the kernel alone: 32 x 576 query rows with no prefix, paged against linear (TFLOP/s of the causal attention), and 64 / 576 new rows
    over a 2 464-position prefix.
"""
import argparse
import json
import math
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


def _events(fn, reps):
    """Median ms of fn() over reps, CUDA events, after one warm-up call."""
    fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def _with_question(enc, seed):
    """The same series and ids, the last 64 ids (the question) replaced."""
    ids = enc["input_ids"].clone()
    ids[:, -64:] = torch.from_numpy(np.random.default_rng(seed).integers(0, 150000, (ids.shape[0], 64)))
    return dict(enc, input_ids=ids)


def _prefill(model, enc):
    """One prefill as generate() runs it (cache lookup, allocation, prefill, registration, first token on the host); returns
    (prefill ms by CUDA events, time to first token ms by the host clock, cached positions)."""
    t0 = time.perf_counter()
    _, _, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
    pts, held, keys, cached = model._alloc_prompt(lay, enc["timeseries"], 1)
    try:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        logits = model._prefill(lay, counts, enc["timeseries"], pts, cached=cached)
        b.record()
        model._prefix_register(keys, pts, lay.lens, cached)
        first = logits.argmax(-1).cpu()                      # the first token reaches the host
        ttft = (time.perf_counter() - t0) * 1e3
        torch.cuda.synchronize()
        return a.elapsed_time(b), ttft, int(cached.sum()) if cached is not None else 0, int(lay.lens.sum()), first
    finally:
        model.pool.release(held)


def _cold_warm(model, make, reps):
    cold, warm = [], []
    hit = total = 0
    for r in range(reps):
        model._prefix_clear()
        cold.append(_prefill(model, make(0))[:2])
        p, t, hit, total, _ = _prefill(model, make(1 + r))
        warm.append((p, t))
    c, w = np.median(np.array(cold), 0), np.median(np.array(warm), 0)
    return dict(cold_prefill_ms=float(c[0]), cold_ttft_ms=float(c[1]), warm_prefill_ms=float(w[0]), warm_ttft_ms=float(w[1]),
                warm_hit_positions=hit, positions=total, prefill_speedup=float(c[0] / w[0]))


def _chat(model, bench, cfg, reps):
    """Three turns: turn k's prompt is turn k-1's prompt + its 16 generated ids + a new 64-id question, the same 8 series."""
    enc0 = bench.make_batch(cfg, 1, seed=3)

    def run(clear):
        enc, times = dict(enc0), []
        for turn in range(3):
            if clear:
                model._prefix_clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = model.generate(**enc, max_new_tokens=16, ignore_eos=True)
            times.append((time.perf_counter() - t0) * 1e3)
            q = torch.from_numpy(np.random.default_rng(turn + 10).integers(0, 150000, (1, 64)))
            ids = torch.cat([out, q], 1)
            enc = dict(enc, input_ids=ids, attention_mask=torch.ones_like(ids))
        return times, int(model.last_cached_positions[0])

    run(False)
    cold = np.median([run(True)[0] for _ in range(reps)], 0)
    warm_runs = [run(False) for _ in range(reps)]
    warm = np.median([t for t, _ in warm_runs], 0)
    return dict(cold_turn_ms=[float(x) for x in cold], warm_turn_ms=[float(x) for x in warm], last_turn_hit_positions=warm_runs[-1][1])


def _kernel(reps):
    from chatts_b200 import _cabi
    c = _cabi.get_context()
    nh, nkv, d, page, dt = 40, 8, 128, 64, torch.bfloat16
    scale = 1.0 / math.sqrt(d)
    out = {}

    def paged_case(prefix, q_len, B):
        L = prefix + q_len
        np_ = (L + page - 1) // page
        kc = torch.randn(B * np_ + 1, nkv, page, d, device="cuda", dtype=dt)
        vc = torch.randn_like(kc)
        pt = torch.arange(B * np_, device="cuda", dtype=torch.int32).view(B, np_)
        q = torch.randn(B * q_len, nh * d, device="cuda", dtype=dt)
        o = torch.empty_like(q)
        cu = torch.arange(0, B * q_len + 1, q_len, device="cuda", dtype=torch.int32)
        kvl = torch.full((B,), L, device="cuda", dtype=torch.int32)
        ms = _events(lambda: c.attn_prefill_paged(q, cu, kvl, kc, vc, pt, B, q_len, nh, nkv, d, page, scale, o), reps)
        flops = 4.0 * nh * d * B * sum(prefix + i + 1 for i in range(q_len))
        return ms, flops / ms / 1e9, (q, kc, vc, pt, cu)

    ms_p, tf_p, (q, kc, vc, pt, cu) = paged_case(0, 576, 32)
    k_lin = kc[:32 * 9].permute(0, 2, 1, 3).reshape(-1, nkv * d)[: 32 * 576].contiguous()
    v_lin = vc[:32 * 9].permute(0, 2, 1, 3).reshape(-1, nkv * d)[: 32 * 576].contiguous()
    o = torch.empty_like(q)
    ms_l = _events(lambda: c.attn_prefill(q, k_lin, v_lin, cu, 32, 576, nh, nkv, d, scale, o), reps * 4)
    ms_p = _events(lambda: c.attn_prefill_paged(q, cu, torch.full((32,), 576, device="cuda", dtype=torch.int32), kc, vc, pt, 32, 576, nh,
                                                nkv, d, page, scale, torch.empty_like(q)), reps * 4)
    flops = 4.0 * nh * d * 32 * 576 * 577 / 2
    out["no_prefix_32x576"] = dict(paged_ms=ms_p, paged_tflops=flops / ms_p / 1e9, linear_ms=ms_l, linear_tflops=flops / ms_l / 1e9,
                                   paged_over_linear_time=ms_p / ms_l)
    for q_len in (64, 576):
        ms, tf, _ = paged_case(2464, q_len, 8)
        out[f"prefix2464_q{q_len}_b8"] = dict(ms=ms, tflops=tf)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--out", default=None, help="directory for bench_prefix_cache.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prefix_cache needs an H100")
    res = dict(gpu=_gpu_info(), kernel=_kernel(args.reps))
    if not args.skip_model:
        import bench
        from chatts_b200 import ChatTSConfig
        from chatts_b200.model import ChatTSForCausalLM
        cfg = ChatTSConfig.chatts_14b()
        model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, max_batch=32, max_seq_len=2560, page_size=64, enable_prefix_caching=True)
        for B in (1, 8, 32):
            base = bench.make_batch(cfg, B, seed=0)
            res[f"bench_prompt_b{B}"] = _cold_warm(model, lambda s: base if s == 0 else _with_question(base, s), args.reps)
        big = bench.make_batch(cfg, 8, seed=0, n_series=30, series_len=512)
        res["config4_b8"] = _cold_warm(model, lambda s: big if s == 0 else _with_question(big, s), max(2, args.reps // 2))
        res["chat_3_turns_b1"] = _chat(model, bench, cfg, max(2, args.reps // 2))
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_prefix_cache.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
