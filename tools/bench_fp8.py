#!/usr/bin/env python
"""FP8 weight-only side line of the benchmark (ChatTSForCausalLM.quantize_fp8, vLLM's quantization="fp8"): ChatTS-14B synthetic weights
and bench.py's prompts (8 series x 256 points) at b = 1 / 8 / 32.  In ONE process the bf16 model is timed, then quantize_fp8() is called
on the same model and it is timed again:
  * decode ms/step and tok/s from CUDA events over CUDA-graph replays, greedy agreement of the two token streams
  * prefill seconds at b = 1 and b = 32 (the FP8 model dequantises every projection before its GEMM), generate() end-to-end tok/s
  * resident weight bytes (torch.cuda.memory_allocated around quantize_fp8)
  * per-projection kernel microseconds of cts_gemm_fp8 against cts_gemm(CTS_EPI_PARTIAL_F32) at t = 1 / 8 / 32, each timed over all layers
    in turn so that no weight is served from L2
  * whole-step HBM fraction from shape-computed bytes over the measured step time (3.35 TB/s data-sheet HBM3 bandwidth)
The GPU name and power limit are read by a query in the same run.  Writes DIR/bench_fp8.json and prints it.

    python tools/bench_fp8.py --out DIR [--steps 32] [--layers N]
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
import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def events(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--layers", type=int, default=0, help="truncate the model (0: all 48 layers of ChatTS-14B)")
    args = ap.parse_args()
    from chatts_b200 import ChatTSConfig
    from chatts_b200._cabi import EPI_PARTIAL_F32
    from chatts_b200.model import ChatTSForCausalLM
    os.makedirs(args.out, exist_ok=True)
    cfg = ChatTSConfig.chatts_14b()
    if args.layers:
        cfg.num_hidden_layers = args.layers
    steps, batches = args.steps, (1, 8, 32)
    out = {"card": card(), "steps": steps, "layers": cfg.num_hidden_layers, "by_batch": {}, "kernels_us": {}}
    model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, max_batch=32, max_seq_len=1024, page_size=64)
    c, L, H, I = model.ctx, model.L, model.H, model.I
    encs = {b: bench.make_batch(cfg, b) for b in batches}

    def decode(b):
        enc = encs[b]
        ids_cpu, am_cpu, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
        pts, held = model._alloc_pages(lay.lens, steps + 16)
        try:
            logits = model._prefill(lay, counts, enc["timeseries"], pts)
            st = model._decode_state(b, steps + 16)
            lens32 = torch.from_numpy(lay.lens.astype(np.int32))
            st.page_table.copy_(torch.from_numpy(pts)); st.positions.copy_(lens32 - 1); st.seq_lens.copy_(lens32); st.step_ptr.zero_()
            c.greedy_advance(logits, b, st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.page_table, model.page_size)
            for _ in range(4):
                model._decode_step(st)
            torch.cuda.synchronize()
            ms = events(lambda i: model._decode_step(st), steps)
            return ms, st.out_tokens[:, : int(st.step_ptr[0])].cpu().numpy().copy(), int(lay.lens.max())
        finally:
            model.pool.release(held)

    def prefill(b, reps=3):
        enc = encs[b]
        ids_cpu, am_cpu, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
        pts, held = model._alloc_pages(lay.lens, 0)
        try:
            model._prefill(lay, counts, enc["timeseries"], pts)
            torch.cuda.synchronize()
            return events(lambda i: model._prefill(lay, counts, enc["timeseries"], pts), reps) / 1e3, int(lay.total)
        finally:
            model.pool.release(held)

    def e2e(b, new=64):
        model.generate(**encs[b], max_new_tokens=4, ignore_eos=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.generate(**encs[b], max_new_tokens=new, ignore_eos=True)
        torch.cuda.synchronize()
        return b * new / (time.perf_counter() - t0)

    shapes = dict(qkv=(model._n_qkv, H), o=(H, model.nh * model.d), gu=(2 * I, H), d=(H, I))
    xs = {t: torch.randn(t, max(H, I), device=model.device).to(model.dtype) for t in (1, 8, 32)}
    ws = torch.empty(16 * 32 * 2 * I, device=model.device, dtype=torch.float32)

    def kernels(fp8):
        res = {}
        for kind, (n, k) in shapes.items():
            for t in (1, 8, 32):
                x = xs[t][:, :k]
                if fp8:
                    sp = c.gemm_fp8_suggest_split(n, k, t)
                    f = lambda i: c.gemm_fp8(x, *model.fp8[kind][i % L][:2], k, ws, sp, t=t)
                else:
                    sp = c.suggest_split(n, k, t, kind == "gu")
                    w = {"qkv": model.wqkv, "o": model.wo, "gu": model.wgu, "d": model.wd}[kind]
                    f = lambda i: c.gemm(x, w[i % L], ws, epilogue=EPI_PARTIAL_F32, split_k=sp, t=t)
                for i in range(L):
                    f(i)
                res[f"{kind}_t{t}"] = 1e3 * events(f, 2 * L)
        return res

    # ---------------- bf16
    bf16 = {}
    for b in batches:
        bf16[b] = decode(b)
    pre16 = {b: prefill(b) for b in (1, 32)}
    e2e16 = {b: e2e(b) for b in batches}
    k16 = kernels(False)
    torch.cuda.synchronize()
    mem16 = torch.cuda.memory_allocated()
    # ---------------- FP8, same model
    model.quantize_fp8()
    torch.cuda.synchronize()
    mem8 = torch.cuda.memory_allocated()
    fp8 = {b: decode(b) for b in batches}
    pre8 = {b: prefill(b) for b in (1, 32)}
    e2e8 = {b: e2e(b) for b in batches}
    k8 = kernels(True)
    # bytes a decode step streams (shape-computed): projections (2 B / 1 B + 4 B per row scale), lm_head + final norm 16-bit, KV cache
    proj_elems = sum(n * k for n, k in shapes.values())
    proj_rows = sum(n for n, _ in shapes.values())
    hbm = 3.35e12
    for b in batches:
        (ms16, t16, plen), (ms8, t8, _) = bf16[b], fp8[b]
        n = min(t16.shape[1], t8.shape[1])
        agree = [int(next((i for i in range(n) if t16[r, i] != t8[r, i]), n)) for r in range(b)]
        kv = b * (plen + steps // 2) * L * 2 * model.nkv * model.d * 2
        rest = 2 * H * model.V + kv
        out["by_batch"][str(b)] = {
            "bf16_ms_per_step": ms16, "fp8_ms_per_step": ms8, "decode_speedup": ms16 / ms8,
            "bf16_tok_per_s": b / (ms16 / 1e3), "fp8_tok_per_s": b / (ms8 / 1e3),
            "bf16_step_hbm_frac": (L * proj_elems * 2 + rest) / (ms16 / 1e3) / hbm,
            "fp8_step_hbm_frac": (L * (proj_elems + 4 * proj_rows) + rest) / (ms8 / 1e3) / hbm,
            "greedy_agreement_min_of_%d" % n: int(min(agree)),
            "bf16_generate_tok_per_s": e2e16[b], "fp8_generate_tok_per_s": e2e8[b]}
    for b in (1, 32):
        out["by_batch"][str(b)].update({"prefill_tokens": pre16[b][1], "bf16_prefill_s": pre16[b][0], "fp8_prefill_s": pre8[b][0],
                                        "fp8_over_bf16_prefill": pre8[b][0] / pre16[b][0]})
    out["kernels_us"] = {key: {"cts_gemm_partial": k16[key], "cts_gemm_fp8": k8[key], "speedup": k16[key] / k8[key]} for key in k16}
    out["resident_gb"] = {"bf16_model": mem16 / 1e9, "fp8_model": mem8 / 1e9, "projection_weights_bf16": L * proj_elems * 2 / 1e9,
                          "projection_codes_fp8": L * proj_elems / 1e9}
    line = json.dumps(out)
    open(os.path.join(args.out, "bench_fp8.json"), "w").write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
