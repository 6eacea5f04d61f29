"""Beam search on ChatTS-14B shapes (synthetic bf16 weights, bench.py's prompts: 8 series + 64 prompt ids each).  Prints one JSON object
(and writes it to DIR/bench_beam.json with --out DIR).

    python tools/bench_beam.py [--reps 200] [--out DIR]

  * step: generate(num_beams=4) of 1 and 8 prompts (4 and 32 beam rows) against a greedy generate() of 4 and 32 prompts, step time =
    (t(40 tokens) - t(8 tokens)) / 32, ignore_eos so every step runs, alternately, two runs each;
  * select + fork: cts_beam_select + cts_beam_fork_kv alone at 1 x 4 and 8 x 4 rows, a CUDA graph of --reps launch pairs, with every
    row the child of another row at tail offsets page_size - 1 (the most bytes a fork can move: the bound), CUDA events;
  * fork bytes: forked rows x (page_size - 1) x layers x 2 x nkv x head_dim x 2 bytes, computed from the shapes, and the rate over the
    measured select + fork time;
  * end to end: generate(num_beams=4, max_new_tokens=40) wall time.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _gen_ms(model, enc, n, nb):
    kw = dict(num_beams=nb, num_return_sequences=1) if nb > 1 else {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model.generate(**enc, max_new_tokens=n, sync_every=16, ignore_eos=True, **kw)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def bench_steps(model, bench, cfg):
    out = {}
    for B in (1, 8):
        beam_enc, greedy_enc = bench.make_batch(cfg, B, seed=0), bench.make_batch(cfg, 4 * B, seed=0)
        _gen_ms(model, beam_enc, 8, 4), _gen_ms(model, greedy_enc, 8, 1)
        runs = {"beam": [], "greedy": [], "beam_e2e_40": []}
        for _ in range(2):
            long_, short = _gen_ms(model, beam_enc, 40, 4), _gen_ms(model, beam_enc, 8, 4)
            runs["beam"].append(round((long_ - short) / 32, 4))
            runs["beam_e2e_40"].append(round(long_, 2))
            long_, short = _gen_ms(model, greedy_enc, 40, 1), _gen_ms(model, greedy_enc, 8, 1)
            runs["greedy"].append(round((long_ - short) / 32, 4))
        out[f"{B}x4"] = dict(step_ms=runs, rows=4 * B, overhead_pct=round((np.mean(runs["beam"]) / np.mean(runs["greedy"]) - 1) * 100, 2))
    return out


def bench_select_fork(model, reps):
    from chatts_b200 import beam as beammod
    c, dev, ps, L, nkv, d = model.ctx, model.device, model.page_size, model.L, model.nkv, model.d
    out = {}
    for B in (1, 8):
        nb, keep, V, max_new = 4, 8, model.config.vocab_size, reps + 2
        R, MP = B * nb, model.max_pages
        g = torch.Generator(device=dev).manual_seed(0)
        cand_ids = torch.stack([torch.randperm(V, device=dev, generator=g)[:keep] for _ in range(R)]).int()
        cand_lp = -torch.rand(R, keep, device=dev, generator=g).sort(1, descending=False).values
        own = torch.arange(R * MP, device=dev, dtype=torch.int32).view(R, MP) % (model.kv.shape[2] - R) + R
        spare = torch.arange(R, device=dev, dtype=torch.int32)
        table = own.clone()
        # position ps - 2 before the step: every selected row lands at offset ps - 1 of its tail, the largest copy a fork makes
        pos = torch.full((R,), ps - 2, dtype=torch.int32, device=dev)
        state = dict(run=torch.zeros(R, device=dev), fin=torch.full((R,), -1e9, device=dev), info=torch.zeros(R, 4, dtype=torch.int32, device=dev),
                     flags=torch.zeros(B, 2, dtype=torch.int32, device=dev), step=torch.zeros(2, dtype=torch.int32, device=dev),
                     bp_tok=torch.zeros(max_new, R, dtype=torch.int32, device=dev), bp_par=torch.zeros(max_new, R, dtype=torch.int32, device=dev),
                     cur=torch.zeros(R, dtype=torch.int32, device=dev), sl=torch.zeros(R, dtype=torch.int32, device=dev),
                     slot=torch.zeros(R, dtype=torch.int32, device=dev), old=torch.zeros_like(table), fork=torch.zeros(R, 3, dtype=torch.int32, device=dev))
        den = torch.from_numpy(beammod.len_den(max_new, 1.0)).to(dev)
        eos = torch.tensor([V - 1], dtype=torch.int32, device=dev)
        p = torch.zeros(R, dtype=torch.int32, device=dev)
        fresh = torch.tensor([1, 0], dtype=torch.int32, device=dev).repeat(B, 1)

        def pair():
            p.copy_(pos)                                           # every replay forks from the same offset
            state["flags"].copy_(fresh)                            # and runs the finished-set merge and the heuristic (not done)
            c.beam_select(B, nb, keep, V, cand_ids, cand_lp, eos, den, max_new, False, 1.0, state["run"], state["fin"], state["info"],
                          state["flags"], state["step"], state["bp_tok"], state["bp_par"], state["cur"], p, state["sl"], state["slot"],
                          table, state["old"], own, spare, ps, state["fork"])
            c.beam_fork_kv(model.kv, state["fork"], R)
        pair()
        torch.cuda.synchronize()
        forked = int((state["fork"][:, 2] > 0).sum())
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            pair()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        state["step"].zero_()
        with torch.cuda.graph(graph):
            for _ in range(reps):
                pair()
        times = []
        for _ in range(5):
            state["step"].zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / reps * 1e3)
        us = float(np.median(times))
        fork_bytes = forked * (ps - 1) * L * 2 * nkv * d * 2
        out[f"{B}x4"] = dict(select_fork_us=round(us, 2), forked_rows=forked, fork_bytes_from_shapes=fork_bytes,
                             fork_rate_GBps=round(fork_bytes / (us * 1e-6) / 1e9, 1), includes="a reset of the positions and the prompt flags per pair")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_beam needs an H100")
    from bench_structured import _gpu_info
    import bench
    from chatts_b200 import ChatTSConfig
    from chatts_b200.model import ChatTSForCausalLM
    cfg = ChatTSConfig.chatts_14b()
    model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, max_batch=32, max_seq_len=1024, page_size=64)
    res = dict(gpu=_gpu_info(), select_fork=bench_select_fork(model, args.reps), steps=bench_steps(model, bench, cfg), gpu_after=_gpu_info())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_beam.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
