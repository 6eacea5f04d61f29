#!/usr/bin/env python
"""Overlapped timeline of ONE decode step inside its CUDA-graph replay (csrc/trace.cuh): ncu serialises kernels and runs them
cold, so it cannot show where the HBM stream idles between the ~440 PDL-chained kernels of a step.  This tool installs the
device-side trace buffer, replays the captured step once, and writes the raw {tag, %globaltimer} records
(gpurun_out/trace_b<B>.npy) plus a per-launch table; `--analyze file.npy` re-runs the analysis offline.

    python tools/trace_decode_step.py --batch 32 [--layers N]        # on the GPU
    python tools/trace_decode_step.py --analyze gpurun_out/trace_b32.npy

The traced replay is a diagnostic run (atomics + timer reads in every CTA): none of its times is a benchmark value."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
KINDS = {1: "gemm", 2: "attn", 3: "norm", 4: "swiglu", 5: "rope", 6: "fused", 7: "other"}


def decode(rec):
    tag = rec[:, 0].astype(np.uint64)
    return dict(kind=(tag >> np.uint64(56)).astype(np.int64) & 0xff, phase=(tag >> np.uint64(52)).astype(np.int64) & 0xf,
                gx=(tag >> np.uint64(40)).astype(np.int64) & 0xfff, gz=(tag >> np.uint64(32)).astype(np.int64) & 0xff,
                sm=(tag >> np.uint64(24)).astype(np.int64) & 0xff, cta=tag.astype(np.int64) & 0xffffff, t=rec[:, 1].astype(np.int64))


def launches(rec, gap_ns=4000):
    """Group the records into kernel launches: per (kind, grid) stream the phase-0 records are walked in time order and a new launch
    opens when a CTA id repeats (the CTAs of ONE grid may enter in several batches, as SM resources are freed by the predecessor)."""
    d = decode(rec)
    out = []
    keys = sorted(set(zip(d["kind"].tolist(), d["gx"].tolist(), d["gz"].tolist())))
    for k in keys:
        m = (d["kind"] == k[0]) & (d["gx"] == k[1]) & (d["gz"] == k[2])
        t, ph, cta = d["t"][m], d["phase"][m], d["cta"][m]
        o = np.argsort(t, kind="stable")
        t, ph, cta = t[o], ph[o], cta[o]
        launch_of = np.zeros(t.shape[0], dtype=np.int64)
        cur = {p_: 0 for p_ in range(16)}
        seen = {p_: set() for p_ in range(16)}
        for i in range(t.shape[0]):
            p_, c = int(ph[i]), int(cta[i])
            if c in seen[p_]:
                cur[p_] += 1
                seen[p_] = set()
            seen[p_].add(c)
            launch_of[i] = cur[p_]
        for j in range(int(launch_of.max()) + 1):
            mm = launch_of == j
            if not (mm & (ph == 0)).any():
                continue
            e = dict(kind=KINDS.get(k[0], str(k[0])), gx=k[1], gz=k[2], enter_first=int(t[mm & (ph == 0)].min()), enter_last=int(t[mm & (ph == 0)].max()))
            for name, p_ in (("wait", 1), ("lastload", 2), ("exit", 3)):
                sel = mm & (ph == p_)
                if sel.any():
                    e[name + "_first"], e[name + "_last"] = int(t[sel].min()), int(t[sel].max())
            e["ctas"] = int((mm & (ph == 0)).sum())
            out.append(e)
    out.sort(key=lambda e: e["enter_first"])
    return out


def report(rec, out=sys.stdout, max_rows=60):
    ls = launches(rec)
    if not ls:
        print("no records", file=out)
        return
    T0 = ls[0]["enter_first"]
    us = lambda v: (v - T0) / 1e3
    print(f"{len(ls)} launches traced, span {us(max(e.get('exit_last', e['enter_last']) for e in ls)):.1f} us", file=out)
    print("  kind    grid     ctas | enter(first..last)  wait released(first..last)  last load issued  exit(last) | stream_us", file=out)
    for e in ls[:max_rows]:
        g = f"({e['gx']},{e['gz']})"
        w = f"{us(e['wait_first']):9.1f}..{us(e['wait_last']):9.1f}" if "wait_first" in e else " " * 20
        ll = f"{us(e['lastload_last']):9.1f}" if "lastload_last" in e else " " * 9
        ex = f"{us(e['exit_last']):9.1f}" if "exit_last" in e else " " * 9
        st = f"{(e['lastload_last'] - e['enter_first']) / 1e3:7.1f}" if "lastload_last" in e else ""
        print(f"  {e['kind']:6s} {g:9s} {e['ctas']:4d} | {us(e['enter_first']):9.1f}..{us(e['enter_last']):9.1f}  {w}  {ll}  {ex} | {st}", file=out)
    # HBM-stream view: the weight streams are the gemm launches [first CTA entered (its TMA prefetch starts) .. last load issued]; attention streams KV
    gem = [e for e in ls if e["kind"] in ("gemm", "fused") and "lastload_last" in e]
    if len(gem) > 8:
        busy = sum(e["lastload_last"] - e["enter_first"] for e in gem)
        span = gem[-1]["lastload_last"] - gem[0]["enter_first"]
        gaps = [(b["enter_first"] - a["lastload_last"]) / 1e3 for a, b in zip(gem[:-1], gem[1:])]
        print(f"weight streams: {len(gem)} GEMM launches, sum of [first entry .. last load issued] {busy / 1e3:.1f} us of a {span / 1e3:.1f} us span "
              f"({busy / span:.3f}); gaps between consecutive streams: mean {np.mean(gaps):.2f} us, median {np.median(gaps):.2f}, max {np.max(gaps):.2f}", file=out)
        # per slot of the layer (period = launches per layer): mean duration and mean gap to the next GEMM
        per = {}
        for a, b in zip(gem[:-1], gem[1:]):
            k = (a["gx"], a["gz"], b["gx"], b["gz"])
            per.setdefault(k, []).append(((a["lastload_last"] - a["enter_first"]) / 1e3, (b["enter_first"] - a["lastload_last"]) / 1e3,
                                          (a["wait_last"] - a["enter_first"]) / 1e3 if "wait_last" in a else float("nan"),
                                          (a.get("exit_last", a["lastload_last"]) - a["lastload_last"]) / 1e3))
        print("  GEMM (grid) -> next GEMM (grid): n, mean stream us, mean idle gap us to the next stream, mean entry->wait-released us, mean lastload->exit us", file=out)
        for k, v in per.items():
            a = np.array(v)
            print(f"  ({k[0]},{k[1]}) -> ({k[2]},{k[3]}): n={len(v):3d} stream {a[:, 0].mean():6.1f}  gap {a[:, 1].mean():6.2f}  wait {a[:, 2].mean():6.2f}  drain {a[:, 3].mean():5.2f}", file=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--layers", type=int, default=0)
    ap.add_argument("--analyze", default=None)
    ap.add_argument("--rows", type=int, default=60)
    a = ap.parse_args()
    if a.analyze:
        report(np.load(a.analyze), max_rows=a.rows)
        return
    import torch
    import bench
    from chatts_b200 import ChatTSConfig
    from chatts_b200.model import ChatTSForCausalLM
    cfg = ChatTSConfig.chatts_14b()
    if a.layers:
        cfg.num_hidden_layers = a.layers
    world, rank, local = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:                     # tensor parallel: every rank runs the step, rank 0 traces its own GPU
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, tp_rank=rank, tp_size=world, max_batch=a.batch, max_seq_len=1024, page_size=64)
    enc = bench.make_batch(cfg, a.batch)
    ids_cpu, am_cpu, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
    pts, held = model._alloc_pages(lay.lens, 64)
    logits = model._prefill(lay, counts, enc["timeseries"], pts)
    st = model._decode_state(a.batch, 64)
    lens32 = torch.from_numpy(lay.lens.astype(np.int32))
    st.page_table.copy_(torch.from_numpy(pts))
    st.positions.copy_(lens32 - 1)
    st.seq_lens.copy_(lens32)
    st.step_ptr.zero_()
    model.ctx.greedy_advance(logits, a.batch, st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.page_table, model.page_size)
    if world > 1:
        dist.barrier()
    for _ in range(6):
        model._decode_step(st)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(8):
        model._decode_step(st)
    e1.record()
    torch.cuda.synchronize()
    if rank == 0:
        print(f"untraced: {e0.elapsed_time(e1) / 8:.3f} ms/step (b={a.batch}, {cfg.num_hidden_layers} layers, tp {world})")
        model.ctx.trace_begin(1 << 20)
    if world > 1:
        dist.barrier()
    e0.record()
    model._decode_step(st)
    e1.record()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    if rank != 0:
        dist.destroy_process_group()
        return
    rec = model.ctx.trace_end()
    print(f"traced replay: {e0.elapsed_time(e1):.3f} ms, {rec.shape[0]} records")
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    tag = f"b{a.batch}" + (f"_L{a.layers}" if a.layers else "") + (f"_tp{world}" if world > 1 else "") + (os.environ.get("TRACE_TAG", ""))
    np.save(os.path.join(ROOT, "gpurun_out", f"trace_{tag}.npy"), rec)
    with open(os.path.join(ROOT, "gpurun_out", f"trace_{tag}.txt"), "w") as f:
        report(rec, out=f, max_rows=a.rows)
    report(rec, max_rows=a.rows)
    model.pool.release(held)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
