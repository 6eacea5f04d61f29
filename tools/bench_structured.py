"""Structured outputs on ChatTS-14B shapes (V = 152 064, synthetic bf16 weights): the one-time mask build, the per-step kernels, and the
decode step with and without a constraint.  Prints one JSON object (and writes it to DIR/bench_structured.json with --out DIR).

    python tools/bench_structured.py [--reps 200] [--skip-model] [--out DIR]

  * mask_build: cts_struct_mask_build at V = 152 064 over a synthetic vocabulary of random 1-8-byte printable-ASCII tokens (a stand-in
    for a byte-level BPE vocabulary: no tokenizer is downloaded), for a 10-way choice and the regexes below; CUDA events, median of 5;
  * per step: cts_struct_mask_apply + cts_struct_advance at batch 1 / 8 / 32, CUDA events around a CUDA graph of --reps pairs;
  * decode step: generate() of bench.py's prompts at batch 1 / 8 / 32, step time = (t(72 tokens) - t(8 tokens)) / 64, unconstrained
    (ignore_eos) against the regex [a-z ]{80,} (whose first stop is past the 72nd token), alternately, two runs each.
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
REGEXES = [r"\d{1,3}(\.\d+)?", r"(yes|no)", r"col: \d+(; col: \d+)*", r"[a-z ]{80,}"]
CHOICE = ["increase", "decrease", "steady", "fluctuating", "periodic", "spike", "drop", "trend up", "trend down", "no change"]


def _gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi failed: {e}"


def _vocab(seed=0):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 9, size=V)
    offsets = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    data = rng.integers(32, 127, size=int(offsets[-1])).astype(np.uint8)
    data[rng.random(len(data)) < 0.3] = rng.integers(48, 58, size=1)          # digits more often, so numeric patterns have many tokens
    return torch.from_numpy(offsets).cuda(), torch.from_numpy(data).cuda()


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
    from chatts_b200 import structured as so
    c = _cabi.get_context()
    off, data = _vocab()
    stops = torch.tensor([151643, 151645], dtype=torch.int32, device="cuda")
    build, autos = {}, {}
    for name, params in [("choice10", so.StructuredOutputsParams(choice=CHOICE))] + [(r, so.StructuredOutputsParams(regex=r)) for r in REGEXES]:
        dfa = so.compile_params(params)
        auto = so.DeviceAutomaton(c, dfa, off, data, stops, V, "cuda")
        ms = _events_ms(lambda: c.struct_mask_build(auto.trans, auto.accept, off, data, stops, auto.allowed))
        n0 = int(np.unpackbits(auto.allowed[0].cpu().numpy().view(np.uint8)).sum())
        build[name] = dict(states=dfa.num_states, ms=round(ms, 3), allowed_at_start=n0)
        autos[name] = auto
    step = {}
    auto = autos[r"[a-z ]{80,}"]
    for B in (1, 8, 32):
        logits = torch.randn(B, V, device="cuda").bfloat16()
        state = torch.zeros(B, dtype=torch.int32, device="cuda")
        cur = torch.full((B,), ord("a"), dtype=torch.int32, device="cuda")

        def pair():
            auto.mask_apply(c, logits, B, state)
            auto.advance(c, cur, B, state)
        pair()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(reps):
                pair()
        g.replay()
        torch.cuda.synchronize()
        step[f"b{B}"] = dict(us_per_step=round(_events_ms(g.replay, 3) * 1e3 / reps, 2))
    return dict(mask_build=build, per_step=step)


def _gen_ms(model, enc, n, constrained):
    kw = dict(structured_outputs={"regex": r"[a-z ]{80,}"}) if constrained else dict(ignore_eos=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ids = model.generate(**enc, max_new_tokens=n, sync_every=16, **kw)
    torch.cuda.synchronize()
    assert ids.shape[1] == enc["input_ids"].shape[1] + n
    return (time.perf_counter() - t0) * 1e3


def bench_decode(model, bench, cfg):
    out = {}
    for B in (1, 8, 32):
        enc = bench.make_batch(cfg, B, seed=0)
        for con in (False, True):
            _gen_ms(model, enc, 8, con)
        runs = {"off": [], "regex": []}
        for _ in range(2):
            for con in (False, True):
                long_, short = _gen_ms(model, enc, 72, con), _gen_ms(model, enc, 8, con)
                runs["regex" if con else "off"].append(round((long_ - short) / 64, 4))
        off = float(np.mean(runs["off"]))
        out[f"b{B}"] = dict(step_ms=runs, overhead_pct=round((np.mean(runs["regex"]) / off - 1) * 100, 2),
                            overhead_us=round((np.mean(runs["regex"]) - off) * 1e3, 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_structured needs an H100")
    res = dict(gpu=_gpu_info(), **bench_kernels(args.reps))
    if not args.skip_model:
        import bench
        from chatts_b200 import ChatTSConfig
        from chatts_b200.model import ChatTSForCausalLM
        cfg = ChatTSConfig.chatts_14b()
        model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, max_batch=32, max_seq_len=1024, page_size=64)
        res["decode"] = bench_decode(model, bench, cfg)
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_structured.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
