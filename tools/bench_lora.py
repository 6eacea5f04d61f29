#!/usr/bin/env python
"""bench_lora.py -- BASELINE config 5: ChatTS-8B LoRA fine-tune step (forward + backward + clip + AdamW) on N GPUs,
data parallel.  Same measurement contract as bench.py (one JSON line on rank 0; CUDA events; barrier + synchronize on
both sides; max over ranks; clocks sampled during the timed region), for the SECOND workload of the hot path -- bench.py
itself stays on the headline decode metric.

    python tools/bench_lora.py [--steps K] [--warmup W] [--samples S]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 --master-port 29511 \
        tools/bench_lora.py --gpus 4

A "step" = LoraTrainer.train_step on one synthetic QA micro-batch per rank: S samples (default 16), each 4 series x 256
points (4 x (46 prefix ids + <ts> + 16 patch rows + <ts/>) = 256 merged positions) + 64 prompt ids + 128 answer ids = 448
positions, labels on the 128 answer ids (chatts/align/uts_template_qa.py:127-131 record shape).  ChatTS-8B = Qwen3-8B
shape + TS encoder, synthetic bf16 weights, LoRA r=16 / alpha=32 on q,k,v,o,gate,up,down.  Weak scaling: every rank
takes its own S samples, gradients meet in ONE all-reduce of the fp32 arena.  `value` = merged positions of all ranks per
second with the series tensor already in HBM; `e2e` = the same through train_step with pinned HOST tensors and the loss
read back every step.  Roofline: tensor cores -- 4 flop per frozen decoder parameter and position (forward 2, input
gradient 2; the frozen weights take no weight gradient) + attention, against the measured bf16 peak.
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
from bench import ClockSampler, make_series  # noqa: E402

N_SERIES, SERIES_LEN, PREFIX_IDS, PROMPT_IDS, ANSWER_IDS = 4, 256, 46, 64, 128


def make_records_batch(cfg, samples, seed):
    """Token-id level records (no tokenizer offline): input = 4 x (prefix ids, <ts>, <ts/>) + prompt ids; output = answer ids."""
    from chatts_b200.processor import sp_encoding
    rng = np.random.default_rng(seed)
    ids, lab, series = [], [], []
    for b in range(samples):
        row = []
        for k in range(N_SERIES):
            row += rng.integers(0, 150000, PREFIX_IDS).tolist() + [cfg.ts_token_start_index, cfg.ts_token_start_index + 1]
            series.append(sp_encoding(make_series(seed * 1000 + b, k))[0])
        row += rng.integers(0, 150000, PROMPT_IDS).tolist()
        ans = rng.integers(0, 150000, ANSWER_IDS).tolist()
        ids.append(row + ans)
        lab.append([-100] * len(row) + ans)
    ids = torch.tensor(ids, dtype=torch.long)
    return {"input_ids": ids, "attention_mask": torch.ones_like(ids), "labels": torch.tensor(lab, dtype=torch.long),
            "timeseries": torch.from_numpy(np.stack(series)).to(torch.float32)}


def tensor_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return float(d.get("bf16_tflops_sustained", d["bf16_tflops"])), "measured (MEASURED_PEAKS.json, sustained cuBLAS bf16)"
    return 989.0, "H100 SXM data sheet (dense bf16)"


def step_flops(cfg, positions, label_rows, lens):
    per_layer = (cfg.hidden_size * (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * cfg.head_dim +
                 cfg.hidden_size * cfg.num_attention_heads * cfg.head_dim + 3 * cfg.hidden_size * cfg.intermediate_size)
    dec = cfg.num_hidden_layers * per_layer
    gemm = 4.0 * dec * positions + 4.0 * cfg.hidden_size * cfg.vocab_size * label_rows
    # causal attention: forward 4 S^2/2 d nh per layer; backward 2.5x (dQ, dK, dV, dP + recomputed S)
    attn = sum(3.5 * 4 * (s * s / 2) * cfg.head_dim * cfg.num_attention_heads for s in lens) * cfg.num_hidden_layers
    return gemm + attn


def run(args):
    import torch.distributed as dist
    from chatts_b200 import ChatTSConfig, _cabi
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.train import LoraTrainer

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    cfg = ChatTSConfig.chatts_8b()
    if args.layers:
        cfg.num_hidden_layers = args.layers
    model = ChatTSForCausalLM.from_synthetic(cfg, seed=1234, max_batch=1, max_seq_len=1024, page_size=64, use_cuda_graph=False)
    tr = LoraTrainer(model, r=16, lora_alpha=32, lr=1e-4, max_grad_norm=1.0, seed=rank)
    host = make_records_batch(cfg, args.samples, seed=rank + 1)
    dev = dict(host)
    dev["timeseries"] = host["timeseries"].to("cuda", torch.bfloat16)
    pinned = {k: v.pin_memory() for k, v in host.items()}

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    def timed(batch, steps, read_loss):
        sync_all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = model.ctx.launches
        t0 = time.perf_counter()
        e0.record()
        loss = None
        for _ in range(steps):
            loss = tr.train_step(batch)
            if read_loss:
                loss = float(loss[0])                    # D2H of the step's result
        e1.record()
        torch.cuda.synchronize()
        ms, wall = e0.elapsed_time(e1), time.perf_counter() - t0
        if world > 1:
            t = torch.tensor([ms, wall], device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms, wall = float(t[0]), float(t[1])
        return ms, wall, model.ctx.launches - l0, float(loss if read_loss else loss[0])

    with ClockSampler(local) as clk:
        for _ in range(max(args.warmup, 3)):
            tr.train_step(dev)
        ms, _, launches, loss = timed(dev, args.steps, False)
        _, wall, _, loss_e2e = timed(pinned, args.steps, True)
    clocks = clk.summary()
    S = host["input_ids"].shape[1] + N_SERIES * (SERIES_LEN // 16)
    positions = args.samples * S
    label_rows = args.samples * ANSWER_IDS
    flops = step_flops(cfg, positions, label_rows, [S] * args.samples)
    peak, src = tensor_peak()
    ach = flops / (ms / args.steps * 1e-3) / 1e12
    if rank == 0:
        h2d = sum(v.numel() * v.element_size() for k, v in host.items() if k != "timeseries") // 2 + host["timeseries"].numel() * 4
        line = {"metric": "lora_finetune_positions_per_s", "value": world * positions * args.steps / (ms / 1e3), "unit": "tokens/s",
                "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps,
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
                "config": {"workload": (f"ChatTS-8B (Qwen3-8B shape + TS encoder, synthetic bf16 weights) LoRA r=16 fine-tune step "
                                        f"(forward+backward+clip+AdamW), {args.samples} samples/GPU x {S} merged positions "
                                        f"({N_SERIES} series x {SERIES_LEN} points, {PROMPT_IDS} prompt ids, {ANSWER_IDS} answer ids with labels)"),
                           "samples_per_gpu": args.samples, "positions_per_gpu": positions, "parallelism": f"dp{world}",
                           "l2_policy": "inputs larger than L2: 16 GB of frozen weights + 15 GB of transposed copies streamed per step"},
                "clocks": clocks, "gpu_launches": int(launches), "loss": loss,
                "e2e": {"value": world * positions * args.steps / wall, "unit": "tokens/s", "h2d_bytes_per_step": int(h2d),
                        "d2h_bytes_per_step": 4, "loss": loss_e2e,
                        "definition": "train_step(pinned host tensors): H2D of ids/labels maps and series, TS encode, forward, backward, "
                                      "all-reduce, clip, AdamW, pack; loss read back every step"},
                "roofline": {"bound": "tensor", "achieved": ach, "peak": peak, "unit": "TFLOP/s", "frac": ach / peak, "traffic": None,
                             "algorithmic_flops_per_step": flops, "peak_source": src},
                "arch": model.ctx.arch, "lib": os.path.relpath(_cabi.LIB_PATH, ROOT)}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_reference(args):
    """CPU arm for config 5: what the external recipe executes on a host -- stock transformers Qwen3ForCausalLM at the ChatTS-8B
    layer shape with peft-style LoRA modules around its seven projections (peft itself is not installed: the same
    `base(x) + B(A(x)) * alpha/r` wrapper the oracle tests use), forward + backward + AdamW on ONE synthetic sample of 448
    positions.  Bounded sample: `layers_sample` decoder layers are instantiated and timed, the per-layer time is scaled to 36
    layers (embedding / lm_head / loss timed with 0 layers and added once)."""
    import torch.nn as nn
    from transformers import Qwen3Config, Qwen3ForCausalLM
    if int(os.environ.get("RANK", "0")) != 0:
        return
    threads = os.cpu_count() or 1
    torch.set_num_threads(threads)
    S = N_SERIES * (PREFIX_IDS + 2 + SERIES_LEN // 16) + PROMPT_IDS + ANSWER_IDS
    full_layers, layers_sample = 36, 2

    class LoRALinear(nn.Module):
        def __init__(self, base, r=16, alpha=32):
            super().__init__()
            self.base, self.scaling = base, alpha / r
            self.lora_A = nn.Parameter(torch.randn(r, base.in_features, dtype=base.weight.dtype) * 0.01)
            self.lora_B = nn.Parameter(torch.zeros(base.out_features, r, dtype=base.weight.dtype))

        def forward(self, x):
            return self.base(x) + nn.functional.linear(nn.functional.linear(x, self.lora_A), self.lora_B) * self.scaling

    def step_time(nl):
        cfg = Qwen3Config(hidden_size=4096, intermediate_size=12288, num_hidden_layers=nl, num_attention_heads=32, num_key_value_heads=8,
                          head_dim=128, vocab_size=151936, rms_norm_eps=1e-6, rope_theta=1e6, max_position_embeddings=40960,
                          tie_word_embeddings=False, attention_bias=False)
        with torch.device("meta"):
            m = Qwen3ForCausalLM(cfg)
        m = m.to_empty(device="cpu").to(torch.bfloat16)
        g = torch.Generator().manual_seed(0)
        with torch.no_grad():
            for p_ in m.parameters():
                if p_.dim() == 1:
                    p_.fill_(1.0)
                else:
                    blk = (torch.randn(4096, generator=g) * 0.02).to(torch.bfloat16)
                    p_.view(-1)[: (p_.numel() // 4096) * 4096].view(-1, 4096).copy_(blk)
        for mod in m.modules():
            if hasattr(mod, "inv_freq") and hasattr(mod, "compute_default_rope_parameters"):
                inv, _ = mod.compute_default_rope_parameters(cfg, "cpu")
                mod.inv_freq = inv
                mod.original_inv_freq = inv.clone()
        for p_ in m.parameters():
            p_.requires_grad_(False)
        train = []
        for layer in m.model.layers:
            for mod, names in ((layer.self_attn, ("q_proj", "k_proj", "v_proj", "o_proj")), (layer.mlp, ("gate_proj", "up_proj", "down_proj"))):
                for nm in names:
                    w = LoRALinear(getattr(mod, nm))
                    setattr(mod, nm, w)
                    train += [w.lora_A, w.lora_B]
        opt = torch.optim.AdamW(train, lr=1e-4) if train else None
        ids = torch.randint(0, 150000, (1, S))
        labels = ids.clone()
        labels[:, : S - ANSWER_IDS] = -100
        ts = []
        for it in range(3):
            t0 = time.perf_counter()
            out = m(input_ids=ids, labels=labels)
            if train:
                out.loss.backward()
                opt.step()
                opt.zero_grad(set_to_none=True)
            ts.append(time.perf_counter() - t0)
        del m
        return float(np.median(ts[1:]))

    t_s, t_0 = step_time(layers_sample), step_time(0)
    per_layer = max(t_s - t_0, 0.0) / layers_sample
    step = t_0 + per_layer * full_layers
    v = S / step
    base = {"value": v, "unit": "tokens/s", "cores": threads, "kind": "reference",
            "sample": (f"stock transformers Qwen3ForCausalLM + LoRA wrappers (r=16 on q,k,v,o,gate,up,down), bf16, {threads} threads, ChatTS-8B layer "
                       f"shape, ONE sample of {S} positions ({ANSWER_IDS} labels): forward+backward+AdamW; timed {layers_sample} of 36 decoder layers "
                       f"(median of 2 steps), per-layer time scaled x36 (head {t_0 * 1e3:.0f} ms, layer {per_layer * 1e3:.0f} ms)")}
    line = {"impl": "reference", "metric": "lora_finetune_positions_per_s", "value": v, "unit": "tokens/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": step * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
            "data": "synthetic", "config": {"workload": f"ChatTS-8B LoRA r=16 fine-tune step, 1 sample x {S} merged positions (CPU arm)"},
            "cpu_baseline": base, "e2e": {"value": v, "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--samples", type=int, default=16, help="samples per GPU and step (448 merged positions each)")
    ap.add_argument("--layers", type=int, default=0, help="debug: fewer decoder layers (INVALID as a benchmark)")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run(args)


if __name__ == "__main__":
    main()
