"""torchrun --nproc-per-node 2 tools/tp_check.py [--fp8] : tensor-parallel path (NCCL prefill all-reduce + fused peer-memory
decode all-reduce) against the single-GPU path on the same weights.  --fp8: both models quantize_fp8()'d (the row maximum of the K-sliced
o_proj / down_proj all-reduced over the ranks, so both hold the same FP8 weights)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer  # noqa: E402
from chatts_b200.model import ChatTSForCausalLM  # noqa: E402
from chatts_b200.weights import synthetic_state_dict  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    dt = torch.bfloat16
    cfg = ChatTSConfig.tiny(num_attention_heads=8, num_key_value_heads=4, hidden_size=512, intermediate_size=1024, vocab_size=1024,
                            ts_token_start_index=1000, eos_token_id=1022, pad_token_id=1023)
    cfg.ts["hidden_size"] = 512
    sd = synthetic_state_dict(cfg, seed=11, device="cpu", dtype=dt, std=0.05)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    x = np.arange(256)
    enc = proc(text=["A <ts><ts/> then B <ts><ts/> ?", "plain text only prompt"], timeseries=[np.sin(x / 10) * 5, x[:90] * 0.1],
               padding=True, return_tensors="pt")
    fp8 = "--fp8" in sys.argv[1:]
    tp = ChatTSForCausalLM(cfg, sd, dtype=dt, tp_rank=rank, tp_size=world, max_batch=4, max_seq_len=512, page_size=16)
    if fp8:
        tp.quantize_fp8()
    # a prefill whose total token count is NOT a multiple of the world size and above the peer-memory path's limit: the NCCL exchange of the
    # row-parallel projections (fp32 reduce-scatter over padded token shards + 16-bit all-gather, model.py:_tp_row_parallel)
    filler = "the quick brown fox jumps over the lazy dog " * 3
    for extra in range(0, 8):
        enc = proc(text=["A <ts><ts/> then B <ts><ts/> ? " + filler + "x" * extra, "plain text only prompt " + filler], timeseries=[np.sin(x / 10) * 5, x[:90] * 0.1],
                   padding=True, return_tensors="pt")
        T = int(tp._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])[3].total)
        if T % world != 0 and T > tp.peer_tokens:
            break
    if rank == 0:
        print(f"[tp_check] prefill tokens {T} (mod world = {T % world}), exchange = {tp.tp_prefill_exchange}, nccl = {tp._nccl}", flush=True)
    lg_tp = tp.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0].float().cpu()
    ids_tp = tp.generate(**enc, max_new_tokens=24, ignore_eos=True)
    ok = True
    if rank == 0:
        ref = ChatTSForCausalLM(cfg, sd, dtype=dt, max_batch=4, max_seq_len=512, page_size=16)
        if fp8:
            ref.quantize_fp8()
        lg = ref.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0].float().cpu()
        ids = ref.generate(**enc, max_new_tokens=24, ignore_eos=True)
        err = float((lg_tp - lg).abs().max() / lg.abs().max())
        S = enc["input_ids"].shape[1]
        agree = [int(next((i for i in range(24) if ids[b, S + i] != ids_tp[b, S + i]), 24)) for b in range(2)]
        print(f"[tp_check] world={world} fp8={int(fp8)} logits rel err vs single GPU {err:.3e}; greedy agreement {agree}/24", flush=True)
        ok = err < 2e-2
    # all ranks must hold identical tokens (the fused all-reduce sums in rank order on every rank)
    t = ids_tp.cuda()
    lst = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(lst, t)
    same = all(torch.equal(lst[0], l) for l in lst)
    if rank == 0:
        print(f"[tp_check] identical tokens on all ranks: {same}", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if (ok and same) else 1)


if __name__ == "__main__":
    main()
