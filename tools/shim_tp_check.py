"""tools/tp_check.py on a machine WITHOUT a GPU: the tensor-parallel model with its RANKS AS PROCESSES, every kernel from its own source
through the "CUDA on CPU" shim (tests/cuda_on_cpu), the symmetric buffers as POSIX shared memory behind cts_ipc_*, torch.distributed on
gloo for what NCCL does on the box (handle exchange, prefill all-reduce, vocab gather).  Same checks as tp_check.py: logits against the
single-rank model, greedy agreement, identical tokens on all ranks.  TEST INFRASTRUCTURE ONLY.

    CTS_PEER_LL=1 CTS_DECODE_FUSED=2 python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29631 tools/shim_tp_check.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import shim_gpu_tests  # noqa: E402,F401   (applies the host patches and installs the shim context)
# the stand-alone low-latency all-reduce splits a token over several CTAs that wait for each other (not a cluster): let small grids run
# concurrently, as they do on the GPU
shim_gpu_tests._ctx.lib.shim_concurrent_grid(1)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer  # noqa: E402
from chatts_b200.model import ChatTSForCausalLM  # noqa: E402
from chatts_b200.weights import synthetic_state_dict  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo")
    dt = torch.bfloat16
    cfg = ChatTSConfig.tiny(num_attention_heads=8, num_key_value_heads=4, hidden_size=512, intermediate_size=1024, vocab_size=1024,
                            ts_token_start_index=1000, eos_token_id=1022, pad_token_id=1023)
    cfg.ts["hidden_size"] = 512
    sd = synthetic_state_dict(cfg, seed=11, device="cpu", dtype=dt, std=0.05)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    x = np.arange(256)
    enc = proc(text=["A <ts><ts/> then B <ts><ts/> ?", "plain text only prompt"], timeseries=[np.sin(x / 10) * 5, x[:90] * 0.1],
               padding=True, return_tensors="pt")
    new = int(os.environ.get("TP_CHECK_NEW", "12"))
    tp = ChatTSForCausalLM(cfg, sd, dtype=dt, tp_rank=rank, tp_size=world, max_batch=4, max_seq_len=512, page_size=16)
    lg_tp = tp.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0].float()
    runs = [dict(), dict(repetition_penalty=1.3)]          # the penalty alone runs on the eager decode step over the gathered logits
    ids_tp = [tp.generate(**enc, max_new_tokens=new, ignore_eos=True, **kw) for kw in runs]
    ok = True
    if rank == 0:
        ref = ChatTSForCausalLM(cfg, sd, dtype=dt, max_batch=4, max_seq_len=512, page_size=16, use_fused_decode=0)
        lg = ref.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0].float()
        ids = [ref.generate(**enc, max_new_tokens=new, ignore_eos=True, **kw) for kw in runs]
        err = float((lg_tp - lg).abs().max() / lg.abs().max())
        S = enc["input_ids"].shape[1]
        agree = [[int(next((i for i in range(new) if a[b, S + i] != t[b, S + i]), new)) for b in range(2)] for a, t in zip(ids, ids_tp)]
        print(f"[shim_tp_check] world={world} peer_ll={int(tp.use_peer_ll)} fused={tp.use_fused_decode} logits rel err vs single rank {err:.3e}; "
              f"greedy agreement {agree[0]}/{new}, with repetition_penalty=1.3 {agree[1]}/{new}", flush=True)
        ok = err < 2e-2 and min(min(a) for a in agree) >= min(new, 4)
    same = True
    for t in ids_tp:
        lst = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(lst, t)
        same = same and all(torch.equal(lst[0], x) for x in lst)
    if rank == 0:
        print(f"[shim_tp_check] identical tokens on all ranks: {same}", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if (ok and same) else 1)


if __name__ == "__main__":
    main()
