"""Tensor-parallel plumbing: symmetric (cudaIpc) buffers shared by the ranks of one NVSwitch domain.

torch.distributed carries only the 64-byte IPC handles (and NCCL the large prefill all-reduces); the decode
all-reduces run over the mapped peer pointers.  By default that is cts_peer_allreduce_ll, the two-shot kernel with its
flags inside the data; CTS_PEER_LL=0 selects cts_peer_allreduce_residual_rmsnorm, the one-shot kernel that pushes every
rank's rows to every peer.  Greedy decoding takes the global argmax with cts_peer_greedy_advance over the candidate tables."""

import torch
import torch.distributed as dist


class _Raw:
    """A device pointer wrapped so the ctypes layer can take .data_ptr() from it."""

    def __init__(self, ptr):
        self.ptr = ptr

    def data_ptr(self):
        return self.ptr


class PeerBuffers:
    def __init__(self, ctx, rank, world, max_tokens, hidden, group=None, n_buffers=2):
        self.ctx, self.rank, self.world = ctx, rank, world
        # per buffer: one [max_tokens, hidden] fp32 slot per source rank (one-shot kernel); never less than 4 slots, which is what the
        # low-latency layout (cts_peer_allreduce_ll: 12 bytes per element + statistics) needs at 2 ranks
        self.floats = max(world, 4) * max_tokens * hidden
        ll_bytes = ctx.peer_ll_region_bytes(world, max_tokens, hidden)
        self.floats = max(self.floats, (ll_bytes + 255) // 256 * 64)
        dev = torch.device(f"cuda:{torch.cuda.current_device()}")
        # one allocation per rank: n_buffers fp32 partial buffers, then the flag array int[world]
        self.part_bytes = self.floats * 4
        self.flag_off = n_buffers * self.part_bytes                          # int32 [n_buffers][world][max_tokens][8 chunks]
        self.max_batch = max_tokens
        self.cand_off = self.flag_off + n_buffers * world * max_tokens * 8 * 4 + 256   # float2 [world][max_tokens]
        self.cflag_off = self.cand_off + world * max_tokens * 8              # int32  [world][max_tokens]
        total = self.cflag_off + world * max_tokens * 4 + 256
        self.local_ptr, handle = ctx.ipc_alloc(total)
        handles = [None] * world
        dist.all_gather_object(handles, handle, group=group)
        self.peer_base = [self.local_ptr if r == rank else ctx.ipc_open(handles[r]) for r in range(world)]
        dist.barrier(group=group)                      # every rank has zeroed and mapped before anyone signals
        self.partials = []
        for b in range(n_buffers):
            arr = torch.tensor([p + b * self.part_bytes for p in self.peer_base], dtype=torch.int64, device=dev)
            self.partials.append(arr)
        self.flags = [torch.tensor([p + self.flag_off + b * world * max_tokens * 8 * 4 for p in self.peer_base], dtype=torch.int64,
                                   device=dev) for b in range(n_buffers)]
        self.state = torch.zeros(2, dtype=torch.int32, device=dev)
        self.cand = torch.tensor([p + self.cand_off for p in self.peer_base], dtype=torch.int64, device=dev)
        self.cand_flags = torch.tensor([p + self.cflag_off for p in self.peer_base], dtype=torch.int64, device=dev)
        self.cand_state = torch.zeros(2, dtype=torch.int32, device=dev)
        self.local = [_Raw(self.local_ptr + b * self.part_bytes) for b in range(n_buffers)]

    def local_partial(self, b):
        """fp32 [max_tokens*hidden] view of this rank's b-th partial buffer (GEMM output target)."""
        return self.local[b]
