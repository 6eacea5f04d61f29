"""TEST INFRASTRUCTURE ONLY: the three kernels of csrc/structured.cu restated with numpy / torch, as the CPU statement the kernel tests
compare against and as the ``struct_*`` entry points of the torch test double (tests/cabi_double.py) for the host tests."""
import numpy as np
import torch

from tests.logprobs_double import LogprobsDouble


def walk(trans, s, data):
    for b in data:
        if s < 0:
            break
        s = int(trans[s, b])
    return s


def mask_build_reference(trans, accept, offsets, data, stops, chunk=256):
    """allowed bits int32 [S, ceil(V / 32)]: token t in state s iff it has bytes and walking them from s stays defined; a stop id iff s
    is accepting.  Walks every (state, token) pair one byte position at a time, keeping only the pairs still alive."""
    trans, accept = np.asarray(trans), np.asarray(accept).astype(bool)
    offsets, data = np.asarray(offsets, dtype=np.int64), np.asarray(data)
    S, V = trans.shape[0], len(offsets) - 1
    lens = np.diff(offsets)
    nz = lens > 0
    first = np.where(nz, data[np.minimum(offsets[:-1], max(len(data) - 1, 0))], 0)
    out = []
    for s0 in range(0, S, chunk):
        st = np.arange(s0, min(S, s0 + chunk))
        allowed = np.zeros((len(st), V), dtype=bool)
        cur = trans[st[:, None], first[None, :]]
        cur[:, ~nz] = -1
        si, ti = np.nonzero(cur >= 0)
        cs = cur[si, ti]
        j = 1
        while len(ti):
            done = lens[ti] <= j
            allowed[si[done], ti[done]] = True
            si, ti, cs = si[~done], ti[~done], cs[~done]
            if not len(ti):
                break
            cs = trans[cs, data[offsets[ti] + j]]
            ok = cs >= 0
            si, ti, cs = si[ok], ti[ok], cs[ok]
            j += 1
        for t in stops:
            allowed[:, int(t)] = accept[st]
        out.append(pack_bits(allowed))
    return np.concatenate(out)


def pack_bits(allowed):
    """bool [S, V] -> int32 words [S, ceil(V / 32)], bit j of word w = entry 32 w + j."""
    S, V = allowed.shape
    W = (V + 31) // 32
    pad = np.zeros((S, W * 32), dtype=bool)
    pad[:, :V] = allowed
    return np.packbits(pad, axis=1, bitorder="little").view("<u4").astype(np.uint32).view(np.int32).reshape(S, W)


def unpack_bits(words, V):
    w = np.ascontiguousarray(np.asarray(words).view(np.uint32).astype("<u4"))
    return np.unpackbits(w.view(np.uint8), axis=1, bitorder="little")[:, :V].astype(bool)


class StructuredDouble(LogprobsDouble):
    """The logprobs double plus cts_struct_mask_build / cts_struct_mask_apply / cts_struct_advance (same arguments as
    chatts_b200._cabi.Context)."""

    def struct_mask_build(self, trans, accept, offsets, token_bytes, stop_ids, allowed):
        ref = mask_build_reference(trans.cpu().numpy(), accept.cpu().numpy(), offsets.cpu().numpy(), token_bytes.cpu().numpy(),
                                   stop_ids.cpu().tolist())
        allowed.copy_(torch.from_numpy(ref))

    def struct_mask_apply(self, logits, batch, state, allowed, vocab=None):
        vocab = logits.shape[-1] if vocab is None else vocab
        bits = torch.from_numpy(unpack_bits(allowed.cpu().numpy(), vocab))
        for b in range(batch):
            s = int(state[b])
            if s >= 0:
                row = logits[b, :vocab]
                row.masked_fill_(~bits[s].to(row.device), float("-inf"))

    def struct_advance(self, cur_ids, batch, state, trans, offsets, token_bytes, stop_ids):
        tr, off, data = trans.cpu().numpy(), offsets.cpu().numpy(), token_bytes.cpu().numpy()
        stops = set(stop_ids.cpu().tolist())
        for b in range(batch):
            s, t = int(state[b]), int(cur_ids[b])
            if s < 0 or t < 0 or t >= len(off) - 1 or t in stops:
                continue
            n = walk(tr, s, data[off[t]:off[t + 1]])
            if n >= 0:
                state[b] = n
