"""TEST INFRASTRUCTURE ONLY: the two kernels of csrc/logit_proc.cu restated with torch in the same fp32 arithmetic and the one rounding,
as the CPU statement the kernel tests compare against and as the ``logit_proc_*`` entry points of the torch test double
(tests/cabi_double.py) for the host tests."""
import torch

from tests.beam_double import BeamDouble


def unpack_seen(seen, V):
    """int32 words [B, ceil(V / 32)] -> bool [B, V], bit j of word w = id 32 w + j."""
    bits = seen.to(torch.int64) & 0xFFFFFFFF
    return ((bits[:, :, None] >> torch.arange(32, device=seen.device)[None, None, :]) & 1).reshape(seen.shape[0], -1)[:, :V].bool()


def process_fp32(x, rep=1.0, presence=0.0, frequency=0.0, seen=None, counts=None, bias=None, stops=(), min_active=False):
    """Steps 1-5 on one fp32 row x [V] before the rounding: (value, touched mask).  seen bool [V], counts int [V] (generated ids),
    bias float32 [V] (-inf: not allowed), stops the row's stop ids (applied when min_active)."""
    f = lambda v: torch.tensor(v, dtype=torch.float32)
    x = x.clone()
    touched = torch.zeros_like(x, dtype=torch.bool)
    if bias is not None:
        off = bias == float("-inf")
        add = ~off & (bias != 0)
        x = torch.where(off, f(float("-inf")), torch.where(add, x + bias, x))
        touched |= off | add
    if min_active:
        ids = [int(s) for s in stops if 0 <= int(s) < x.shape[0]]
        if ids:
            x[ids] = float("-inf")
            touched[ids] = True
    if rep != 1.0 and seen is not None:
        p = f(rep)
        x = torch.where(seen, torch.where(x > 0, x / p, x * p), x)
        touched |= seen
    if counts is not None and (presence != 0.0 or frequency != 0.0):
        c = counts.to(torch.float32)
        m = counts > 0
        x = torch.where(m, (x - f(frequency) * c) - f(presence), x)
        touched |= m
    return x, touched


def apply_reference(logits, batch, rep, presence, frequency, seen, counts, bias, bias_row, n_generated, min_tokens, stop_ids, vocab=None):
    """cts_logit_proc_apply on torch tensors (any device), in place: logits [>= batch, ld] 16-bit, the parameters as the kernel takes
    them (counts int16 read as uint16, or None; bias float32 [n, V] or None; stop_ids int32 [batch, m] padded with -1, or None)."""
    V = logits.shape[-1] if vocab is None else vocab
    rep, presence, frequency = (t.cpu().tolist() for t in (rep, presence, frequency))
    bias_row, n_generated, min_tokens = (t.cpu().tolist() for t in (bias_row, n_generated, min_tokens))
    seen_b = unpack_seen(seen[:batch].cpu(), V)
    for b in range(batch):
        br = bias_row[b]
        use_bias = bias is not None and 0 <= br < bias.shape[0]
        stops = []
        if stop_ids is not None and stop_ids.shape[1] > 0:
            for s in stop_ids[b].cpu().tolist():
                if s < 0:
                    break
                stops.append(s)
        use_min = stop_ids is not None and stop_ids.shape[1] > 0 and n_generated[b] < min_tokens[b]
        use_cnt = counts is not None and (presence[b] != 0 or frequency[b] != 0)
        if not (use_bias or use_min or rep[b] != 1.0 or use_cnt):
            continue
        row = logits[b, :V]
        x, touched = process_fp32(row.float().cpu(), rep[b], presence[b], frequency[b], seen_b[b],
                                  (counts[b, :V].cpu().to(torch.int32) & 0xFFFF) if use_cnt else None,
                                  bias[br, :V].cpu() if use_bias else None, stops, use_min)
        row.copy_(torch.where(touched, x.to(logits.dtype), row.cpu()).to(row.device))


def update_reference(cur_ids, batch, seen, counts, n_generated, vocab):
    """cts_logit_proc_update in place."""
    for b, t in enumerate(cur_ids[:batch].cpu().tolist()):
        if not 0 <= t < vocab:
            continue
        if counts is not None:
            counts[b, t] += 1
        w = seen[b, t >> 5].item() & 0xFFFFFFFF
        w |= 1 << (t & 31)
        seen[b, t >> 5] = w - (1 << 32) if w >= 1 << 31 else w
        n_generated[b] += 1


class LogitProcDouble(BeamDouble):
    """The beam double plus cts_logit_proc_apply / cts_logit_proc_update (same arguments as chatts_b200._cabi.Context), counting its
    calls of both in ``calls``."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = {"apply": 0, "update": 0}

    def logit_proc_apply(self, logits, batch, rep, presence, frequency, seen, counts, bias, bias_row, n_generated, min_tokens, stop_ids,
                         vocab=None):
        self.calls["apply"] += 1
        apply_reference(logits, batch, rep, presence, frequency, seen, counts, bias, bias_row, n_generated, min_tokens, stop_ids, vocab)

    def logit_proc_update(self, cur_ids, batch, seen, counts, n_generated, vocab):
        self.calls["update"] += 1
        update_reference(cur_ids, batch, seen, counts, n_generated, vocab)
