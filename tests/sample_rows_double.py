"""TEST INFRASTRUCTURE ONLY: cts_sample_advance_rows (csrc/sampling.cu) restated row by row on the CPU, on top of the logits-processor
double: a row with !(temperature > 0) takes cts_greedy_advance's token, any other row TorchDouble.sample_reference with its own
parameters and the draw (seed[b], draw_step[b], draw_key[b]); draw_step[b] += 1 for every row, and the advance state moves as
cts_sample_advance moves it."""
import torch

from tests.logit_proc_double import LogitProcDouble


def greedy_reference(row):
    """cts_greedy_advance's token of one row: the first maximum, NaN never wins, 0 when no value exceeds -inf."""
    x = row.float()
    ok = x > float("-inf")                               # False for NaN and -inf
    if not bool(ok.any()):
        return 0
    return int(torch.nonzero(x == x[ok].max())[0, 0])


class SampleRowsDouble(LogitProcDouble):
    """The logits-processor double plus cts_sample_advance_rows (same arguments as chatts_b200._cabi.Context)."""

    def sample_advance_rows(self, logits, B, temperature, top_k, top_p, seed, draw_key, draw_step, out_tokens, step_ptr, cur, pos, sl,
                            slot, pt, page):
        st = int(step_ptr[0])
        for b in range(B):
            t = float(temperature[b])
            if not t > 0:
                tok = greedy_reference(logits[b])
            else:
                tok = self.sample_reference(logits[b], t, int(top_k[b]), float(top_p[b]), int(seed[b]) & ((1 << 64) - 1),
                                            int(draw_step[b]), int(draw_key[b]))[0]
            draw_step[b] += 1
            if out_tokens is not None:
                out_tokens[b, st] = tok
            if cur is not None:
                cur[b] = tok
            if pos is not None:
                pos[b] += 1
                if sl is not None:
                    sl[b] += 1
                if slot is not None and pt is not None:
                    slot[b] = pt[b, int(pos[b]) // page] * page + int(pos[b]) % page
        step_ptr[0] += 1
