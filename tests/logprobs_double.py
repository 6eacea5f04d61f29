"""TEST INFRASTRUCTURE ONLY: cts_logprobs (csrc/sampling.cu) restated with torch, as the CPU statement the kernel tests compare against
and as the ``logprobs`` entry point of the torch test double (tests/cabi_double.py) for the host tests."""
import numpy as np
import torch

from tests.prefix_double import PrefixDouble


def logprobs_reference(logits, chosen, k):
    """logits [R, V] (16-bit), chosen [R] ids (or None) -> (chosen logprob fp32 [R], rank int32 [R], top-k ids int32 [R, k], top-k
    logprobs fp32 [R, k]): log_softmax of the stored values, exact and rounded to fp32, with NaN entries left out of everything; top-k by value
    descending, equal values by the smaller id; slots past the non-NaN entries are (-1, NaN); a NaN chosen logit (or an id outside the
    row) gives NaN and rank 0."""
    x = logits.float().cpu()
    R, V = x.shape
    nan = torch.isnan(x)
    # the exact log_softmax of the stored values, rounded once to fp32: torch's own fp32 log_softmax on the CPU sums 152k terms with
    # an error of up to ~2e-5 in the result (measured against float64), more than the kernel's
    lp = torch.log_softmax(x.double().masked_fill(nan, float("-inf")), dim=-1).float()
    lp_c = torch.full((R,), float("nan"))
    rank = torch.zeros(R, dtype=torch.int32)
    ids = torch.full((R, k), -1, dtype=torch.int32)
    vals = torch.full((R, k), float("nan"))
    xn = x.numpy()
    for r in range(R):
        if chosen is not None:
            c = int(chosen[r])
            if 0 <= c < V and not bool(nan[r, c]):
                lp_c[r] = lp[r, c]
                rank[r] = 1 + int((x[r] > x[r, c]).sum())
        if k:
            valid = np.nonzero(~nan[r].numpy())[0]
            order = valid[np.lexsort((valid, -xn[r, valid].astype(np.float64)))][:k]
            ids[r, :len(order)] = torch.from_numpy(order.astype(np.int32))
            vals[r, :len(order)] = lp[r, torch.from_numpy(order)]
    return lp_c, rank, ids, vals


class LogprobsDouble(PrefixDouble):
    """The prefix-caching double plus cts_logprobs (same arguments as chatts_b200._cabi.Context.logprobs)."""

    def logprobs_workspace_floats(self, rows, vocab, k):
        return 2

    def logprobs(self, logits, rows, chosen, k, out_logprob, out_rank, out_topk_ids, out_topk_logprobs, workspace, counters,
                 step_ptr=None, vocab=None):
        vocab = logits.shape[-1] if vocab is None else vocab
        col = int(step_ptr[0]) - 1 if step_ptr is not None else 0
        ch = chosen[:rows, col] if chosen is not None else None
        lp, rank, ids, vals = logprobs_reference(logits[:rows, :vocab], ch, k)
        if out_logprob is not None:
            out_logprob[:rows, col] = lp
            out_rank[:rows, col] = rank
        if k:
            out_topk_ids[:rows, col] = ids
            out_topk_logprobs[:rows, col] = vals
