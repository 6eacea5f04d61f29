"""Log probabilities of generated and prompt tokens (cts_logprobs, csrc/sampling.cu).

The numbers describe the distribution a token was picked from: log_softmax in fp32 of the 16-bit logits, after the repetition penalty
when one is set and before temperature, top-k and top-p -- vLLM's raw logprobs whenever repetition_penalty == 1.  The rank of a token
is 1 + the number of entries with a larger logit; the top-k entries are ordered by value, equal values by the smaller id."""
from collections import namedtuple
from dataclasses import dataclass

import numpy as np
import torch

from ._cabi import LOGPROBS_MAX_K

# one prompt position: the token, its logprob and rank, and the top-k (ids, logprobs) of the distribution that predicted it
PromptLogprob = namedtuple("PromptLogprob", "token_id logprob rank top_ids top_logprobs")


def check_k(k, name):
    """None (not asked) or an int in [0, 20]; anything else raises ValueError."""
    if k is None:
        return None
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 0 <= int(k) <= LOGPROBS_MAX_K:
        raise ValueError(f"{name} must be an integer in [0, {LOGPROBS_MAX_K}] or None, got {k!r}")
    return int(k)


@dataclass
class GenerationLogprobs:
    """What generate() leaves in ``model.last_logprobs``.  Decode fields (None unless ``logprobs`` was asked): per row and generated
    token, ``logprobs`` [B, n] and ``ranks`` [B, n] of the token, ``top_ids`` / ``top_logprobs`` [B, n, k].  Columns past a row's
    end of sequence belong to the padding generate() returns there.  ``prompt`` (None unless ``prompt_logprobs`` was asked): per row, one
    entry per non-padding column of the caller's input_ids -- None for the first one, and for ``<ts>`` / ``<ts/>`` in overwrite mode
    (they have no merged position) -- else a PromptLogprob."""
    logprobs: np.ndarray = None
    ranks: np.ndarray = None
    top_ids: np.ndarray = None
    top_logprobs: np.ndarray = None
    prompt: list = None


class LogprobBuffers:
    """Device outputs of cts_logprobs for ``rows`` x ``cols`` entries at top-k ``k``, with the workspace and arrival counters.  The
    top-k buffers are laid out [rows, cols, k] for the k of the launch (any k up to the one they were made for); one launch covers at
    most ``launch_rows`` rows (default: all)."""

    def __init__(self, ctx, rows, cols, k, vocab, device, launch_rows=None):
        launch_rows = rows if launch_rows is None else launch_rows
        self.ctx, self.rows, self.cols, self.k, self.vocab = ctx, rows, cols, k, vocab
        self.lp = torch.zeros(rows, cols, dtype=torch.float32, device=device)
        self.rank = torch.zeros(rows, cols, dtype=torch.int32, device=device)
        self.ids = torch.zeros(rows * cols * max(k, 1), dtype=torch.int32, device=device)
        self.vals = torch.zeros(rows * cols * max(k, 1), dtype=torch.float32, device=device)
        self.ws = torch.empty(max(ctx.logprobs_workspace_floats(launch_rows, vocab, k), 2), dtype=torch.float32, device=device)
        self.counters = torch.zeros(launch_rows, dtype=torch.int32, device=device)

    def topk_views(self, k):
        n = self.rows * self.cols * k
        return self.ids[:n].view(self.rows, self.cols, k), self.vals[:n].view(self.rows, self.cols, k)

    def launch(self, logits, rows, chosen, k=None, step_ptr=None, row0=0):
        """Entries of rows [row0, row0 + rows) from logits [rows, >= vocab]: at column step_ptr[0] - 1 (the column the advance just
        wrote), or at column 0 without step_ptr."""
        k = self.k if k is None else k
        ids, vals = self.topk_views(k)
        lp, rank = self.lp[row0:], self.rank[row0:]
        ids, vals = ids[row0:], vals[row0:]
        self.ctx.logprobs(logits, rows, chosen, k, lp, rank, ids, vals, self.ws, self.counters, step_ptr=step_ptr, vocab=self.vocab)

    def host(self, cols, k=None):
        """(logprobs [rows, cols], ranks, top_ids [rows, cols, k], top_logprobs) on the host."""
        k = self.k if k is None else k
        ids, vals = self.topk_views(k)
        return (self.lp[:, :cols].cpu().numpy(), self.rank[:, :cols].cpu().numpy(), ids[:, :cols].cpu().numpy(),
                vals[:, :cols].cpu().numpy())


def prompt_targets(lay):
    """The prompt tokens that get a logprob, in merged order: (pred, target, row, col) -- the merged position whose logits predict the
    token (the one before it, which can be a patch row: in insert mode ``<ts/>`` is predicted by the last patch row of its series),
    the token id, its batch row and its column in the caller's input_ids.  A sequence's first position has no prediction; patch rows
    are not tokens of the input, and in overwrite mode ``<ts>`` / ``<ts/>`` have no merged position."""
    cu = lay.cu_seqlens.astype(np.int64)
    j = np.nonzero(lay.src_col >= 0)[0]
    b = np.searchsorted(cu, j, side="right") - 1
    keep = j > cu[b]
    j, b = j[keep], b[keep]
    return j - 1, lay.ids[j].astype(np.int32), b, lay.src_col[j].astype(np.int64)


def prompt_entries(ids_cpu, am_cpu, rows, cols, targets, lp, rank, top_ids, top_lps):
    """Per row, the list of GenerationLogprobs.prompt: one entry per non-padding column of input_ids."""
    B, S = ids_cpu.shape
    am = np.ones((B, S), dtype=bool) if am_cpu is None else np.asarray(am_cpu).astype(bool)
    out = []
    for b in range(B):
        kept = np.nonzero(am[b])[0]
        idx = np.full(S, -1, dtype=np.int64)
        idx[kept] = np.arange(kept.shape[0])
        out.append([None] * kept.shape[0])
        for i in np.nonzero(rows == b)[0]:
            out[b][idx[cols[i]]] = PromptLogprob(int(targets[i]), float(lp[i]), int(rank[i]), top_ids[i].tolist(), top_lps[i].tolist())
    return out
