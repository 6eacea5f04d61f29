"""Logits processors of vLLM's and OpenAI's sampling parameters: ``allowed_token_ids``, ``logit_bias``, ``min_tokens`` and the
repetition, presence and frequency penalties, applied by csrc/logit_proc.cu between the decode step and the advance.

Every step works on the row's 16-bit logits ``x``, in fp32, rounded once to the logits' dtype:
  1. allowed_token_ids: x[t] = -inf for every t outside the set;
  2. logit_bias: x[t] += bias[t] (values clamped to [-100, 100], as vLLM does);
  3. min_tokens: while the row has generated fewer than min_tokens tokens, x[s] = -inf for each of its stop ids;
  4. repetition_penalty, over the ids of the prompt and the output: x / p where x > 0, else x * p;
  5. x[t] = (x[t] - frequency_penalty * c[t]) - presence_penalty where c[t] > 0 counts t among the GENERATED tokens.
This is vLLM v1's order (allowed mask, logit bias and min_tokens, then apply_penalties); vLLM keeps the result in fp32.

``LogitProcState`` holds the per-row parameters on the device: one launch serves a generate() batch, whose rows are equal, and the
continuous engine's slots, whose rows differ.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch

MAX_STOP_IDS = 64                   # cts_logit_proc_apply reads at most 64 stop ids per row
PENALTY_BOUND = 2.0                 # vLLM's range for presence_penalty and frequency_penalty
BIAS_BOUND = 100.0                  # vLLM's clamp of logit_bias values


@dataclass
class Processors:
    """The validated, non-neutral processor fields of one request (see ``resolve``)."""
    repetition_penalty: float = 1.0
    presence_penalty: float = 0.0
    frequency_penalty: float = 0.0
    logit_bias: dict = None             # {token id: clamped bias}
    allowed_token_ids: list = None      # sorted distinct ids
    min_tokens: int = 0

    def bias_vector(self, vocab):
        """The bias table row: -inf outside allowed_token_ids, the clamped bias where one is set, 0 elsewhere (None: no row needed)."""
        if self.logit_bias is None and self.allowed_token_ids is None:
            return None
        row = np.zeros(vocab, dtype=np.float32)
        if self.allowed_token_ids is not None:
            row[:] = -np.inf
            row[np.asarray(self.allowed_token_ids, dtype=np.int64)] = 0.0
        for t, v in (self.logit_bias or {}).items():
            if row[t] != -np.inf:                       # a masked id stays -inf whatever its bias
                row[t] = v
        return row


def _penalty(v, name):
    v = float(v)
    if not -PENALTY_BOUND <= v <= PENALTY_BOUND:
        raise ValueError(f"{name} must be in [-2, 2], got {v}")
    return v


def resolve(presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=None, logit_bias=None, allowed_token_ids=None,
            min_tokens=None, max_tokens=None, vocab=None):
    """Validate the processor fields of a request (ValueError on a bad one) and return them as ``Processors``, or None when every field
    is neutral: penalties 0 (1 for repetition), logit_bias None or {}, allowed_token_ids None, min_tokens None or 0.  String keys of
    logit_bias are token ids, as OpenAI sends them.  Token ids are checked against ``vocab`` and min_tokens against ``max_tokens``
    when they are given."""
    p = Processors(presence_penalty=_penalty(presence_penalty or 0.0, "presence_penalty"),
                   frequency_penalty=_penalty(frequency_penalty or 0.0, "frequency_penalty"))
    if repetition_penalty is not None:
        rp = float(repetition_penalty)
        if not (rp > 0 and math.isfinite(rp)):
            raise ValueError(f"repetition_penalty must be > 0, got {repetition_penalty}")
        p.repetition_penalty = rp
    if logit_bias:
        if not isinstance(logit_bias, dict):
            raise ValueError("logit_bias must map token ids to biases")
        bias = {}
        for k, v in logit_bias.items():
            try:
                t = int(k)
            except (TypeError, ValueError):
                raise ValueError(f"logit_bias keys must be token ids, got {k!r}") from None
            if t < 0:
                raise ValueError(f"logit_bias token id {t} is negative")
            v = float(v)
            if math.isnan(v):
                raise ValueError(f"logit_bias value for token {t} is NaN")
            bias[t] = min(max(v, -BIAS_BOUND), BIAS_BOUND)
        p.logit_bias = bias
    if allowed_token_ids is not None:
        ids = sorted({int(t) for t in allowed_token_ids})
        if not ids:
            raise ValueError("allowed_token_ids must not be empty")
        if ids[0] < 0:
            raise ValueError(f"allowed_token_ids holds a negative id {ids[0]}")
        p.allowed_token_ids = ids
    mt = int(min_tokens or 0)
    if mt < 0:
        raise ValueError(f"min_tokens must be >= 0, got {mt}")
    if max_tokens is not None and mt > int(max_tokens):
        raise ValueError(f"min_tokens ({mt}) must be <= max_tokens ({max_tokens})")
    p.min_tokens = mt
    if vocab is not None:
        check_vocab(p, vocab)
    if (p.presence_penalty == 0 and p.frequency_penalty == 0 and p.repetition_penalty == 1 and p.logit_bias is None
            and p.allowed_token_ids is None and p.min_tokens == 0):
        return None
    return p


def check_vocab(p, vocab):
    """Every id of logit_bias and allowed_token_ids must be < vocab (ValueError)."""
    if p is None:
        return
    bad = [t for t in (p.logit_bias or {}) if t >= vocab] + [t for t in (p.allowed_token_ids or []) if t >= vocab]
    if bad:
        raise ValueError(f"token id(s) {sorted(set(bad))[:8]} in logit_bias / allowed_token_ids are outside the vocabulary of {vocab}")


def check_stop_ids(p, stop_ids):
    if p is not None and p.min_tokens > 0 and len(stop_ids) > MAX_STOP_IDS:
        raise ValueError(f"min_tokens works with at most {MAX_STOP_IDS} stop ids per request, got {len(stop_ids)}")


class LogitProcState:
    """Per-row processor parameters on the device for ``rows`` rows of ``vocab`` logits.  The generated-token counts (uint16) and the
    bias table are allocated when a row first needs them; stop ids grow to the widest row."""

    def __init__(self, ctx, rows, vocab, n_pos, device):
        # counts are uint16 (stored as int16): a row generates fewer tokens than the model's positions
        assert n_pos < 65536, f"uint16 token counts need fewer than 65536 positions per row, got {n_pos}"
        self.ctx, self.rows, self.V, self.dev = ctx, int(rows), int(vocab), device
        f32 = dict(dtype=torch.float32, device=device)
        i32 = dict(dtype=torch.int32, device=device)
        self.rep, self.presence, self.frequency = torch.ones(rows, **f32), torch.zeros(rows, **f32), torch.zeros(rows, **f32)
        self.seen = torch.zeros(rows, (vocab + 31) // 32, **i32)
        self.bias_row = torch.full((rows,), -1, **i32)
        self.n_generated, self.min_tokens = torch.zeros(rows, **i32), torch.zeros(rows, **i32)
        self.counts = self.bias = self.stop_ids = None

    def set_rows(self, idx, p, stop_ids, shared_bias):
        """Rows ``idx`` (list of ints) start a request with processors ``p``: parameters set, counts / seen / n_generated zeroed.
        shared_bias: one bias-table row serves them all (generate()); else row i of the table belongs to row i (the engine)."""
        ix = torch.as_tensor(idx, dtype=torch.long, device=self.dev)
        self.rep[ix], self.presence[ix], self.frequency[ix] = p.repetition_penalty, p.presence_penalty, p.frequency_penalty
        self.seen[ix] = 0
        self.n_generated[ix] = 0
        self.min_tokens[ix] = p.min_tokens
        if p.presence_penalty != 0 or p.frequency_penalty != 0:
            if self.counts is None:
                self.counts = torch.zeros(self.rows, self.V, dtype=torch.int16, device=self.dev)
        if self.counts is not None:
            self.counts[ix] = 0
        stops = sorted({int(s) for s in stop_ids}) if p.min_tokens > 0 else []
        check_stop_ids(p, stops)
        if stops:
            w = len(stops) if self.stop_ids is None else max(len(stops), self.stop_ids.shape[1])
            if self.stop_ids is None or self.stop_ids.shape[1] < w:
                grown = torch.full((self.rows, w), -1, dtype=torch.int32, device=self.dev)
                if self.stop_ids is not None:
                    grown[:, :self.stop_ids.shape[1]] = self.stop_ids
                self.stop_ids = grown
        if self.stop_ids is not None:
            self.stop_ids[ix] = -1                           # a row without stop ids must not keep those of an earlier request
            if stops:
                self.stop_ids[ix, :len(stops)] = torch.tensor(stops, dtype=torch.int32, device=self.dev)
        vec = p.bias_vector(self.V)
        if vec is None:
            self.bias_row[ix] = -1
        else:
            n = 1 if shared_bias else self.rows
            if self.bias is None or self.bias.shape[0] < n:
                self.bias = torch.zeros(n, self.V, dtype=torch.float32, device=self.dev)
            d = torch.from_numpy(vec).to(self.dev)
            if shared_bias:
                self.bias[0] = d
                self.bias_row[ix] = 0
            else:
                self.bias[ix] = d
                self.bias_row[ix] = ix.to(torch.int32)

    def reset_rows(self, idx):
        """Neutral parameters: the apply kernel skips the rows."""
        ix = torch.as_tensor(idx, dtype=torch.long, device=self.dev)
        self.rep[ix], self.presence[ix], self.frequency[ix] = 1.0, 0.0, 0.0
        self.bias_row[ix] = -1
        self.min_tokens[ix] = 0
        if self.stop_ids is not None:
            self.stop_ids[ix] = -1

    def mark_prompt(self, tokens, rows):
        """Occurrence bits of the prompt ids (int32 device tensors) for the repetition penalty."""
        self.ctx.rep_penalty_mark(tokens, rows, self.seen, self.V)

    def apply(self, logits, batch, slots=None):
        """Processors over logits rows [0, batch); ``slots``: logits row i belongs to state row slots[i] (default: row i)."""
        ix = None if slots is None else torch.as_tensor(slots, dtype=torch.long, device=self.dev)
        at = lambda t: t if ix is None or t is None else t[ix]
        self.ctx.logit_proc_apply(logits, batch, at(self.rep), at(self.presence), at(self.frequency), at(self.seen), at(self.counts),
                                  self.bias, at(self.bias_row), at(self.n_generated), at(self.min_tokens), at(self.stop_ids), vocab=self.V)

    def update(self, cur_ids, batch, slots=None):
        """Counts the new tokens cur_ids[:batch]; ``slots`` as in apply (every other row gets -1, which the kernel leaves alone)."""
        if slots is not None:
            cur = torch.full((self.rows,), -1, dtype=torch.int32, device=self.dev)
            cur[torch.as_tensor(slots, dtype=torch.long, device=self.dev)] = cur_ids[:batch]
            cur_ids, batch = cur, self.rows
        self.ctx.logit_proc_update(cur_ids, batch, self.seen, self.counts, self.n_generated, self.V)


class RepetitionPenaltyState:
    """repetition_penalty alone, one value for every row, with LogitProcState's interface: the occurrence bits of the prompt and
    generated ids, applied by cts_rep_penalty_apply, which touches only the marked ids where cts_logit_proc_apply reads every logit."""

    def __init__(self, ctx, rows, vocab, penalty, device):
        self.ctx, self.V, self.penalty = ctx, int(vocab), float(penalty)
        self.seen = torch.zeros(rows, (vocab + 31) // 32, dtype=torch.int32, device=device)

    def mark_prompt(self, tokens, rows):
        self.ctx.rep_penalty_mark(tokens, rows, self.seen, self.V)

    def apply(self, logits, batch):
        self.ctx.rep_penalty_apply(logits, batch, self.seen, self.penalty)

    def update(self, cur_ids, batch):
        self.ctx.rep_penalty_mark(cur_ids, None, self.seen, self.V)
