"""Beam search for ``generate(num_beams=...)``: the host side of csrc/beam.cu.

The semantics are transformers' vectorised ``GenerationMixin._beam_search`` (read against transformers 5.5.0): step 0 runs on the
prefill logits with beam 0 at score 0 and the other beams at -1e9; every step adds each beam's running score to the fp32 log_softmax
of its logits and keeps the top ``max(2, 1 + n_eos) * num_beams`` over the prompt's flattened [num_beams * vocab] scores; the running
beams are the best ``num_beams`` of those that hit no stopping criterion; the finished hypotheses come from the top ``num_beams`` that
hit EOS or the length limit, scored ``sum_logprobs / generated_len ** length_penalty``, with the ``early_stopping`` True / False /
"never" rules.  Ties, which torch.topk leaves unspecified, go to the smaller flattened index ``beam * vocab + id`` (within one row: the
smaller id, as cts_logprobs orders its top-k), then to the better-ranked candidate, then to the older finished hypothesis.

Pages: each prompt is prefilled once and its full prompt pages are shared by all its beams.  Every beam row owns one page for every page
index from the prompt's tail page to the end of ``max_new_tokens`` (beam 0's first one is the prompt's own tail page) plus one spare;
a page is written only while it is the tail of exactly one row, and a child of another row gets a copy of its parent's partial tail
(cts_beam_fork_kv)."""
import numpy as np

EARLY_STOPPING = {False: 0, True: 1, "never": 2}
MAX_KEEP = 20                          # the top-k limit of cts_logprobs: the per-row candidates


def beams_to_keep(num_beams, n_eos):
    return max(2, 1 + n_eos) * num_beams


def check_args(num_beams, length_penalty, early_stopping, num_return_sequences, n_eos, batch, max_batch, do_sample=False,
               num_beam_groups=None, diversity_penalty=None, repetition_penalty=None, logprobs=None, prompt_logprobs=None,
               structured_outputs=None, streamer=None, tp_size=1):
    """Every refusal of a beam-search call, raised as ValueError before any page is taken or any kernel runs.  -> beams_to_keep."""
    if isinstance(num_beams, bool) or not isinstance(num_beams, (int, np.integer)) or num_beams < 1:
        raise ValueError(f"num_beams must be a positive integer, got {num_beams!r}")
    if do_sample:
        raise ValueError("beam sampling is not supported: pass do_sample=False with num_beams > 1 (the checkpoint's generation "
                         "defaults may set do_sample=True)")
    if (num_beam_groups or 1) > 1 or diversity_penalty:
        raise ValueError("group / diverse beam search (num_beam_groups > 1, diversity_penalty) is not supported")
    if repetition_penalty not in (None, 1, 1.0):
        raise ValueError("repetition_penalty != 1 is not supported with num_beams > 1 (it may come from the checkpoint's generation "
                         "defaults: pass repetition_penalty=1.0)")
    for name, v in (("logprobs", logprobs), ("prompt_logprobs", prompt_logprobs), ("structured_outputs", structured_outputs),
                    ("streamer", streamer)):
        if v is not None:
            raise ValueError(f"{name} cannot be combined with num_beams > 1")
    if tp_size > 1:
        raise ValueError("beam search is single-GPU only (tensor_parallel_size must be 1)")
    if early_stopping not in (False, True, "never") or not isinstance(early_stopping, (bool, str)):
        raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
    if not isinstance(length_penalty, (int, float, np.floating)) or not np.isfinite(length_penalty):
        raise ValueError(f"length_penalty must be a finite number, got {length_penalty!r}")
    if isinstance(num_return_sequences, bool) or not isinstance(num_return_sequences, (int, np.integer)) \
            or not 1 <= num_return_sequences <= num_beams:
        raise ValueError(f"num_return_sequences must be in [1, num_beams = {num_beams}], got {num_return_sequences!r}")
    keep = beams_to_keep(num_beams, n_eos)
    if keep > MAX_KEEP:
        raise ValueError(f"max(2, 1 + number of EOS ids) * num_beams = {keep} candidates per step exceeds {MAX_KEEP}, the top-k limit "
                         f"of cts_logprobs: with {n_eos} EOS id(s) num_beams can be at most {MAX_KEEP // max(2, 1 + n_eos)}")
    if batch * num_beams > max_batch:
        raise ValueError(f"batch {batch} x num_beams {num_beams} = {batch * num_beams} rows exceeds max_batch {max_batch}")
    return keep


def len_den(max_new, length_penalty):
    """float32 [max_new + 1]: entry L is L ** length_penalty computed as transformers does (a Python number, then one rounding to
    fp32 where it divides an fp32 score)."""
    d = np.ones(max_new + 1, dtype=np.float32)
    for L in range(1, max_new + 1):
        d[L] = np.float32(L ** length_penalty)
    return d


def extra_pages(lens, needs, num_beams, page_size):
    """Pages a beam search takes beyond the prompt's own allocation (which already covers beam 0): every other beam's own page for
    each index from the prompt's tail page to the last page, and one spare per beam."""
    return sum((num_beams - 1) * (int(n) - int(L) // page_size) + num_beams for L, n in zip(lens, needs))


def page_plan(page_tables, lens, needs, num_beams, page_size, extra):
    """-> (page_table, own_pages int32 [B * num_beams, max_pages] (-1 outside the row's pages), spare int32 [B * num_beams]).
    Row b * num_beams + j starts with the prompt's full pages and its own page at the tail index (beam 0: the prompt's tail page)."""
    B, max_pages = page_tables.shape
    R = B * num_beams
    table = np.zeros((R, max_pages), dtype=np.int32)
    own = np.full((R, max_pages), -1, dtype=np.int32)
    spare = np.zeros(R, dtype=np.int32)
    it = iter(extra)
    for b in range(B):
        p0, n = int(lens[b]) // page_size, int(needs[b])
        for j in range(num_beams):
            r = b * num_beams + j
            table[r, :p0] = page_tables[b, :p0]
            own[r, p0:n] = page_tables[b, p0:n] if j == 0 else [next(it) for _ in range(p0, n)]
            spare[r] = next(it)
            table[r, p0] = own[r, p0]
    return table, own, spare


def hypothesis(bp_tokens, bp_parents, info):
    """Generated tokens of one finished slot {step, parent row, token, finished}: the parent row's history through the back-pointers,
    then the token.  An unfinished slot is the empty hypothesis (transformers returns the bare prompt there)."""
    step, row, tok, fin = (int(v) for v in info)
    if not fin:
        return []
    out = [tok]
    for s in range(step - 1, -1, -1):
        out.append(int(bp_tokens[s, row]))
        row = int(bp_parents[s, row])
    return out[::-1]
