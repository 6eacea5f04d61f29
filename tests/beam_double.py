"""TEST INFRASTRUCTURE ONLY: the two kernels of csrc/beam.cu restated with numpy in the same fp32 arithmetic, as the CPU statement the
kernel tests compare against and as the ``beam_*`` entry points of the torch test double (tests/cabi_double.py) for the host tests;
plus ``beam_search``, a whole beam search driven by a log-prob function through the same restatement, which the host tests check
against transformers' ``generate(num_beams=...)``."""
import numpy as np
import torch

from chatts_b200 import beam as beammod
from tests.structured_double import StructuredDouble

F32 = np.float32
BIG = F32(-1.0e9)


def row_candidates(log_probs, keep):
    """Per row the top ``keep`` (ids int32, log-probs fp32) of fp32 log-probs [R, V], by value descending then the smaller id (the order
    of cts_logprobs)."""
    lp = np.asarray(log_probs, dtype=np.float32)
    R, V = lp.shape
    ids = np.empty((R, keep), dtype=np.int32)
    for r in range(R):
        ids[r] = np.lexsort((np.arange(V), -lp[r]))[:keep]
    return ids, np.take_along_axis(lp, ids.astype(np.int64), 1)


def select_reference(B, nb, keep, vocab, cand_ids, cand_lp, eos, den, max_new, early_stopping, length_penalty, run, fin_scores, fin_info,
                     flags, step_ptr, bp_tok, bp_par, cur_ids, positions, seq_lens, slot_map, table, own, spare, page_size, fork):
    """cts_beam_select on numpy arrays, updated in place (shapes as in include/chatts_b200.h; early_stopping 0 / 1 / 2)."""
    s = int(step_ptr[0])
    eos = set(int(e) for e in eos)
    R = B * nb
    old_table = table.copy()
    max_pages = table.shape[1]
    cand_ids, cand_lp = cand_ids.reshape(R, keep), cand_lp.reshape(R, keep)
    for b in range(B):
        r0 = b * nb
        old_run = run[r0:r0 + nb].copy()
        cands = []
        for j in range(nb):
            for i in range(keep):
                idx, lp = int(cand_ids[r0 + j, i]), F32(cand_lp[r0 + j, i])
                ok = 0 <= idx < vocab and lp == lp
                cands.append((F32(old_run[j] + lp) if ok else F32(-np.inf), j * vocab + idx if ok else nb * vocab + j * keep + i))
        cands.sort(key=lambda t: (-float(t[0]), t[1]))
        top = cands[:keep]
        t_score = [v for v, _ in top]
        t_tok = [f % vocab if f < nb * vocab else -1 for _, f in top]
        t_beam = [f // vocab if f < nb * vocab else 0 for _, f in top]
        t_hit = [s + 1 >= max_new or t in eos for t in t_tok]
        r_val = [F32(v + BIG) if h else v for v, h in zip(t_score, t_hit)]
        sel = sorted(range(keep), key=lambda c: (-float(r_val[c]), c))[:nb]
        if not flags[b, 1]:
            unsat = bool(flags[b, 0])
            full = early_stopping == 1 and all(fin_info[r0:r0 + nb, 3] != 0)
            merged = [(F32(fin_scores[r0 + i]), tuple(int(v) for v in fin_info[r0 + i])) for i in range(nb)]
            for c in range(keep):
                q = F32(t_score[c] / F32(den[min(s + 1, max_new)]))
                if full:
                    q = F32(q + BIG)
                if not unsat:
                    q = F32(q + BIG)
                did = t_hit[c] and c < nb
                if not did:
                    q = F32(q + BIG)
                merged.append((q, (s, r0 + t_beam[c], t_tok[c], int(did))))
            order = sorted(range(nb + keep), key=lambda u: (-float(merged[u][0]), u))[:nb]
            for i, u in enumerate(order):
                fin_scores[r0 + i] = merged[u][0]
                fin_info[r0 + i] = merged[u][1]
            best_len = max_new if (early_stopping == 2 and length_penalty > 0) else s + 1
            best = F32(r_val[sel[0]] / F32(den[best_len]))
            worst = F32(fin_scores[r0:r0 + nb].min())
            fins = fin_info[r0:r0 + nb, 3] != 0
            unsat_new = unsat and any(best > (worst if f else BIG) for f in fins)
            flags[b, 0] = int(unsat_new)
            flags[b, 1] = int((not unsat_new) or (early_stopping == 1 and bool(fins.all())) or all(t_hit))
        for i in range(nb):
            r, c = r0 + i, sel[i]
            parent = r0 + t_beam[c]
            pos = int(positions[r]) + 1
            pg, off = pos // page_size, pos % page_size
            f = (0, 0, 0)
            slot = -1
            if pg < max_pages:
                table[r, :pg] = old_table[parent, :pg]
                if off == 0:
                    tail = int(own[r, pg])
                elif parent != r:
                    tail = int(spare[r])
                    spare[r] = old_table[r, pg]
                    f = (int(old_table[parent, pg]), tail, off)
                else:
                    tail = int(old_table[r, pg])
                table[r, pg] = tail
                slot = tail * page_size + off
            else:
                table[r, :max_pages] = old_table[parent, :max_pages]
            fork[r] = f
            if s < max_new:
                bp_tok[s, r], bp_par[s, r] = t_tok[c], parent
            run[r] = r_val[c]
            cur_ids[r] = max(t_tok[c], 0)
            positions[r] = pos
            seq_lens[r] += 1
            slot_map[r] = slot
    step_ptr[0] = s + 1
    step_ptr[1] = 0


def fork_reference(kv, fork, rows):
    """cts_beam_fork_kv on kv [L, 2, P, nkv, page, d]: all copies read the cache as it was before the launch."""
    src = kv.clone() if isinstance(kv, torch.Tensor) else kv.copy()
    for r in range(rows):
        a, d, n = (int(v) for v in fork[r])
        if n > 0:
            kv[:, :, d, :, :n] = src[:, :, a, :, :n]


class BeamDouble(StructuredDouble):
    """The structured-outputs double plus cts_beam_select / cts_beam_fork_kv (same arguments as chatts_b200._cabi.Context)."""

    def beam_select(self, batch, num_beams, keep, vocab, cand_ids, cand_logprobs, eos_ids, len_den, max_new, early_stopping,
                    length_penalty, run_scores, fin_scores, fin_info, prompt_flags, step_ptr, bp_tokens, bp_parents, cur_ids, positions,
                    seq_lens, slot_map, page_table, page_table_old, own_pages, spare_pages, page_size, fork):
        R = batch * num_beams
        n = lambda t: t.numpy()                                             # CPU tensors: numpy views share the storage
        select_reference(batch, num_beams, keep, vocab, n(cand_ids), n(cand_logprobs), n(eos_ids).tolist(), n(len_den), max_new,
                         beammod.EARLY_STOPPING[early_stopping], length_penalty, n(run_scores), n(fin_scores), n(fin_info).reshape(R, 4),
                         n(prompt_flags).reshape(batch, 2), n(step_ptr), n(bp_tokens), n(bp_parents), n(cur_ids), n(positions),
                         n(seq_lens), n(slot_map), n(page_table), n(own_pages).reshape(R, -1), n(spare_pages), page_size,
                         n(fork).reshape(R, 3))

    def beam_fork_kv(self, kv, fork, rows):
        fork_reference(kv, fork, rows)


def _merge_margin(vals, nb):
    """Smallest (gap / allowed error) between neighbours among the best nb + 1 of (value, error) pairs (inf with fewer than two)."""
    vals = sorted(vals, key=lambda t: -t[0])[:nb + 1]
    return min([(a[0] - b[0]) / (a[1] + b[1]) for a, b in zip(vals, vals[1:])], default=np.inf)


def beam_search(next_log_probs, prompt_len, B, nb, vocab, max_new, eos=(), length_penalty=1.0, early_stopping=False, nrs=1):
    """A whole beam search through select_reference, without pages: ``next_log_probs(seqs)`` gets the B * nb generated-token lists
    and returns fp32 log-probs [B * nb, vocab] of their next token, or (log-probs, tol) where tol bounds the error of every log-prob
    of that step.  -> (per prompt, nrs lists of generated tokens, best first; scores fp32 [B * nrs]; steps run; margin).

    margin (inf without tolerances): the smallest ratio, over every decision that shapes the output of a prompt not yet done, of the
    distance between the compared scores to the error they can carry, counting a running score of s + 1 tokens as s + 1 times the
    largest tol so far, divided by the length penalty where one applies.  The decisions: which continuations run on (the num_beams-th
    against the next one that does not finish), whether a finishing continuation is among the best num_beams, which finished
    hypotheses are kept and in what order, and the early-stop heuristic's comparison once every finished slot is filled.  Which slot a
    running beam takes does not change the output and is not a decision here.  margin > 1: any log-probs within tol of these give the
    same output."""
    keep = beammod.beams_to_keep(nb, len(eos))
    R = B * nb
    z = lambda *shape, dt=np.int32: np.zeros(shape, dtype=dt)
    run = np.zeros(R, dtype=np.float32)
    run.reshape(B, nb)[:, 1:] = -1e9
    fin_scores = np.full(R, -1e9, dtype=np.float32)
    fin_info, flags, step = z(R, 4), z(B, 2), z(2)
    flags[:, 0] = 1
    bp_tok, bp_par = z(max_new, R), z(max_new, R)
    cur, pos, sl, slot = z(R), np.full(R, prompt_len - 1, dtype=np.int32), np.full(R, prompt_len, dtype=np.int32), z(R)
    big = max_new + prompt_len + 1                                           # one page: the page plan is not exercised here
    table, own, spare, fork = z(R, 1), z(R, 1), z(R), z(R, 3)
    den = beammod.len_den(max_new, length_penalty)
    es = beammod.EARLY_STOPPING[early_stopping]
    seqs = [[] for _ in range(R)]
    steps, tol, margin = 0, 0.0, np.inf
    while steps < max_new:
        got = next_log_probs(seqs)
        lp_all, t = (got if isinstance(got, tuple) else (got, None))
        lp_all = np.asarray(lp_all, dtype=np.float32)
        s = steps
        live = [b for b in range(B) if not flags[b, 1]]
        if t is not None:
            tol = max(tol, float(t))
            err_run = 2 * (s + 1) * tol                            # two running scores of s + 1 log-probs each
            for b in live:
                r0 = b * nb
                sc = (run[r0:r0 + nb, None] + lp_all[r0:r0 + nb]).reshape(-1)
                order = np.argsort(-sc, kind="stable")[:keep + nb + 1]
                hit = [s + 1 >= max_new or int(f % vocab) in set(eos) for f in order]
                free = [float(sc[f]) for f, h in zip(order, hit) if not h]
                if len(free) > nb:                                 # which continuations run on
                    margin = min(margin, (free[nb - 1] - free[nb]) / err_run)
                if hit[nb - 1] or hit[nb]:                         # whether a finishing candidate is among the best num_beams
                    margin = min(margin, float(sc[order[nb - 1]] - sc[order[nb]]) / err_run)
                if flags[b, 0] and not (es == 1 and (fin_info[r0:r0 + nb, 3] != 0).all()):
                    vals = [(float(sc[f]) / den[s + 1], (s + 1) * tol / abs(float(den[s + 1]))) for f, h in zip(order[:nb], hit) if h]
                    vals += [(float(fin_scores[r0 + i]), (fin_info[r0 + i, 0] + 1) * tol / abs(float(den[fin_info[r0 + i, 0] + 1])))
                             for i in range(nb) if fin_info[r0 + i, 3]]
                    margin = min(margin, _merge_margin(vals, nb))  # which hypotheses are kept, and their order
        ids, lps = row_candidates(lp_all, keep)
        select_reference(B, nb, keep, vocab, ids, lps, list(eos), den, max_new, es, length_penalty, run, fin_scores, fin_info, flags, step,
                         bp_tok, bp_par, cur, pos, sl, slot, table, own, spare, big, fork)
        if t is not None:
            bl = max_new if (es == 2 and length_penalty > 0) else s + 1
            for b in live:
                r0 = b * nb
                if flags[b, 0] or (fin_info[r0:r0 + nb, 3] == 0).any():
                    continue                                       # unsatisfied heuristic, or a slot still empty: nothing compared
                w = int(np.argmin(fin_scores[r0:r0 + nb]))
                err = (s + 1) * tol / abs(float(den[bl])) + (fin_info[r0 + w, 0] + 1) * tol / abs(float(den[fin_info[r0 + w, 0] + 1]))
                margin = min(margin, abs(float(run[r0]) / float(den[bl]) - float(fin_scores[r0 + w])) / err)
        steps += 1
        seqs = [beammod.hypothesis(bp_tok, bp_par, (steps - 1, bp_par[steps - 1, r], bp_tok[steps - 1, r], 1)) for r in range(R)]
        if flags[:, 1].all():
            break
    hyps = [[beammod.hypothesis(bp_tok, bp_par, fin_info[b * nb + i]) for i in range(nrs)] for b in range(B)]
    return hyps, np.concatenate([fin_scores[b * nb:b * nb + nrs] for b in range(B)]), steps, margin
