"""Iteration-level ("continuous") batching over the decode step (SURVEY.md 8(f) N3; what the reference gets from vLLM's
scheduler, chatts/utils/llm_utils.py:147-190 / vllm_stream_qa.py:34-59).

The decode step of ``ChatTSForCausalLM`` is one CUDA graph over STATIC per-slot state (current id, position, sequence
length, KV slot, page-table row); nothing in it depends on which requests occupy the slots.  So a request can join or leave
between two replays by rewriting its slot's few integers:

  * admission: waiting requests are prefilled together (TS encode + decoder prefill into freshly allocated KV pages, first
    token by the greedy kernel) and copied into free slots;
  * every round runs ``steps_per_round`` graph replays for ALL slots, then one device->host read of the produced tokens;
    finished requests (EOS / max_new_tokens) free their pages and their slot;
  * free slots keep decoding a dummy sequence inside one reserved scratch page (their work is wasted, never wrong): the graph
    always runs at its full width, the price of never re-capturing.

Greedy decoding; per-row arithmetic does not depend on the other rows, so a request produces the tokens a stand-alone
``generate()`` call produces.  Host logic only (torch copies of a few int32 per slot); every number comes from the kernels.
"""
from collections import deque
from dataclasses import dataclass, field

import numpy as np
import torch


@dataclass
class Request:
    rid: int
    input_ids: torch.Tensor            # [S] un-expanded ids (the <ts><ts/> pairs still in place)
    series: torch.Tensor               # [n_series, 2 Lmax, 1] encoded series of THIS request (may be empty)
    max_new_tokens: int
    eos: set
    ignore_eos: bool = False
    tokens: list = field(default_factory=list)
    slot: int = -1
    pages: list = field(default_factory=list)
    done: bool = False
    error: Exception = None            # set when the request could not be admitted (over-long, or larger than the whole KV pool)


class ContinuousEngine:
    def __init__(self, model, slots=None, steps_per_round=4, max_prefill_batch=8):
        if model.tp_size != 1:
            raise ValueError("ContinuousEngine drives a single-GPU model (tensor-parallel ranks would have to step in lock-step)")
        self.m = model
        self.B = int(slots or model.max_batch)
        if self.B > model.max_batch:
            raise ValueError(f"{self.B} slots exceed the model's max_batch {model.max_batch}")
        self.k = int(steps_per_round)
        self.max_prefill = int(max_prefill_batch)
        self.waiting = deque()
        self.active = {}                                   # slot -> Request
        self.finished = []
        self._next = 0
        self.st = model._decode_state(self.B, max(self.k, 1))
        self.scratch = model.pool.alloc(1)[0]              # dummy sequences of the free slots live here
        dev = model.device
        self.st.page_table.fill_(self.scratch)
        self.st.cur_ids.fill_(int(model.config.pad_token_id) % model.embed.shape[0])
        self._reset_free(list(range(self.B)))
        self.rounds = 0
        self.occupancy = []                                # active slots per round (observability / tests)

    # ------------------------------------------------------------------------------------------ public
    def add_request(self, input_ids, series=None, max_new_tokens=16, eos_token_id=None, ignore_eos=False):
        cfg = self.m.config
        eos = cfg.eos_token_id if eos_token_id is None else eos_token_id
        eos = set(eos) if isinstance(eos, (list, tuple, set)) else {int(eos)}
        ids = torch.as_tensor(input_ids, dtype=torch.long).reshape(-1)
        ts = series if series is not None else torch.zeros(0, 0, 1)
        r = Request(self._next, ids, ts, int(max_new_tokens), eos, ignore_eos)
        self._next += 1
        self.waiting.append(r)
        return r.rid

    def has_work(self):
        return bool(self.waiting or self.active)

    def step(self):
        """One scheduling round: admit, decode ``steps_per_round`` steps, harvest.  Returns the requests finished in it."""
        n0 = len(self.finished)
        self._admit()
        if self.active:
            self._decode_round()
        self.rounds += 1
        return self.finished[n0:]                          # incl. requests that ended with their very first token

    def run(self):
        done = []
        while self.has_work():
            done += self.step()
        return sorted(done, key=lambda r: r.rid)

    def close(self):
        for r in list(self.active.values()):
            self._release(r)
        self.m.pool.release([self.scratch])

    # ------------------------------------------------------------------------------------------ admission
    def _free_slots(self):
        return [s for s in range(self.B) if s not in self.active]

    def _admit(self):
        m = self.m
        free = self._free_slots()
        while self.waiting and free:
            group = []
            while self.waiting and len(group) < min(len(free), self.max_prefill):
                group.append(self.waiting.popleft())
            # one left-padded batch for the group's prefill (the layout drops the padding again)
            S = max(int(r.input_ids.shape[0]) for r in group)
            pad = int(m.config.pad_token_id)
            ids = torch.full((len(group), S), pad, dtype=torch.long)
            am = torch.zeros(len(group), S, dtype=torch.long)
            for i, r in enumerate(group):
                n = int(r.input_ids.shape[0])
                ids[i, S - n:], am[i, S - n:] = r.input_ids, 1
            parts = [r.series for r in group if r.series is not None and r.series.shape[0] > 0]
            if parts:
                L = max(int(p.shape[1]) for p in parts)
                ts = torch.zeros(sum(int(p.shape[0]) for p in parts), L, 1, dtype=parts[0].dtype)
                o = 0
                for p in parts:
                    ts[o: o + p.shape[0], : p.shape[1]] = p
                    o += p.shape[0]
            else:
                ts = None
            try:
                _, _, counts, lay = m._prepare_inputs(ids, am, ts)
                pts, held = m._alloc_pages(lay.lens, max(r.max_new_tokens for r in group) + self.k)
            except RuntimeError as e:                      # KV cache full (_alloc_pages takes nothing when it fails)
                if self.active:                            # pages will come back: put the group back and wait for a release
                    for r in reversed(group):
                        self.waiting.appendleft(r)
                    return
                if len(group) > 1:                         # nothing in flight: retry with the head of the queue alone
                    for r in reversed(group):
                        self.waiting.appendleft(r)
                    self._admit_one()
                    return
                # a single request that does not fit an EMPTY pool can never run: fail it instead of retrying forever
                self._fail(group[0], e)
                continue
            except (ValueError, AssertionError) as e:      # an invalid request (over-long, <ts>/series mismatch) fails alone
                if len(group) == 1:
                    self._fail(group[0], e)
                else:                                      # find the offender(s) by admitting the group one request at a time
                    for r in reversed(group):
                        self.waiting.appendleft(r)
                    saved, self.max_prefill = self.max_prefill, 1
                    try:
                        for _ in range(len(group)):
                            if not self._free_slots():
                                break
                            self._admit_one()
                    finally:
                        self.max_prefill = saved
                    free = self._free_slots()
                continue
            logits = m._prefill(lay, counts, ts, pts)
            # first token + advanced per-sequence state through the greedy kernel on a group-sized scratch state
            g = len(group)
            dev = m.device
            lens32 = torch.from_numpy(lay.lens.astype(np.int32)).to(dev)
            t_out = torch.zeros(g, 1, dtype=torch.int32, device=dev)
            t_step = torch.zeros(2, dtype=torch.int32, device=dev)
            t_cur = torch.zeros(g, dtype=torch.int32, device=dev)
            t_pos, t_seq = lens32 - 1, lens32.clone()
            t_slot = torch.zeros(g, dtype=torch.int32, device=dev)
            t_pt = torch.from_numpy(pts).to(dev)
            m.ctx.greedy_advance(logits, g, t_out, t_step, t_cur, t_pos, t_seq, t_slot, t_pt, m.page_size)
            first = t_out[:, 0].cpu().tolist()             # host read: the request's first token (and EOS check)
            slots = torch.tensor(free[:g], device=dev)
            st = self.st
            st.cur_ids[slots], st.positions[slots], st.seq_lens[slots], st.slot_map[slots] = t_cur, t_pos, t_seq, t_slot
            st.page_table[slots] = t_pt
            for i, r in enumerate(group):
                need = (int(lay.lens[i]) + max(q.max_new_tokens for q in group) + self.k + m.page_size - 1) // m.page_size
                r.pages = [int(x) for x in pts[i, :need]]
                r.slot = free[i]
                r.tokens.append(int(first[i]))
                self.active[r.slot] = r
                self._check_done(r)
            free = free[g:]
            for r in [q for q in group if q.done]:
                self._retire(r)
            free = self._free_slots()

    def _admit_one(self):
        """Admit exactly the request at the head of the queue (used to isolate an invalid request of a failed group)."""
        if not self.waiting:
            return
        head = self.waiting.popleft()
        rest, self.waiting = self.waiting, deque([head])
        try:
            self._admit()
        finally:
            self.waiting.extend(rest)

    def _fail(self, r, err):
        r.error, r.done = err, True
        self.finished.append(r)

    # ------------------------------------------------------------------------------------------ decode
    def _decode_round(self):
        m, st = self.m, self.st
        free = self._free_slots()
        if free:
            self._reset_free(free)
        st.step_ptr.zero_()
        for _ in range(self.k):
            m._decode_step(st, sample=True)
        toks = st.out_tokens[:, : self.k].cpu().numpy()    # the round's one device->host read
        self.occupancy.append(len(self.active))
        out = []
        for slot, r in list(self.active.items()):
            for j in range(self.k):
                if r.done:
                    break
                r.tokens.append(int(toks[slot, j]))
                self._check_done(r)
            if r.done:
                self._retire(r)
                out.append(r)
        return out

    def _check_done(self, r):
        if len(r.tokens) >= r.max_new_tokens or (not r.ignore_eos and r.tokens[-1] in r.eos):
            r.done = True

    def _retire(self, r):
        self._release(r)
        self.finished.append(r)

    def _release(self, r):
        if r.slot in self.active:
            del self.active[r.slot]
        if r.pages:
            self.m.pool.release(r.pages)
            r.pages = []
        if r.slot >= 0:
            self.st.page_table[r.slot].fill_(self.scratch)
            self._reset_free([r.slot])

    def _reset_free(self, slots):
        """Dummy sequence of a free slot: one token at position 0 of the scratch page (restarted every round so that it never
        grows past the page / the RoPE table)."""
        st, ps = self.st, self.m.page_size
        idx = torch.tensor(slots, device=self.m.device)
        st.positions[idx] = 0
        st.seq_lens[idx] = 1
        st.slot_map[idx] = self.scratch * ps
        if self.k >= ps:
            raise ValueError("steps_per_round must be smaller than the KV page size (the dummy sequences stay inside one page)")
