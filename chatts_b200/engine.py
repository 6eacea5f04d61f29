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

Per-row arithmetic does not depend on the other rows, so a greedy request produces the tokens a stand-alone ``generate()`` call
produces.  A request may sample (temperature, top_k, top_p, seed) and may carry vLLM's logits processors (chatts_b200.logit_proc), one
parameter set per slot.  A round in which some active slot samples or uses processors runs each step as the decode step without its
advance followed by the stages of chatts_b200.token_pipeline.  Their pick is cts_sample_advance_rows when some active slot samples
(greedy slots, free ones included, take cts_greedy_advance's token, sampled ones their own draw) and cts_greedy_advance otherwise.  A
round in which no active slot does either replays the plain graph.

The draw rule: token i of a sampled request is drawn with u(seed, i, seed_row), the draw generate(seed=seed) makes for its row
seed_row at step i.  It depends neither on the slot the request lands in nor on the round its steps fall in, so a seeded request is
reproducible, and n requests for one prompt with one seed and seed_row = 0..n-1 give the n completions of
``LLM.generate([prompt], SamplingParams(n=n, seed=seed))``.  An unseeded request draws a fresh seed, kept in ``Request.seed``.
Host logic only (torch copies of a few numbers per slot); every number comes from the kernels.
"""
import math
import os
from collections import deque
from dataclasses import dataclass, field
from types import SimpleNamespace

import numpy as np
import torch

from . import logit_proc as lpmodp
from . import logprobs as lpmod
from ._cabi import LOGPROBS_MAX_K
from .token_pipeline import SamplingState, TokenPipeline, stop_ids


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
    cached_positions: int = 0          # prompt positions whose KV came from the prefix cache (model built with enable_prefix_caching)
    logprobs: int = None               # top-k of the logprobs asked for (None: none)
    token_logprobs: list = field(default_factory=list)   # per token: (logprob, rank, top-k ids, top-k logprobs), as in generate()
    procs: lpmodp.Processors = None    # logits processors (None: none)
    temperature: float = 0.0           # 0: greedy (top_k, top_p and seed unused)
    top_k: int = 0                     # 0 or -1: off
    top_p: float = 1.0
    seed: int = None                   # the seed the request's tokens were drawn with (None for a greedy request)
    seed_row: int = 0                  # the draw key: token i is u(seed, i, seed_row), generate(seed=seed)'s row seed_row at step i

    @property
    def samples(self):
        return self.temperature > 0


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
        self._lpb = None                                   # logprob outputs of a round, made when a request first asks
        self._proc = None                                  # per-slot logits processors, made when a request first asks
        self._samp = SamplingState(model.ctx, self.B, dev)  # per-slot sampling parameters (free slots: greedy)

    # ------------------------------------------------------------------------------------------ public
    def add_request(self, input_ids, series=None, max_new_tokens=16, eos_token_id=None, ignore_eos=False, logprobs=None,
                    presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=None, logit_bias=None, allowed_token_ids=None,
                    min_tokens=None, temperature=0.0, top_k=0, top_p=1.0, seed=None, seed_row=0):
        """logprobs = k (0..20): every token's logprob and rank and the k most likely tokens, in Request.token_logprobs.
        presence_penalty, frequency_penalty, repetition_penalty, logit_bias, allowed_token_ids, min_tokens: the logits processors of
        generate() (its min_new_tokens is min_tokens here), from the first token on.
        temperature > 0 samples with top_k (0 or -1: off) and top_p in (0, 1]; token i is drawn with u(seed, i, seed_row), as
        generate(seed=seed) draws its row seed_row at step i; seed None draws a fresh one (kept in Request.seed).  temperature 0 is
        greedy and ignores the other three.  ValueError on a bad value, before anything is queued."""
        temperature = float(temperature)
        if not (math.isfinite(temperature) and temperature >= 0):
            raise ValueError(f"temperature must be a finite number >= 0, got {temperature}")
        top_k, top_p = int(top_k or 0), float(top_p)
        if top_k < -1:
            raise ValueError(f"top_k must be -1, 0 (off) or a positive count, got {top_k}")
        if not 0 < top_p <= 1:
            raise ValueError(f"top_p must be in (0, 1], got {top_p}")
        if not 0 <= int(seed_row) < 1 << 31:
            raise ValueError(f"seed_row must be in [0, 2^31), got {seed_row}")
        if temperature > 0 and seed is None:
            seed = int.from_bytes(os.urandom(8), "little")          # a fresh seed, kept so that the request can be replayed
        k = lpmod.check_k(logprobs, "logprobs")
        cfg = self.m.config
        procs = lpmodp.resolve(presence_penalty, frequency_penalty, repetition_penalty, logit_bias, allowed_token_ids, min_tokens,
                               max_new_tokens, vocab=cfg.vocab_size)
        eos = stop_ids(eos_token_id, cfg.eos_token_id)
        lpmodp.check_stop_ids(procs, [] if ignore_eos else eos)
        ids = torch.as_tensor(input_ids, dtype=torch.long).reshape(-1)
        ts = series if series is not None else torch.zeros(0, 0, 1)
        r = Request(self._next, ids, ts, int(max_new_tokens), eos, ignore_eos, logprobs=k, procs=procs)
        if temperature > 0:
            r.temperature, r.top_k, r.top_p, r.seed, r.seed_row = temperature, top_k, top_p, int(seed), int(seed_row)
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
                pts, held, keys, cached = m._alloc_prompt(lay, ts, max(r.max_new_tokens for r in group) + self.k)
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
            logits = m._prefill(lay, counts, ts, pts, cached=cached)
            m._prefix_register(keys, pts, lay.lens, cached)
            # first token + advanced per-sequence state through the pipeline on a group-sized scratch state, processor rows = the slots
            # taken.  A row without processors maps to a free slot, whose parameters are neutral (never set, or reset by _release):
            # the apply kernel returns at once for it.
            g = len(group)
            dev = m.device
            lens32 = torch.from_numpy(lay.lens.astype(np.int32)).to(dev)
            i32 = dict(dtype=torch.int32, device=dev)
            t = SimpleNamespace(out_tokens=torch.zeros(g, 1, **i32), step_ptr=torch.zeros(2, **i32), cur_ids=torch.zeros(g, **i32),
                                positions=lens32 - 1, seq_lens=lens32.clone(), slot_map=torch.zeros(g, **i32),
                                page_table=torch.from_numpy(pts).to(dev))
            prows = [i for i, r in enumerate(group) if r.procs is not None]
            if prows:
                self._set_procs([group[i] for i in prows], [free[i] for i in prows])
            for i, r in enumerate(group):
                if r.samples:
                    self._samp.set_rows([free[i]], r.temperature, r.top_k, r.top_p, r.seed, r.seed_row)
            samples = any(r.samples for r in group)
            ks = [r.logprobs for r in group if r.logprobs is not None]
            lpb = lpmod.LogprobBuffers(m.ctx, g, 1, max(ks), m.config.vocab_size, dev) if ks else None
            TokenPipeline(m.ctx, t, g, m.page_size, sampling=self._samp if samples else None, processors=self._proc if prows else None,
                          slots=free[:g], logprobs=(lpb, max(ks)) if ks else None).step(logits)
            first = t.out_tokens[:, 0].cpu().tolist()           # host read: the request's first token (and EOS check)
            if ks:
                first_lp = lpb.host(1)
            slots = torch.tensor(free[:g], device=dev)
            st = self.st
            st.cur_ids[slots], st.positions[slots], st.seq_lens[slots], st.slot_map[slots] = t.cur_ids, t.positions, t.seq_lens, t.slot_map
            st.page_table[slots] = t.page_table
            for i, r in enumerate(group):
                need = (int(lay.lens[i]) + max(q.max_new_tokens for q in group) + self.k + m.page_size - 1) // m.page_size
                r.pages = [int(x) for x in pts[i, :need]]
                r.slot = free[i]
                r.cached_positions = int(cached[i]) if cached is not None else 0
                r.tokens.append(int(first[i]))
                if r.logprobs is not None:
                    r.token_logprobs.append(self._entry(first_lp, i, 0, r.logprobs))
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

    def _set_procs(self, reqs, slots):
        m = self.m
        if self._proc is None:
            self._proc = lpmodp.LogitProcState(m.ctx, self.B, m.config.vocab_size, m.n_pos, m.device)
        for r, slot in zip(reqs, slots):
            self._proc.set_rows([slot], r.procs, [] if r.ignore_eos else r.eos, shared_bias=False)
            if r.procs.repetition_penalty != 1:            # the prompt ids, as generate() marks them
                tok = r.input_ids.to(torch.int32).to(m.device)
                self._proc.mark_prompt(tok, torch.full_like(tok, slot))

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
        ks = [r.logprobs for r in self.active.values() if r.logprobs is not None]
        if ks and self._lpb is None:
            self._lpb = lpmod.LogprobBuffers(m.ctx, self.B, self.k, LOGPROBS_MAX_K, m.config.vocab_size, m.device)
        procs = any(r.procs is not None for r in self.active.values())
        samples = any(r.samples for r in self.active.values())
        pipe = TokenPipeline(m.ctx, st, self.B, m.page_size, sampling=self._samp if samples else None,
                             processors=self._proc if procs else None,
                             logprobs=(self._lpb, max(ks)) if ks else None)          # logprobs: all slots at the largest k asked
        for _ in range(self.k):
            m._decode_step(st, sample=pipe.fused)
            pipe.step()
        toks = st.out_tokens[:, : self.k].cpu().numpy()    # the round's one device->host read
        lps = self._lpb.host(self.k, max(ks)) if ks else None
        self.occupancy.append(len(self.active))
        out = []
        for slot, r in list(self.active.items()):
            for j in range(self.k):
                if r.done:
                    break
                r.tokens.append(int(toks[slot, j]))
                if r.logprobs is not None:
                    r.token_logprobs.append(self._entry(lps, slot, j, r.logprobs))
                self._check_done(r)
            if r.done:
                self._retire(r)
                out.append(r)
        return out

    @staticmethod
    def _entry(host, row, col, k):
        lp, rank, ids, vals = host
        return float(lp[row, col]), int(rank[row, col]), ids[row, col, :k].tolist(), vals[row, col, :k].tolist()

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
            if r.procs is not None:
                self._proc.reset_rows([r.slot])
            if r.samples:
                self._samp.reset_rows([r.slot])
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
