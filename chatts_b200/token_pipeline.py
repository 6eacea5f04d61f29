"""The per-step token stages of generate() and the continuous engine, after the decode step (or the prefill) has written a logits
buffer [rows, >= V].  Each step runs, on the device and with no host round trip:

  1. the structured-output mask: the logits of the tokens a row's automaton refuses become -inf (cts_struct_mask_apply);
  2. the logits processors (chatts_b200.logit_proc states their order): cts_rep_penalty_apply when repetition_penalty is the only one
     set, cts_logit_proc_apply otherwise;
  3. the pick and advance of every row's decode state: cts_greedy_advance; cts_sample_advance with temperature / top-k / top-p and a
     draw that is a function of (seed, step, row), one parameter set for every row (generate()); or cts_sample_advance_rows with each
     row's own parameters and a draw that is a function of (seed, draw step, draw key) of the row (SamplingState: the engine's slots);
  4. the processor update (the new token's occurrence bit and count) and the automaton's walk over the new token;
  5. the logprobs (cts_logprobs) of the logits the token was picked from, at the column the advance wrote.

When nothing but a greedy pick is asked, the caller replays the decode step with its own advance and the pipeline only adds the
logprobs.  ``resolve_generate`` resolves generate()'s options and refusals before any page is taken."""
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import beam as beammod
from . import logit_proc as lpmodp
from . import logprobs as lpmod
from . import structured


def stop_ids(eos_token_id, default):
    """The set of stop ids of an ``eos_token_id`` argument: one id or a list of ids; None gives ``default``."""
    eos = default if eos_token_id is None else eos_token_id
    return {int(e) for e in (eos if isinstance(eos, (list, tuple, set)) else [eos])}


@dataclass
class GenerateOptions:
    max_new_tokens: int
    eos: set                      # stop ids: empty under ignore_eos
    pad: int
    logprobs: int = None          # top-k of the token logprobs (None: not asked)
    prompt_logprobs: int = None
    automaton: object = None      # the structured-output constraint (structured.DeviceAutomaton)
    procs: object = None          # logit_proc.Processors, repetition_penalty included (None: neutral)
    sampling: tuple = None        # (temperature, top_k, top_p, seed); None: greedy
    beams: int = None             # candidates kept per beam and step (beam.check_args); None: no beam search


def resolve_generate(model, input_ids, *, max_new_tokens, max_length, do_sample, temperature, top_p, top_k, streamer, eos_token_id,
                     pad_token_id, ignore_eos, seed, repetition_penalty, logprobs, prompt_logprobs, structured_outputs, tokenizer, num_beams,
                     length_penalty, early_stopping, num_return_sequences, num_beam_groups, diversity_penalty, presence_penalty,
                     frequency_penalty, logit_bias, allowed_token_ids, min_new_tokens):
    """generate()'s arguments as GenerateOptions, the checkpoint's generation defaults filled in; each refusal is a ValueError."""
    cfg = model.config
    lpk, plk = lpmod.check_k(logprobs, "logprobs"), lpmod.check_k(prompt_logprobs, "prompt_logprobs")
    if (lpk is not None or plk is not None) and model.tp_size > 1:
        raise ValueError("logprobs / prompt_logprobs are single-GPU only (tensor_parallel_size must be 1)")
    so = structured.resolve(structured_outputs)
    if so is not None and model.tp_size > 1:
        raise ValueError("structured_outputs are single-GPU only (tensor_parallel_size must be 1)")
    if so is not None and ignore_eos:
        raise ValueError("structured_outputs end the output with a stop id: they cannot be combined with ignore_eos")
    # every processor but repetition_penalty, which runs alone under tensor parallelism and is refused with beams by check_args
    procs = lpmodp.resolve(presence_penalty, frequency_penalty, None, logit_bias, allowed_token_ids, min_new_tokens, vocab=cfg.vocab_size)
    if procs is not None:
        if num_beams not in (None, 1):
            raise ValueError("presence_penalty, frequency_penalty, logit_bias, allowed_token_ids and min_new_tokens do not work with "
                             "beam search (num_beams > 1)")
        if model.tp_size > 1:
            raise ValueError("logits processors are single-GPU only (tensor_parallel_size must be 1)")
        if so is not None and (procs.allowed_token_ids is not None or procs.min_tokens > 0):
            raise ValueError("allowed_token_ids and min_new_tokens cannot be combined with structured_outputs: either can refuse "
                             "every token the automaton allows")
    gd = getattr(model, "generation_defaults", None) or {}      # checkpoint defaults apply only where the caller said nothing
    if do_sample is None and gd.get("do_sample"):
        do_sample = True
        temperature = gd.get("temperature", 1.0) if temperature is None else temperature
        top_p = gd.get("top_p") if top_p is None else top_p
        top_k = gd.get("top_k") if top_k is None else top_k
    eos_token_id = gd.get("eos_token_id") if eos_token_id is None else eos_token_id
    pad_token_id = gd.get("pad_token_id") if pad_token_id is None else pad_token_id
    repetition_penalty = gd.get("repetition_penalty") if repetition_penalty is None else repetition_penalty
    if max_new_tokens is None and max_length is None and gd.get("max_new_tokens"):
        max_new_tokens = gd["max_new_tokens"]
    shape = torch.as_tensor(input_ids).shape
    if max_new_tokens is None:
        max_new_tokens = (max_length - shape[-1]) if max_length is not None else 20
    o = GenerateOptions(int(max_new_tokens), set() if ignore_eos else stop_ids(eos_token_id, cfg.eos_token_id),
                        cfg.pad_token_id if pad_token_id is None else pad_token_id, lpk, plk)
    if num_beams not in (None, 1):
        o.beams = beammod.check_args(num_beams, length_penalty, early_stopping, num_return_sequences, len(o.eos),
                                     int(shape[0]) if len(shape) > 1 else 1, model.max_batch, do_sample=do_sample,
                                     num_beam_groups=num_beam_groups, diversity_penalty=diversity_penalty,
                                     repetition_penalty=repetition_penalty, logprobs=logprobs, prompt_logprobs=prompt_logprobs,
                                     structured_outputs=structured_outputs, streamer=streamer, tp_size=model.tp_size)
        return o
    if o.max_new_tokens <= 0:
        return o
    if procs is not None:
        if procs.min_tokens > o.max_new_tokens:
            raise ValueError(f"min_new_tokens ({procs.min_tokens}) must be <= max_new_tokens ({o.max_new_tokens})")
        lpmodp.check_stop_ids(procs, o.eos)
    o.procs = lpmodp.resolve(presence_penalty, frequency_penalty, repetition_penalty, logit_bias, allowed_token_ids, min_new_tokens,
                             vocab=cfg.vocab_size)
    if so is not None:
        # compiled (or found in the cache) before any page is taken: a pattern error leaves the pool as it was
        if getattr(model, "_struct_cache", None) is None:
            model._struct_cache = structured.AutomatonCache(model.ctx, model.device)
        o.automaton = model._struct_cache.get(so, tokenizer, cfg.vocab_size, o.eos)
    if do_sample and temperature is None:
        temperature = 1.0                                   # HF GenerationConfig default when do_sample=True names no temperature
    if do_sample and temperature > 0:
        if seed is None:
            # an unseeded call draws a fresh seed; under tensor parallelism rank 0's seed is broadcast so every rank picks the same tokens
            seed = int.from_bytes(os.urandom(7), "little")
            if model.tp_size > 1:
                box = [seed]
                torch.distributed.broadcast_object_list(box, src=0, group=model.comm)
                seed = int(box[0])
        o.sampling = (temperature, top_k or 0, 1.0 if top_p is None else top_p, int(seed))
    return o


def generate_processors(ctx, procs, ids_cpu, am_cpu, stops, vocab, n_pos, device):
    """The processors state of a generate() batch, whose rows share ``procs``, with the prompt ids (the un-expanded input_ids, as HF
    sees them) marked for the repetition penalty.  repetition_penalty alone keeps the sparse kernels (RepetitionPenaltyState)."""
    if procs is None:
        return None
    B = ids_cpu.shape[0]
    if procs == lpmodp.Processors(repetition_penalty=procs.repetition_penalty):
        state = lpmodp.RepetitionPenaltyState(ctx, B, vocab, procs.repetition_penalty, device)
    else:
        state = lpmodp.LogitProcState(ctx, B, vocab, n_pos, device)
        state.set_rows(list(range(B)), procs, stops, shared_bias=True)
    if procs.repetition_penalty != 1:
        rr, cc = np.nonzero(np.ones_like(ids_cpu) if am_cpu is None else am_cpu)
        state.mark_prompt(torch.from_numpy(ids_cpu[rr, cc].astype(np.int32)).to(device), torch.from_numpy(rr.astype(np.int32)).to(device))
    return state


class SamplingState:
    """Per-row sampling parameters on the device for ``rows`` rows (the continuous engine's slots), read by cts_sample_advance_rows:
    temperature (<= 0: greedy), top_k (<= 0: off), top_p, seed, and the draw of a row's token i, u(seed, draw_step, draw_key) with
    draw_step = i: the kernel adds 1 per token.  A row that was never set, or was reset, is greedy."""

    def __init__(self, ctx, rows, device):
        self.ctx, self.rows, self.dev = ctx, int(rows), device
        f32, i32 = dict(dtype=torch.float32, device=device), dict(dtype=torch.int32, device=device)
        self.temperature, self.top_p = torch.zeros(rows, **f32), torch.ones(rows, **f32)
        self.top_k, self.draw_key, self.draw_step = torch.zeros(rows, **i32), torch.zeros(rows, **i32), torch.zeros(rows, **i32)
        self.seed = torch.zeros(rows, dtype=torch.int64, device=device)

    def set_rows(self, idx, temperature, top_k, top_p, seed, draw_key):
        """Rows ``idx`` (list of ints) start a request with these parameters; its first token is draw 0."""
        ix = torch.as_tensor(idx, dtype=torch.long, device=self.dev)
        self.temperature[ix], self.top_k[ix], self.top_p[ix] = float(temperature), int(top_k), float(top_p)
        s = int(seed) & ((1 << 64) - 1)
        self.seed[ix] = s - (1 << 64) if s >= 1 << 63 else s          # stored as int64, read as uint64
        self.draw_key[ix], self.draw_step[ix] = int(draw_key), 0

    def reset_rows(self, idx):
        self.set_rows(idx, 0.0, 0, 1.0, 0, 0)

    def advance(self, logits, n, out_tokens, step_ptr, cur_ids, positions, seq_lens, slot_map, page_table, page_size, slots=None):
        """Pick and advance logits rows [0, n); ``slots``: logits row i uses state row slots[i] (default: row i)."""
        adv = (out_tokens, step_ptr, cur_ids, positions, seq_lens, slot_map, page_table, page_size)
        if slots is None:
            self.ctx.sample_advance_rows(logits, n, self.temperature, self.top_k, self.top_p, self.seed, self.draw_key, self.draw_step,
                                         *adv)
            return
        ix = torch.as_tensor(slots, dtype=torch.long, device=self.dev)[:n]
        step = self.draw_step[ix]
        self.ctx.sample_advance_rows(logits, n, self.temperature[ix], self.top_k[ix], self.top_p[ix], self.seed[ix], self.draw_key[ix],
                                     step, *adv)
        self.draw_step[ix] = step


class TokenPipeline:
    """The stages above for ``rows`` rows of one logits buffer.  ``st`` holds the advance buffers (out_tokens, step_ptr, cur_ids,
    positions, seq_lens, slot_map, page_table) and, after a decode step, its ``full_logits``.  sampling: (temperature, top_k, top_p,
    seed) for every row, or a SamplingState, or None for greedy; automaton: (structured.DeviceAutomaton, int32 state [rows]);
    processors: a LogitProcState or a RepetitionPenaltyState; when ``slots`` is given, row slots[i] of the processors and of a
    SamplingState belongs to logits row i; logprobs: (LogprobBuffers, k)."""

    def __init__(self, ctx, st, rows, page_size, sampling=None, automaton=None, processors=None, slots=None, logprobs=None):
        self.ctx, self.st, self.rows, self.page_size, self.sampling, self.processors = ctx, st, rows, page_size, sampling, processors
        self.proc_slots = () if slots is None else (slots,)
        self.auto, self.auto_state = automaton or (None, None)
        self.lpb, self.lpk = logprobs or (None, None)
        self.fused = sampling is None and automaton is None and processors is None     # the decode step's own greedy advance

    def step(self, logits=None):
        """One token for every row.  ``logits``: a buffer no step has picked from yet (the prefill's); None: the decode step's
        full_logits, already picked when the step was the fused one."""
        c, st, n = self.ctx, self.st, self.rows
        picked = logits is None and self.fused
        if picked and self.lpb is None:
            return                                # (the tensor-parallel greedy advance leaves no full_logits)
        lg = st.full_logits if logits is None else logits
        if not picked:
            if self.auto is not None:
                self.auto.mask_apply(c, lg, n, self.auto_state)
            if self.processors is not None:
                self.processors.apply(lg, n, *self.proc_slots)
            adv = (st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.page_table, self.page_size)
            if self.sampling is None:
                c.greedy_advance(lg, n, *adv)
            elif isinstance(self.sampling, SamplingState):
                self.sampling.advance(lg, n, *adv, *self.proc_slots)
            else:
                c.sample_advance(lg, n, *self.sampling, *adv)
            if self.processors is not None:
                self.processors.update(st.cur_ids, n, *self.proc_slots)
            if self.auto is not None:
                self.auto.advance(c, st.cur_ids, n, self.auto_state)
        if self.lpb is not None:
            self.lpb.launch(lg, n, st.out_tokens, k=self.lpk, step_ptr=st.step_ptr)
