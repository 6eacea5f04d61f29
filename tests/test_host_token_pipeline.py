"""The per-step token stages of generate() on CPU, through the C-ABI double: for every combination of the pick (greedy, or sampled
with a seed), the logits processors (none, repetition_penalty alone, presence_penalty with logit_bias, min_new_tokens with a large EOS
bias), structured outputs (where allowed) and logprobs, at batch 1 and 3, generate() returns the tokens and logprobs of a reference
loop that drives the decode step without its advance and calls the kernels in the documented order (structured-output mask ->
processors -> pick and advance -> processor and automaton update -> logprobs), and it launches each per-step kernel as often as that
order asks: the sparse repetition-penalty kernel when repetition_penalty is the only processor, none at all for neutral values, and
the decode step with its fused greedy advance when nothing else is asked."""
import itertools
from collections import Counter

import numpy as np
import pytest
import torch

from tests.logit_proc_double import LogitProcDouble
from tests.test_host_model import _build

EOS = 998
STEPS = 5
PER_STEP = ("greedy_advance", "sample_advance", "rep_penalty_apply", "rep_penalty_mark", "logit_proc_apply", "logit_proc_update",
            "struct_mask_apply", "struct_advance", "logprobs")
SAMPLING = dict(temperature=0.8, top_k=20, top_p=0.9, seed=7)
PROCS = {"none": {}, "rep": dict(repetition_penalty=1.3), "presence_bias": dict(presence_penalty=0.6, logit_bias={97: 3.0, 101: -2.0}),
         "min_tokens": dict(min_new_tokens=3, logit_bias={EOS: 50.0})}
CHOICE = {"choice": ["yes", "no", "maybe"]}
PROMPTS = {1: ["abcabc abc"], 3: ["a", "bb b", "the rain in spain"]}


class CountingDouble(LogitProcDouble):
    """The logits-processor double, counting its calls of every per-step kernel."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.n = Counter()

    def __getattribute__(self, name):
        f = super().__getattribute__(name)
        if name in PER_STEP:
            def counted(*a, **k):
                self.n[name] += 1
                return f(*a, **k)
            return counted
        return f


@pytest.fixture
def cabi_double(cabi_double, monkeypatch):
    from chatts_b200 import _cabi
    dbl = CountingDouble()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: dbl)
    return dbl


def _reference(model, enc, sampled, procs, structured, lpk):
    """Tokens [B, STEPS] and logprobs (when lpk is not None) of the documented order, with the kernels called directly."""
    from chatts_b200 import structured as smod
    c, dev, V, ps = model.ctx, model.device, model.config.vocab_size, model.page_size
    ids_cpu, am_cpu, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], None)
    B = ids_cpu.shape[0]
    pts, held = model._alloc_pages(lay.lens, STEPS)
    try:
        logits = model._prefill(lay, counts, None, pts)
        st = model._decode_state(B, STEPS)
        lens = torch.from_numpy(lay.lens.astype(np.int32))
        st.page_table.copy_(torch.from_numpy(pts))
        st.positions.copy_(lens - 1)
        st.seq_lens.copy_(lens)
        st.step_ptr.zero_()
        auto = sstate = None
        if structured:
            auto = smod.AutomatonCache(c, dev).get(smod.resolve(CHOICE), None, V, {EOS})
            sstate = torch.zeros(B, dtype=torch.int32)
        words = (V + 31) // 32
        seen = torch.zeros(B, words, dtype=torch.int32)
        kw = PROCS[procs]
        if procs == "rep":
            rr, cc = np.nonzero(am_cpu)
            c.rep_penalty_mark(torch.from_numpy(ids_cpu[rr, cc].astype(np.int32)), torch.from_numpy(rr.astype(np.int32)), seen, V)
        elif procs != "none":
            bias = torch.zeros(1, V)
            for t, v in kw["logit_bias"].items():
                bias[0, t] = v
            par = dict(rep=torch.ones(B), presence=torch.full((B,), kw.get("presence_penalty", 0.0)), frequency=torch.zeros(B),
                       seen=seen, counts=torch.zeros(B, V, dtype=torch.int16) if "presence_penalty" in kw else None, bias=bias,
                       bias_row=torch.zeros(B, dtype=torch.int32), n_generated=torch.zeros(B, dtype=torch.int32),
                       min_tokens=torch.full((B,), kw.get("min_new_tokens", 0), dtype=torch.int32),
                       stop_ids=torch.full((B, 1), EOS, dtype=torch.int32) if "min_new_tokens" in kw else None)
        k = lpk or 0
        lp, rank = torch.zeros(B, STEPS), torch.zeros(B, STEPS, dtype=torch.int32)
        top_ids, top_lp = torch.zeros(B, STEPS, k, dtype=torch.int32), torch.zeros(B, STEPS, k)
        ws, cnt = torch.zeros(2), torch.zeros(B, dtype=torch.int32)
        adv = (st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.page_table, ps)
        for step in range(STEPS):
            if step:
                model._decode_step(st, sample=False)
                logits = st.full_logits
            if auto is not None:
                c.struct_mask_apply(logits, B, sstate, auto.allowed)
            if procs == "rep":
                c.rep_penalty_apply(logits, B, seen, 1.3)
            elif procs != "none":
                c.logit_proc_apply(logits, B, *par.values(), vocab=V)
            if sampled:
                c.sample_advance(logits, B, SAMPLING["temperature"], SAMPLING["top_k"], SAMPLING["top_p"], SAMPLING["seed"], *adv)
            else:
                c.greedy_advance(logits, B, *adv)
            if procs == "rep":
                c.rep_penalty_mark(st.cur_ids, None, seen, V)
            elif procs != "none":
                c.logit_proc_update(st.cur_ids, B, seen, par["counts"], par["n_generated"], V)
            if auto is not None:
                c.struct_advance(st.cur_ids, B, sstate, auto.trans, auto.offsets, auto.data, auto.stops)
            if lpk is not None:
                c.logprobs(logits, B, st.out_tokens, k, lp, rank, top_ids, top_lp, ws, cnt, step_ptr=st.step_ptr, vocab=V)
        toks = st.out_tokens[:, :STEPS].numpy().copy()
    finally:
        model.pool.release(held)
    return toks, (lp.numpy(), rank.numpy(), top_ids.numpy(), top_lp.numpy())


CASES = [(s, p, so, lpk, b) for s, p, so, lpk, b in itertools.product((False, True), PROCS, (False, True), (None, 2), (1, 3))
         if not (so and p == "min_tokens")]


@pytest.mark.parametrize("sampled,procs,structured,lpk,batch", CASES)
def test_generate_matches_documented_order(cabi_double, sampled, procs, structured, lpk, batch):
    _, _, model, proc = _build(cabi_double)
    enc = proc(text=PROMPTS[batch], timeseries=[], padding=True, return_tensors="pt")
    S = enc["input_ids"].shape[1]
    want, want_lp = _reference(model, enc, sampled, procs, structured, lpk)

    modes = []
    step = model._decode_step
    model._decode_step = lambda st, sample=True: (modes.append(sample), step(st, sample))
    kw = dict(PROCS[procs], eos_token_id=EOS, logprobs=lpk)
    if sampled:
        kw.update(do_sample=True, **SAMPLING)
    if structured:
        kw["structured_outputs"] = CHOICE
    cabi_double.n.clear()
    got = model.generate(**enc, max_new_tokens=STEPS, **kw)[:, S:].numpy()

    # tokens: each row as the reference, cut after its first EOS and padded to the longest row
    ends = [list(r).index(EOS) + 1 if EOS in r else STEPS for r in want]
    n_out = max(ends)
    assert got.shape == (batch, n_out)
    for b in range(batch):
        assert got[b].tolist() == want[b, :ends[b]].tolist() + [model.config.pad_token_id] * (n_out - ends[b]), (b, got, want)
    if lpk is not None:
        res = model.last_logprobs
        lp, rank, ids, vals = (a[:, :n_out].copy() for a in want_lp)
        if structured:                            # a token the automaton refused: an empty top-k slot
            gone = np.isneginf(vals)
            ids[gone], vals[gone] = -1, np.nan
        np.testing.assert_array_equal(res.logprobs, lp)
        np.testing.assert_array_equal(res.ranks, rank)
        np.testing.assert_array_equal(res.top_ids, ids)
        np.testing.assert_array_equal(res.top_logprobs, vals)
    else:
        assert model.last_logprobs is None

    # launches: one prefill pick, then STEPS - 1 decode steps
    fused = not sampled and procs == "none" and not structured
    assert modes == [fused] * (STEPS - 1)
    n = {k: v for k, v in cabi_double.n.items() if v}
    expect = {("sample_advance" if sampled else "greedy_advance"): STEPS}
    if structured:
        expect.update(struct_mask_apply=STEPS, struct_advance=STEPS)
    if procs == "rep":
        expect.update(rep_penalty_apply=STEPS, rep_penalty_mark=1 + STEPS)
    elif procs != "none":
        expect.update(logit_proc_apply=STEPS, logit_proc_update=STEPS)
    if lpk is not None:
        expect["logprobs"] = STEPS
    assert n == expect
