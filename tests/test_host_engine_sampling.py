"""Per-request sampling in the continuous engine (chatts_b200/engine.py) and per-prompt SamplingParams in LLM.generate, on CPU through
the C-ABI double: a sampled request's tokens are generate()'s row seed_row under the same seed, whatever slot and round it lands in;
a list of differing SamplingParams gives each seeded prompt exactly its own single-params LLM.generate (n > 1 included) and an
all-equal list the single-params call; the refusals leave the KV pool as it was; Request.seed replays an unseeded request; a reused
slot is greedy again; and a round launches cts_sample_advance_rows only when some active slot samples (a round whose only non-greedy
slots use processors keeps cts_greedy_advance)."""
from collections import Counter

import pytest
import torch

from tests.sample_rows_double import SampleRowsDouble
from tests.test_host_model import _build

PICKS = ("greedy_advance", "sample_advance", "sample_advance_rows")
SAMPLED = dict(temperature=0.8, top_k=20, top_p=0.9)


class CountingDouble(SampleRowsDouble):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.n = Counter()

    def __getattribute__(self, name):
        f = super().__getattribute__(name)
        if name in PICKS:
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


def _ids(proc, text):
    return proc(text=[text], timeseries=[], return_tensors="pt")["input_ids"][0]


def _generate_rows(model, proc, text, n, steps, **kw):
    enc = proc(text=[text] * n, timeseries=[], padding=True, return_tensors="pt")
    S = enc["input_ids"].shape[1]
    return model.generate(**enc, max_new_tokens=steps, ignore_eos=True, do_sample=True, **kw)[:, S:].tolist()


def test_request_tokens_are_generate_row_seed_row(cabi_double):
    """Three copies of one prompt with seed_row 0..2, next to a greedy and a processor request in a 4-slot engine whose rounds end
    mid-request, give generate(seed=...)'s rows 0..2; the greedy request gives greedy generate()."""
    from chatts_b200.engine import ContinuousEngine
    _, _, model, proc = _build(cabi_double)
    want = _generate_rows(model, proc, "the rain in spain", 3, 7, seed=41, **SAMPLED)
    assert len({tuple(r) for r in want}) > 1                      # the rows draw differently
    greedy_ids = _ids(proc, "plain greedy prompt")
    enc = proc(text=["plain greedy prompt"], timeseries=[], return_tensors="pt")
    greedy_want = model.generate(**enc, max_new_tokens=5, ignore_eos=True)[0, enc["input_ids"].shape[1]:].tolist()
    pages0 = len(model.pool.free)
    eng = ContinuousEngine(model, slots=4, steps_per_round=3)
    g = eng.add_request(greedy_ids, None, max_new_tokens=5, ignore_eos=True)
    eng.add_request(_ids(proc, "with processors"), None, max_new_tokens=4, ignore_eos=True, presence_penalty=0.7, temperature=1.1, seed=3)
    rids = [eng.add_request(_ids(proc, "the rain in spain"), None, max_new_tokens=7, ignore_eos=True, seed=41, seed_row=j, **SAMPLED)
            for j in range(3)]
    done = {r.rid: r for r in eng.run()}
    assert [done[r].tokens for r in rids] == want
    assert done[g].tokens == greedy_want
    eng.close()
    assert len(model.pool.free) == pages0


def test_unseeded_request_replays_from_its_seed(cabi_double):
    """The replay runs on the same engine, so the decode shapes, and with them every logit, are the first run's."""
    from chatts_b200.engine import ContinuousEngine
    _, _, model, proc = _build(cabi_double)
    ids = _ids(proc, "abc abc abc")
    eng = ContinuousEngine(model, slots=2, steps_per_round=2)
    r0 = eng.add_request(ids, None, max_new_tokens=6, ignore_eos=True, temperature=1.0)
    first = eng.run()[0]
    assert first.rid == r0 and first.seed is not None
    eng.add_request(ids, None, max_new_tokens=6, ignore_eos=True, temperature=1.0, seed=first.seed)
    assert eng.run()[0].tokens == first.tokens
    eng.close()


def test_reused_slot_is_greedy_again(cabi_double):
    from chatts_b200.engine import ContinuousEngine
    _, _, model, proc = _build(cabi_double)
    enc = proc(text=["greedy after sampled"], timeseries=[], return_tensors="pt")
    want = model.generate(**enc, max_new_tokens=6, ignore_eos=True)[0, enc["input_ids"].shape[1]:].tolist()
    eng = ContinuousEngine(model, slots=1, steps_per_round=2)
    eng.add_request(_ids(proc, "hot sampled request"), None, max_new_tokens=3, ignore_eos=True, temperature=1.5, seed=9)
    eng.add_request(enc["input_ids"][0], None, max_new_tokens=6, ignore_eos=True)
    done = eng.run()
    assert done[0].slot == done[1].slot == 0 and done[1].tokens == want
    assert float(eng._samp.temperature[0]) == 0.0
    eng.close()


@pytest.mark.parametrize("kw", [dict(temperature=float("nan")), dict(temperature=float("inf")), dict(temperature=-0.1),
                                dict(temperature=1.0, top_k=-2), dict(temperature=1.0, top_p=0.0), dict(temperature=1.0, top_p=1.5)])
def test_add_request_refuses_bad_values_before_queueing(cabi_double, kw):
    from chatts_b200.engine import ContinuousEngine
    _, _, model, proc = _build(cabi_double)
    eng = ContinuousEngine(model, slots=2)
    with pytest.raises(ValueError):
        eng.add_request(_ids(proc, "x"), None, max_new_tokens=2, **kw)
    assert not eng.waiting
    eng.close()


def test_round_launches(cabi_double):
    """Greedy slots only: the plain graph's greedy advance every step and no cts_sample_advance_rows.  A processor slot and no sampled
    one: the greedy advance after the processors, as before.  A sampled slot: one cts_sample_advance_rows per step (admission
    included) and no greedy advance."""
    from chatts_b200.engine import ContinuousEngine
    _, _, model, proc = _build(cabi_double)
    eng = ContinuousEngine(model, slots=2, steps_per_round=3)
    eng.add_request(_ids(proc, "greedy one"), None, max_new_tokens=4, ignore_eos=True)
    cabi_double.n.clear()
    eng.step()
    assert dict(cabi_double.n) == {"greedy_advance": 1 + 3}
    eng.run()
    eng.add_request(_ids(proc, "with processors"), None, max_new_tokens=4, ignore_eos=True, presence_penalty=0.5)
    cabi_double.n.clear()
    eng.step()
    assert dict(cabi_double.n) == {"greedy_advance": 1 + 3}
    eng.run()
    eng.add_request(_ids(proc, "greedy two"), None, max_new_tokens=4, ignore_eos=True)
    eng.add_request(_ids(proc, "sampled"), None, max_new_tokens=4, ignore_eos=True, temperature=0.7, seed=1)
    cabi_double.n.clear()
    eng.step()
    assert dict(cabi_double.n) == {"sample_advance_rows": 1 + 3}
    eng.close()


PROMPTS = ["first prompt", "second, a little longer prompt", "third"]


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.prompt == y.prompt and len(x.outputs) == len(y.outputs)
        for p, q in zip(x.outputs, y.outputs):
            assert (p.token_ids, p.text, p.finish_reason, p.logprobs, p.cumulative_logprob) == \
                   (q.token_ids, q.text, q.finish_reason, q.logprobs, q.cumulative_logprob)


def test_llm_per_prompt_params_equal_single_prompt_calls(cabi_double):
    from chatts_b200.vllm_compat import LLM, SamplingParams
    _, _, model, proc = _build(cabi_double)
    llm = LLM(model=model)
    sps = [SamplingParams(max_tokens=6, temperature=0.8, top_p=0.9, seed=11, n=3, ignore_eos=True),
           SamplingParams(max_tokens=5, logprobs=2, stop_token_ids=[101], min_tokens=1),
           SamplingParams(max_tokens=7, temperature=1.2, top_k=30, seed=5, presence_penalty=0.5, logprobs=1, ignore_eos=True)]
    pages0 = len(model.pool.free)
    got = llm.generate(PROMPTS, sps)
    assert len(model.pool.free) == pages0
    want = [llm.generate([p], sp)[0] for p, sp in zip(PROMPTS, sps)]
    _same(got, want)
    assert len({tuple(o.token_ids) for o in got[0].outputs}) > 1


def test_llm_all_equal_list_is_the_single_params_call(cabi_double):
    from chatts_b200.vllm_compat import LLM, SamplingParams
    _, _, model, proc = _build(cabi_double)
    llm = LLM(model=model)
    sp = dict(max_tokens=5, temperature=0.9, seed=2, n=2, logprobs=1)
    _same(llm.generate(PROMPTS, [SamplingParams(**sp) for _ in PROMPTS]), llm.generate(PROMPTS, SamplingParams(**sp)))


@pytest.mark.parametrize("case", ["length", "structured", "prompt_logprobs", "streamer"])
def test_llm_per_prompt_refusals_leave_the_pool(cabi_double, case):
    from chatts_b200.vllm_compat import LLM, SamplingParams
    _, _, model, proc = _build(cabi_double)
    llm = LLM(model=model)
    sps = [SamplingParams(max_tokens=3), SamplingParams(max_tokens=4, temperature=0.5, seed=1), SamplingParams(max_tokens=2)]
    kw = {}
    if case == "length":
        sps = sps[:2]
    elif case == "structured":
        sps[2] = SamplingParams(max_tokens=4, structured_outputs={"choice": ["yes", "no"]})
    elif case == "prompt_logprobs":
        sps[0] = SamplingParams(max_tokens=3, prompt_logprobs=1)
    else:
        kw["streamer"] = object()
    pages0 = len(model.pool.free)
    with pytest.raises(ValueError):
        llm.generate(PROMPTS, sps, **kw)
    assert len(model.pool.free) == pages0
