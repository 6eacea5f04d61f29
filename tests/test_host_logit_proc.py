"""Logits processors on CPU: the statement of csrc/logit_proc.cu (tests/logit_proc_double.py) against vLLM's apply_penalties and its
logit-bias / min-tokens / allowed-ids semantics in fp32; validation of SamplingParams and of the server's request body; and through the
C-ABI double: neutral values launch nothing, greedy generate() with every processor equals a reference loop over the model's per-step
logits, min_new_tokens with a large EOS bias, allowed_token_ids, stop strings inside min_tokens, the refused combinations, the
continuous engine against stand-alone generate(), and the server on both schedulers, streaming included."""
import json

import numpy as np
import pytest
import torch

from tests.logit_proc_double import LogitProcDouble, process_fp32
from tests.test_host_model import _build

EOS = 998


@pytest.fixture
def cabi_double(cabi_double, monkeypatch):
    from chatts_b200 import _cabi
    dbl = LogitProcDouble()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: dbl)
    return dbl


# ------------------------------------------------------------------------------------------------------------------ statement
@pytest.mark.parametrize("rep", [1.0, 2.0, 0.5])
def test_statement_matches_vllm(rep):
    """Steps 1-5 in fp32, before the rounding, equal vLLM v1: allowed mask, logit bias, min-tokens mask, then apply_penalties.  The
    repetition penalties are powers of two, where vLLM's multiplication by 1 / p and this project's division by p agree exactly."""
    utils = pytest.importorskip("vllm.model_executor.layers.utils")
    g = torch.Generator().manual_seed(5)
    B, V = 4, 300
    x = torch.randn(B, V, generator=g) * 4
    x[0, 3], x[1, 7] = float("inf"), float("-inf")
    prompt = torch.randint(0, V, (B, 20), generator=g)
    out = torch.randint(0, 40, (B, 30), generator=g)
    pres = torch.tensor([0.5, -1.25, 0.0, 2.0])
    freq = torch.tensor([0.25, 0.0, -0.75, 1.5])
    reps = torch.full((B,), rep)
    allowed = [None, list(range(0, V, 3)), None, list(range(100))]
    bias = [{5: 3.5, 17: -2.0}, {6: 100.0}, None, {1: -100.0, 250: 7.0}]
    stops, min_active = [[EOS % V, 11], [], [12], [13, 14]], [True, False, True, True]
    want = x.clone()
    for b in range(B):
        if allowed[b] is not None:
            m = torch.ones(V, dtype=torch.bool)
            m[allowed[b]] = False
            want[b].masked_fill_(m, float("-inf"))
        for t, v in (bias[b] or {}).items():
            want[b, t] += v
        if min_active[b] and stops[b]:
            want[b, stops[b]] = float("-inf")
    want = utils.apply_penalties(want, prompt, out, pres, freq, reps)
    from chatts_b200.logit_proc import Processors
    for b in range(B):
        seen = torch.zeros(V, dtype=torch.bool)
        seen[prompt[b]] = True
        seen[out[b]] = True
        vec = Processors(logit_bias=bias[b], allowed_token_ids=allowed[b]).bias_vector(V)
        got, _ = process_fp32(x[b], rep, float(pres[b]), float(freq[b]), seen, torch.bincount(out[b], minlength=V),
                              None if vec is None else torch.from_numpy(vec), stops[b], min_active[b])
        assert torch.equal(got.isnan(), want[b].isnan()) and torch.equal(got[~got.isnan()], want[b][~want[b].isnan()]), b


# ------------------------------------------------------------------------------------------------------------------ validation
def test_sampling_params_validation():
    from chatts_b200.vllm_compat import SamplingParams
    sp = SamplingParams(logit_bias={"5": 250.0, 7: -1e9, "9": 0.5}, presence_penalty=2.0, frequency_penalty=-2.0, min_tokens=3,
                        max_tokens=3, allowed_token_ids=[4, 2, 2])
    assert sp.logit_bias == {5: 100.0, 7: -100.0, 9: 0.5}
    for kw in (dict(presence_penalty=2.5), dict(frequency_penalty=-2.01), dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0),
               dict(min_tokens=-1), dict(min_tokens=17, max_tokens=16), dict(allowed_token_ids=[]), dict(logit_bias={"x": 1.0}),
               dict(logit_bias={-3: 1.0}), dict(allowed_token_ids=[-1])):
        with pytest.raises(ValueError):
            SamplingParams(**kw)
    assert SamplingParams(logit_bias={}).logit_bias == {}
    with pytest.raises(ValueError, match="NaN"):
        SamplingParams(logit_bias={3: float("nan")})
    assert SamplingParams(logit_bias={3: float("inf"), 4: float("-inf")}).logit_bias == {3: 100.0, 4: -100.0}


def test_stop_string_cut_rule():
    """One rule with and without min_tokens: the text ends before the earliest-starting stop string that counts."""
    from chatts_b200.vllm_compat import cut_at_stop_string, cut_at_stop_string_after, tokens_before_stop_string

    class Chars:
        def decode(self, ids, **_):
            return "".join(map(chr, ids))
    tok, ids = Chars(), [ord(c) for c in "xabcyb"]
    for stops in (["abc", "b"], ["b", "abc"], ["c"], ["zz"], ["", "y"]):
        assert cut_at_stop_string_after(tok, ids, stops) == cut_at_stop_string("xabcyb", stops)
    assert cut_at_stop_string_after(tok, ids, ["abc", "b"], min_tokens=1) == ("x", True)       # both end after "x"
    assert cut_at_stop_string_after(tok, ids, ["abc", "b"], min_tokens=2) == ("x", True)       # "abc" still ends after "xa"
    assert cut_at_stop_string_after(tok, ids, ["abc", "b"], min_tokens=3) == ("x", True)       # ... and after "xab"
    assert cut_at_stop_string_after(tok, ids, ["b"], min_tokens=3) == ("xabcy", True)          # the first "b" ends inside "xab"
    assert cut_at_stop_string_after(tok, ids, ["abc"], min_tokens=4) == ("xabcyb", False)
    assert tokens_before_stop_string(tok, ids, ["b"], min_tokens=3) == 6


def test_server_body_parsing():
    from chatts_b200.server import PROCESSOR_FIELDS, _sampling_from_body
    neutral = {"presence_penalty": 0, "frequency_penalty": 0.0, "repetition_penalty": 1.0, "logit_bias": {}, "min_tokens": 0,
               "allowed_token_ids": None}
    assert not set(PROCESSOR_FIELDS) & set(_sampling_from_body(neutral)) and _sampling_from_body(neutral) == _sampling_from_body({})
    p = _sampling_from_body({"presence_penalty": 0.5, "frequency_penalty": -1, "repetition_penalty": 1.2, "logit_bias": {"10": 150},
                             "min_tokens": 2, "allowed_token_ids": [3, 1]}, chat=True)
    assert (p["presence_penalty"], p["frequency_penalty"], p["repetition_penalty"]) == (0.5, -1.0, 1.2)
    assert p["logit_bias"] == {10: 100.0} and p["min_tokens"] == 2 and p["allowed_token_ids"] == [1, 3]
    for bad in ({"presence_penalty": 3}, {"frequency_penalty": -2.5}, {"repetition_penalty": 0}, {"min_tokens": 10, "max_tokens": 5},
                {"allowed_token_ids": []}, {"logit_bias": {"a": 1}}, {"min_tokens": -2}):
        with pytest.raises(ValueError):
            _sampling_from_body(bad)


# ------------------------------------------------------------------------------------------------------------------ generate()
def _enc(proc, texts):
    return proc(text=texts, timeseries=[], padding=True, return_tensors="pt")


def test_neutral_values_launch_nothing(cabi_double):
    _, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["some prompt", "another one here"])
    a = model.generate(**enc, max_new_tokens=6, ignore_eos=True)
    b = model.generate(**enc, max_new_tokens=6, ignore_eos=True, presence_penalty=0.0, frequency_penalty=0.0, logit_bias={},
                       allowed_token_ids=None, min_new_tokens=0)
    assert torch.equal(a, b) and cabi_double.calls == {"apply": 0, "update": 0}
    model.generate(**enc, max_new_tokens=6, ignore_eos=True, presence_penalty=0.5)
    assert cabi_double.calls == {"apply": 6, "update": 6}


def _reference_loop(model, enc, n, rep, pres, freq, bias_vec, stops, min_tokens):
    """Greedy decoding over the model's own next-token logits, processed by the statement and rounded once, before every argmax."""
    hist = enc["input_ids"].clone()
    S = hist.shape[1]
    out = []
    for step in range(n):
        lg = model.forward(hist, torch.ones_like(hist)).logits[:, 0]
        row = []
        for b in range(hist.shape[0]):
            V = lg.shape[-1]
            seen = torch.zeros(V, dtype=torch.bool)
            seen[hist[b]] = True
            counts = torch.bincount(hist[b, S:], minlength=V) if step else torch.zeros(V, dtype=torch.long)
            x, touched = process_fp32(lg[b].float(), rep, pres, freq, seen, counts, bias_vec, stops, step < min_tokens)
            row.append(int(torch.where(touched, x.to(lg.dtype), lg[b]).float().argmax()))
        out.append(row)
        hist = torch.cat([hist, torch.tensor(row)[:, None]], 1)
    return np.array(out).T.tolist()


def test_generate_with_every_processor_matches_reference_loop(cabi_double):
    from chatts_b200.logit_proc import Processors
    _, _, model, proc = _build(cabi_double)
    kw = dict(presence_penalty=0.7, frequency_penalty=0.4, repetition_penalty=1.3, logit_bias={"97": 2.5, 98: -1.0},
              allowed_token_ids=list(range(32, 127)) + [EOS], min_new_tokens=4)
    vec = torch.from_numpy(Processors(logit_bias={97: 2.5, 98: -1.0}, allowed_token_ids=kw["allowed_token_ids"]).bias_vector(1000))
    for text in ["abcabc abc", "the rain in spain"]:
        enc = _enc(proc, [text])
        S = enc["input_ids"].shape[1]
        got = model.generate(**enc, max_new_tokens=10, ignore_eos=True, **kw)[:, S:].tolist()
        assert got == _reference_loop(model, enc, 10, 1.3, 0.7, 0.4, vec, [], 4)
        assert got != model.generate(**enc, max_new_tokens=10, ignore_eos=True)[:, S:].tolist()
    # min_new_tokens: the stop ids are refused for exactly the first 4 tokens
    enc = _enc(proc, ["abcabc abc"])
    S = enc["input_ids"].shape[1]
    kw = dict(logit_bias={EOS: 60.0, 997: 70.0}, min_new_tokens=4, eos_token_id=[EOS, 997])
    got = model.generate(**enc, max_new_tokens=10, **kw)[:, S:].tolist()
    assert got == _reference_loop(model, enc, len(got[0]), 1.0, 0.0, 0.0, torch.from_numpy(Processors(logit_bias=kw["logit_bias"]).bias_vector(1000)),
                                  [EOS, 997], 4) and len(got[0]) == 5 and got[0][-1] == 997


@pytest.mark.parametrize("k", [1, 3, 6])
def test_min_new_tokens_with_eos_bias(cabi_double, k):
    _, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["a", "bb b", "ccc"])
    S = enc["input_ids"].shape[1]
    free = model.pool.available()
    ids = model.generate(**enc, max_new_tokens=12, logit_bias={EOS: 100.0}, min_new_tokens=k)
    for row in ids[:, S:].tolist():
        assert row[:k + 1] == row[:k] + [EOS] and EOS not in row[:k], row
    assert ids.shape[1] == S + k + 1 and model.pool.available() == free


def test_allowed_token_ids(cabi_double):
    _, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["hello there", "x"])
    S = enc["input_ids"].shape[1]
    allowed = [100, 101, 102, 500]
    ids = model.generate(**enc, max_new_tokens=8, allowed_token_ids=allowed)
    assert set(ids[:, S:].reshape(-1).tolist()) <= set(allowed)


def test_refusals_take_nothing(cabi_double):
    _, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["abc", "defg"])
    free = model.pool.available()
    cases = [(dict(presence_penalty=0.5, num_beams=2), "beam"), (dict(min_new_tokens=1, structured_outputs={"choice": ["a"]}), "structured"),
             (dict(allowed_token_ids=[1], structured_outputs={"choice": ["a"]}), "structured"), (dict(logit_bias={1000: 1}), "vocabulary"),
             (dict(allowed_token_ids=[5, 1001]), "vocabulary"), (dict(min_new_tokens=5), "max_new_tokens"),
             (dict(presence_penalty=2.5), r"\[-2, 2\]"), (dict(min_new_tokens=1, eos_token_id=list(range(65))), "64 stop ids"),
             (dict(frequency_penalty=0.1, repetition_penalty=0.0), "repetition_penalty"), (dict(repetition_penalty=0.0), "repetition_penalty")]
    for kw, match in cases:
        with pytest.raises(ValueError, match=match):
            model.generate(**enc, max_new_tokens=4, **kw)
    model.tp_size = 2
    with pytest.raises(ValueError, match="single-GPU"):
        model.generate(**enc, max_new_tokens=4, logit_bias={3: 1.0})
    model.tp_size = 1
    assert model.pool.available() == free and cabi_double.calls["apply"] == 0
    # penalties and logit_bias do combine with structured outputs and with logprobs
    S = enc["input_ids"].shape[1]
    ids = model.generate(**enc, max_new_tokens=8, structured_outputs={"choice": ["up", "down"]}, presence_penalty=1.0,
                         logit_bias={ord("d"): 5.0}, logprobs=2)
    for row in ids[:, S:].tolist():
        assert bytes(row[:row.index(EOS)]).decode() in ("up", "down")


def test_stop_string_inside_min_tokens_is_ignored(cabi_double):
    """A stop string counts only if it ends after the text of the first min_tokens tokens (every token here is one letter)."""
    from chatts_b200.vllm_compat import LLM, SamplingParams
    _, _, model, proc = _build(cabi_double)
    llm = LLM(model=model)
    kw = dict(max_tokens=8, ignore_eos=True, allowed_token_ids=list(range(97, 123)))
    base = llm.generate(["stop test"], SamplingParams(**kw))[0].outputs[0]
    assert len(base.text) == 8
    stop = base.text[1:3]                                   # completes with the third token
    cut = llm.generate(["stop test"], SamplingParams(stop=[stop], **kw))[0].outputs[0]
    assert cut.text == base.text[:1] and cut.finish_reason == "stop"
    two = llm.generate(["stop test"], SamplingParams(stop=[stop], min_tokens=2, **kw))[0].outputs[0]
    assert two.text == cut.text                             # ends after the first 2 tokens: it counts
    j = base.text.find(stop, 2)                             # with min_tokens=3 only an occurrence ending after character 3 counts
    three = llm.generate(["stop test"], SamplingParams(stop=[stop], min_tokens=3, logprobs=1, **kw))[0].outputs[0]
    assert three.text == (base.text[:j] if j >= 0 else base.text)
    assert len(three.logprobs) == (j + 2 if j >= 0 else 8)


def test_async_engine_stream_respects_min_tokens(cabi_double):
    import asyncio
    from chatts_b200.vllm_compat import LLM, AsyncLLMEngine, SamplingParams
    _, _, model, proc = _build(cabi_double)
    llm = LLM(model=model)
    kw = dict(max_tokens=8, ignore_eos=True, allowed_token_ids=list(range(97, 123)))
    base = llm.generate(["stream me"], SamplingParams(**kw))[0].outputs[0].text
    sp = SamplingParams(stop=[base[0:2]], min_tokens=4, **kw)
    final = llm.generate(["stream me"], sp)[0].outputs[0].text

    async def run():
        return [o.outputs[0].text async for o in AsyncLLMEngine(llm).generate("stream me", sp)]
    texts = asyncio.run(run())
    assert texts[1] == base[:2] and texts[-1] == final and final.startswith(base[:4])


# ------------------------------------------------------------------------------------------------------------------ engine
def test_engine_matches_generate_and_leaves_neutral_slots_alone(cabi_double):
    from chatts_b200.engine import ContinuousEngine
    _, _, model, proc = _build(cabi_double)
    prompts = ["first prompt", "a second, longer prompt", "third", "fourth one"]
    kws = [dict(), dict(presence_penalty=0.8, frequency_penalty=0.3, repetition_penalty=1.4, logit_bias={101: 3.0}, min_tokens=3),
           dict(allowed_token_ids=list(range(97, 110)) + [EOS], min_tokens=2), dict(logprobs=2)]
    gen_kw = lambda kw: {("min_new_tokens" if k == "min_tokens" else k): v for k, v in kw.items()}
    want, want_lp = [], []
    for p, kw in zip(prompts, kws):
        enc = _enc(proc, [p])
        S = enc["input_ids"].shape[1]
        want.append(model.generate(**enc, max_new_tokens=9, **gen_kw(kw))[0, S:].tolist())
        want_lp.append(model.last_logprobs)
    eng = ContinuousEngine(model, slots=4, steps_per_round=3)
    rids = [eng.add_request(_enc(proc, [p])["input_ids"][0], max_new_tokens=9, **kw) for p, kw in zip(prompts, kws)]
    done = {r.rid: r for r in eng.run()}
    for rid, w in zip(rids, want):
        toks = done[rid].tokens
        assert toks == w[:len(toks)] and (len(toks) == 9 or toks[-1] == EOS), (toks, w)
    lp = want_lp[3]                                         # the logprobs request, in a round with a processors request and a plain one
    got = done[rids[3]].token_logprobs
    assert len(got) == len(done[rids[3]].tokens) and got == [
        (float(lp.logprobs[0, j]), int(lp.ranks[0, j]), lp.top_ids[0, j].tolist(), lp.top_logprobs[0, j].tolist()) for j in range(len(got))]
    assert not eng._proc.min_tokens.any() and bool((eng._proc.bias_row == -1).all()) and bool((eng._proc.rep == 1).all())
    eng.close()
    assert model.pool.available() == model.pool.num_pages
    with pytest.raises(ValueError):
        ContinuousEngine(model, slots=2).add_request(torch.tensor([1, 2]), presence_penalty=5.0)


def test_engine_slot_reuse_keeps_no_state_of_the_previous_request(cabi_double):
    """One slot serves requests with different processor fields in turn; each equals a stand-alone generate()."""
    from chatts_b200.engine import ContinuousEngine
    _, _, model, proc = _build(cabi_double)
    reqs = [("first prompt", dict(min_tokens=2, presence_penalty=0.5, frequency_penalty=0.2, logit_bias={101: 2.0},
                                  allowed_token_ids=list(range(97, 123)) + [EOS], repetition_penalty=1.2)),
            ("second", dict(ignore_eos=True, logit_bias={EOS: 100.0}, min_tokens=3)),
            ("third prompt", dict(presence_penalty=0.3, min_tokens=2, eos_token_id=[EOS, 997])),
            ("fourth", dict()),
            ("fifth one", dict(ignore_eos=True, min_tokens=4, frequency_penalty=0.6))]
    gen_kw = lambda kw: {("min_new_tokens" if k == "min_tokens" else k): v for k, v in kw.items()}
    want = []
    for p, kw in reqs:
        enc = _enc(proc, [p])
        S = enc["input_ids"].shape[1]
        want.append(model.generate(**enc, max_new_tokens=5, **gen_kw(kw))[0, S:].tolist())
    assert want[1] == [EOS] * 5
    eng = ContinuousEngine(model, slots=1, steps_per_round=2)
    rids = [eng.add_request(_enc(proc, [p])["input_ids"][0], max_new_tokens=5, **kw) for p, kw in reqs]
    done = {r.rid: r.tokens for r in eng.run()}
    for rid, w in zip(rids, want):
        toks = done[rid]
        assert toks == w[:len(toks)] and (len(toks) == 5 or toks[-1] in (EOS, 997)), (toks, w)
    eng.close()
    assert model.pool.available() == model.pool.num_pages


# ------------------------------------------------------------------------------------------------------------------ server
@pytest.mark.parametrize("scheduler", ["batch", "continuous"])
def test_server_honours_the_fields(cabi_double, scheduler):
    from starlette.testclient import TestClient
    from chatts_b200.server import create_app
    from chatts_b200.vllm_compat import LLM, SamplingParams
    _, _, model, proc = _build(cabi_double)
    llm = LLM(model=model)
    fields = {"presence_penalty": 1.0, "frequency_penalty": 0.5, "logit_bias": {str(ord("z")): 4.0}, "min_tokens": 3,
              "allowed_token_ids": list(range(97, 123)) + [EOS]}
    want = llm.generate(["penalise me"], SamplingParams(max_tokens=10, **fields))[0].outputs[0].text
    assert set(want) <= set("abcdefghijklmnopqrstuvwxyz") and len(want) >= 3
    app = create_app(llm, scheduler=scheduler, batch_window_ms=5.0, steps_per_round=2)
    with TestClient(app) as http:
        r = http.post("/v1/completions", json={"prompt": "penalise me", "max_tokens": 10, **fields})
        assert r.status_code == 200 and r.json()["choices"][0]["text"] == want
        r = http.post("/v1/chat/completions", json={"messages": [{"role": "user", "content": "<|im_start|>penalise me"}], "max_tokens": 10,
                                                    **fields})
        assert r.status_code == 200
        pieces = []
        with http.stream("POST", "/v1/completions", json={"prompt": "penalise me", "max_tokens": 10, "stream": True, **fields}) as s:
            for line in s.iter_lines():
                if line.startswith("data: ") and line != "data: [DONE]":
                    pieces.append(json.loads(line[6:])["choices"][0]["text"])
        assert "".join(pieces) == want
        for bad in ({"presence_penalty": 9}, {"logit_bias": {"5000": 1}}, {"allowed_token_ids": [1, 100000]}, {"min_tokens": 50}):
            assert http.post("/v1/completions", json={"prompt": "q", "max_tokens": 10, **bad}).status_code == 400, bad
    app.state.engine.close()
