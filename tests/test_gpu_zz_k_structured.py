"""Structured outputs of generate() on the GPU (tiny model, SimpleTokenizer): greedy and seeded sampled decoding at batch 1 and 4 give
only the choices or full matches of the regex; a pattern with one string reproduces it token for token; with logprobs on, no top-k id
is one the automaton refused and the chosen logprob is finite; a constrained call leaves the next unconstrained call bitwise equal to
one made before it; every page goes back to the pool."""
import re

import numpy as np
import pytest
import torch

from tests.test_gpu_zz_h_prefix_cache import _model, _proc

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
PROMPTS = ["did the series go up?", "answer with a label", "x", "what is the value at the peak?"]


def _setup(dt=BF):
    model = _model("tiny", dt, False)
    return model, _proc(model.config)


def _texts(ids, S, eos):
    out = []
    for row in ids[:, S:].tolist():
        stopped = eos in row
        out.append((bytes(row[:row.index(eos)] if stopped else row).decode("utf-8", "replace"), stopped))
    return out


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("sample", [None, 11, 12])
def test_choice(B, sample):
    model, proc = _setup()
    enc = proc(text=PROMPTS[:B], timeseries=[], padding=True, return_tensors="pt")
    S = enc["input_ids"].shape[1]
    kw = {} if sample is None else dict(do_sample=True, temperature=1.0, top_p=0.95, seed=sample)
    choices = ["increase", "decrease", "steady", "yes", "no"]
    ids = model.generate(**enc, max_new_tokens=16, structured_outputs={"choice": choices}, **kw)
    for text, stopped in _texts(ids, S, model.config.eos_token_id):
        assert stopped and text in choices, text
    assert model.pool.available() == model.pool.num_pages


@pytest.mark.parametrize("pattern", [r"\d{1,3}(\.\d+)?", r"(yes|no)", r"col: \d+(; col: \d+)*"])
@pytest.mark.parametrize("sample", [None, 5])
def test_regex(pattern, sample):
    model, proc = _setup()
    enc = proc(text=PROMPTS, timeseries=[], padding=True, return_tensors="pt")
    S = enc["input_ids"].shape[1]
    kw = {} if sample is None else dict(do_sample=True, temperature=0.9, top_k=50, seed=sample)
    ids = model.generate(**enc, max_new_tokens=40, structured_outputs={"regex": pattern}, **kw)
    dfa = __import__("chatts_b200.structured", fromlist=["x"]).compile_regex(pattern)
    for text, stopped in _texts(ids, S, model.config.eos_token_id):
        if stopped:
            assert re.fullmatch(pattern, text), text
        else:                                                # cut by max_new_tokens: a prefix of a match
            assert dfa.walk(text.encode()) >= 0, text
    assert model.pool.available() == model.pool.num_pages


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_single_string_reproduced_token_for_token(dt):
    model, proc = _setup(dt)
    enc = proc(text=PROMPTS[:2], timeseries=[], padding=True, return_tensors="pt")
    S = enc["input_ids"].shape[1]
    target = "col: 17; col: 204"
    ids = model.generate(**enc, max_new_tokens=30, structured_outputs={"regex": re.escape(target).replace("\\ ", " ")})
    for row in ids[:, S:].tolist():
        assert row[:len(target) + 1] == list(target.encode()) + [model.config.eos_token_id]


def test_logprobs_never_list_a_refused_token():
    from chatts_b200.structured import compile_choice
    model, proc = _setup()
    enc = proc(text=PROMPTS, timeseries=[], padding=True, return_tensors="pt")
    S = enc["input_ids"].shape[1]
    choices = ("yes", "no", "maybe")
    ids = model.generate(**enc, max_new_tokens=8, structured_outputs={"choice": list(choices)}, logprobs=5)
    res, dfa, eos = model.last_logprobs, compile_choice(choices), model.config.eos_token_id
    for b in range(len(PROMPTS)):
        state = 0
        for j, t in enumerate(ids[b, S:].tolist()):
            allowed = {x for x in range(256) if dfa.walk(bytes([x]), state) >= 0} | ({eos} if dfa.accept[state] else set())
            assert t in allowed and np.isfinite(res.logprobs[b, j])
            top = [int(i) for i in res.top_ids[b, j] if i >= 0]
            assert top and set(top) <= allowed and top[0] == t          # greedy: the chosen token is the most likely allowed one
            if t == eos:
                break
            state = dfa.walk(bytes([t]), state)


def test_constrained_call_leaves_the_next_call_unchanged():
    model, proc = _setup()
    enc = proc(text=PROMPTS, timeseries=[], padding=True, return_tensors="pt")
    before = model.generate(**enc, max_new_tokens=12)
    sampled = model.generate(**enc, max_new_tokens=12, do_sample=True, temperature=0.7, seed=3)
    model.generate(**enc, max_new_tokens=12, structured_outputs={"regex": r"[a-z ]+"})
    model.generate(**enc, max_new_tokens=12, structured_outputs={"choice": ["a", "b"]}, do_sample=True, temperature=0.7, seed=3)
    assert torch.equal(model.generate(**enc, max_new_tokens=12), before)
    assert torch.equal(model.generate(**enc, max_new_tokens=12, do_sample=True, temperature=0.7, seed=3), sampled)
    assert model.pool.available() == model.pool.num_pages
