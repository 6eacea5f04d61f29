"""Log probabilities on CPU through the C-ABI double with cts_logprobs restated in torch (tests/logprobs_double.py): SamplingParams
validation and the tensor-parallel refusal, the prompt index mapping (insert / overwrite modes, padding, patch rows), generate()'s
results against log_softmax of the same logits, stop trimming, n > 1, cumulative_logprob, the engine's per-request k, and the server's
JSON under both schedulers with its 400 responses."""
import numpy as np
import pytest
import torch

from chatts_b200 import layout
from chatts_b200.logprobs import check_k, prompt_targets
from tests.logprobs_double import LogprobsDouble
from tests.test_host_model import _build, _series


@pytest.fixture
def cabi_double(cabi_double, monkeypatch):
    from chatts_b200 import _cabi
    dbl = LogprobsDouble()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: dbl)
    return dbl


# ------------------------------------------------------------------------------------------------------------------ validation
def test_k_validation_and_sampling_params():
    from chatts_b200.vllm_compat import SamplingParams
    assert check_k(None, "x") is None and check_k(0, "x") == 0 and check_k(20, "x") == 20
    for bad in (21, -1, 1.5, True, "3"):
        with pytest.raises(ValueError):
            check_k(bad, "x")
    assert SamplingParams(logprobs=5, prompt_logprobs=0).logprobs == 5
    with pytest.raises(ValueError):
        SamplingParams(logprobs=21)
    with pytest.raises(ValueError):
        SamplingParams(prompt_logprobs=-1)


def test_tensor_parallel_refused(cabi_double):
    from chatts_b200.vllm_compat import LLM, SamplingParams
    _, _, model, proc = _build(cabi_double)
    enc = proc(text=["a b c"], timeseries=[], return_tensors="pt")
    model.tp_size = 2                                     # what a rank of a tensor-parallel model reports
    with pytest.raises(ValueError, match="single-GPU"):
        model.generate(**enc, max_new_tokens=2, logprobs=1)
    with pytest.raises(ValueError, match="single-GPU"):
        model.generate(**enc, max_new_tokens=2, prompt_logprobs=0)
    llm = LLM.__new__(LLM)
    llm.model = model
    with pytest.raises(ValueError, match="single-GPU"):
        llm.generate(["a b c"], SamplingParams(max_tokens=2, logprobs=0))
    with pytest.raises(ValueError):
        model.tp_size = 1
        model.generate(**enc, max_new_tokens=2, logprobs=21)


# ------------------------------------------------------------------------------------------------------------ prompt mapping
def test_prompt_targets_insert_mode():
    # row 0: 1 2 <ts> <ts/> 3 with 3 patch rows; row 1 left-padded: 9 8
    ids = np.array([[1, 2, 100, 101, 3], [0, 0, 0, 9, 8]])
    am = np.array([[1, 1, 1, 1, 1], [0, 0, 0, 1, 1]])
    lay = layout.hf_layout(ids, am, [3], 100, "insert")
    pred, tgt, rows, cols = prompt_targets(lay)
    # row 0 merged: 1 2 <ts> r r r <ts/> 3  -> targets 2 (by 0), <ts> (by 1), <ts/> (by the last patch row, 5), 3 (by 6)
    assert pred.tolist() == [0, 1, 5, 6, 8] and tgt.tolist() == [2, 100, 101, 3, 8]
    assert rows.tolist() == [0, 0, 0, 0, 1] and cols.tolist() == [1, 2, 3, 4, 4]
    assert lay.ids[5] == -1                               # the predicting position of <ts/> is a patch row


def test_prompt_targets_overwrite_mode():
    ids = np.array([[1, 100, 101, 3, 4]])
    lay = layout.hf_layout(ids, None, [2], 100, "overwrite")
    pred, tgt, rows, cols = prompt_targets(lay)
    # merged: 1 r r 3 4 -> 3 predicted by the last patch row (2), 4 by 3; <ts> / <ts/> have no merged position
    assert pred.tolist() == [2, 3] and tgt.tolist() == [3, 4] and cols.tolist() == [3, 4]


@pytest.mark.parametrize("mode", ["insert", "overwrite"])
def test_generate_prompt_logprobs_match_log_softmax(cabi_double, monkeypatch, mode):
    """Prompt entries = log_softmax of forward(logits_to_keep=0) at the mapped positions; left padding excluded, entry 0 None, and in
    overwrite mode None for <ts> / <ts/>."""
    monkeypatch.setenv("CTS_TS_MERGE_MODE", mode)
    cfg, _, model, proc = _build(cabi_double)
    a, b = _series()
    enc = proc(text=["x <ts><ts/> y z", "hello <ts><ts/> a b c d e"], timeseries=[a, b], padding=True, return_tensors="pt")
    full = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"], logits_to_keep=0).logits
    model.generate(**enc, max_new_tokens=2, prompt_logprobs=3, ignore_eos=True)
    res = model.last_logprobs
    assert res.logprobs is None and len(res.prompt) == 2
    ids, am = enc["input_ids"].numpy(), enc["attention_mask"].numpy()
    _, _, _, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
    cu = lay.cu_seqlens
    for r in range(2):
        kept = np.nonzero(am[r])[0]
        assert len(res.prompt[r]) == kept.shape[0] and res.prompt[r][0] is None
        lp = torch.log_softmax(full[r].float(), -1)
        merged_of_col = {int(c): j - cu[r] for j, c in enumerate(lay.src_col) if cu[r] <= j < cu[r + 1] and c >= 0}
        for e, c in enumerate(kept[1:], start=1):
            ent = res.prompt[r][e]
            tok = int(ids[r, c])
            if mode == "overwrite" and tok in (cfg.ts_token_start_index, cfg.ts_token_start_index + 1):
                assert ent is None
                continue
            j = merged_of_col[int(c)]
            assert ent.token_id == tok and abs(ent.logprob - float(lp[j - 1, tok])) <= 1e-5
            assert ent.rank == 1 + int((full[r][j - 1].float() > full[r][j - 1, tok].float()).sum())
            assert ent.top_ids == torch.topk(lp[j - 1], 3).indices.tolist() or np.allclose(ent.top_logprobs, torch.topk(lp[j - 1], 3).values)


def test_prompt_logprobs_skip_the_prefix_cache(cabi_double):
    _, _, model, proc = _build(cabi_double, enable_prefix_caching=True)
    a, _ = _series()
    enc = proc(text=["some words <ts><ts/> and " + "a long enough question here " * 3], timeseries=[a], return_tensors="pt")
    model.generate(**enc, max_new_tokens=2, ignore_eos=True)
    model.generate(**enc, max_new_tokens=2, ignore_eos=True, prompt_logprobs=0)
    assert int(model.last_cached_positions[0]) == 0 and model.last_logprobs.prompt[0][1] is not None
    model.generate(**enc, max_new_tokens=2, ignore_eos=True)
    assert int(model.last_cached_positions[0]) > 0


# ------------------------------------------------------------------------------------------------------------------ decode
def _reference_steps(model, enc, n):
    """Logits of the greedy continuation, teacher-forced through forward(): [n, V] per row 0."""
    out = model.generate(**enc, max_new_tokens=n, ignore_eos=True)
    S = enc["input_ids"].shape[1]
    rows = []
    for j in range(n):
        lg = model.forward(out[:, : S + j], torch.ones_like(out[:, : S + j]), enc.get("timeseries")).logits[:, 0]
        rows.append(lg[0])
    return out[0, S:], torch.stack(rows)


def test_generate_logprobs_match_log_softmax(cabi_double):
    _, _, model, proc = _build(cabi_double)
    enc = proc(text=["a b c d"], timeseries=[], return_tensors="pt")
    toks, logits = _reference_steps(model, enc, 4)
    out = model.generate(**enc, max_new_tokens=4, ignore_eos=True, logprobs=5)
    assert torch.equal(out[0, -4:], toks)                 # tokens do not change with logprobs on
    res = model.last_logprobs
    assert res.logprobs.shape == (1, 4) and res.top_ids.shape == (1, 4, 5) and res.prompt is None
    lp = torch.log_softmax(logits.float(), -1)
    for j in range(4):
        assert abs(float(res.logprobs[0, j]) - float(lp[j, toks[j]])) <= 1e-5 and int(res.ranks[0, j]) == 1
        assert res.top_ids[0, j, 0] == int(toks[j])
        assert np.allclose(res.top_logprobs[0, j], torch.topk(lp[j], 5).values.numpy(), atol=1e-5)


def test_llm_outputs_stop_trimming_and_n(cabi_double):
    from chatts_b200.vllm_compat import LLM, Logprob, SamplingParams
    _, _, model, _ = _build(cabi_double)
    llm = LLM(model=model)
    a, _ = _series()
    req = {"prompt": "x <ts><ts/> y", "multi_modal_data": {"timeseries": [a]}}
    out = llm.generate([req], SamplingParams(max_tokens=6, ignore_eos=True, logprobs=3, prompt_logprobs=1))[0]
    c = out.outputs[0]
    assert len(c.logprobs) == len(c.token_ids) == 6
    for t, d in zip(c.token_ids, c.logprobs):
        assert t in d and len(d) in (3, 4) and all(isinstance(v, Logprob) for v in d.values())
    assert abs(c.cumulative_logprob - sum(d[t].logprob for t, d in zip(c.token_ids, c.logprobs))) < 1e-9
    assert out.prompt_logprobs[0] is None and all(p is None or len(p) in (1, 2) for p in out.prompt_logprobs[1:])
    # stop id: the stop token and what follows leave with the tokens
    stop = c.token_ids[2]
    cut = llm.generate([req], SamplingParams(max_tokens=6, logprobs=0, stop_token_ids=[stop]))[0].outputs[0]
    assert len(cut.logprobs) == len(cut.token_ids) == c.token_ids.index(stop) and all(len(d) == 1 for d in cut.logprobs)
    # stop string: the logprobs end with the token that completed it
    s = llm.tokenizer.decode(c.token_ids[3:4])
    if s:
        cs = llm.generate([req], SamplingParams(max_tokens=6, ignore_eos=True, logprobs=0, stop=[s]))[0].outputs[0]
        assert s not in cs.text and len(cs.logprobs) <= 4
    # n > 1: each copy carries its own logprobs
    two = llm.generate([req], SamplingParams(max_tokens=3, ignore_eos=True, logprobs=2, n=2))[0]
    assert len(two.outputs) == 2 and all(len(o.logprobs) == 3 for o in two.outputs) and two.outputs[0].logprobs is not two.outputs[1].logprobs


def test_engine_per_request_k(cabi_double):
    from chatts_b200.engine import ContinuousEngine
    _, _, model, proc = _build(cabi_double)
    texts = ["a b c", "d e f g", "h i"]
    eng = ContinuousEngine(model, slots=4, steps_per_round=3)
    ks = [None, 0, 4]
    for t, k in zip(texts, ks):
        eng.add_request(proc(text=[t], timeseries=[], return_tensors="pt")["input_ids"][0], max_new_tokens=5, ignore_eos=True, logprobs=k)
    done = eng.run()
    eng.close()
    for r, t, k in zip(done, texts, ks):
        enc = proc(text=[t], timeseries=[], return_tensors="pt")
        out = model.generate(**enc, max_new_tokens=5, ignore_eos=True, logprobs=k)
        assert r.tokens == out[0, -5:].tolist()
        if k is None:
            assert r.token_logprobs == []
            continue
        res = model.last_logprobs
        assert len(r.token_logprobs) == 5
        for j, (lp, rank, ids, vals) in enumerate(r.token_logprobs):
            assert abs(lp - float(res.logprobs[0, j])) <= 1e-5 and rank == int(res.ranks[0, j])
            assert ids == res.top_ids[0, j].tolist() and len(vals) == k
    with pytest.raises(ValueError):
        ContinuousEngine(model, slots=2).add_request([1, 2], logprobs=21)


# ------------------------------------------------------------------------------------------------------------------ server
@pytest.fixture(params=["batch", "continuous"])
def served(cabi_double, request):
    from starlette.testclient import TestClient
    from chatts_b200.server import create_app
    from chatts_b200.vllm_compat import LLM
    _, _, model, _ = _build(cabi_double)
    app = create_app(LLM(model=model), batch_window_ms=20.0, scheduler=request.param)
    with TestClient(app) as client:
        yield client
    app.state.engine.close()


def test_server_logprobs_json(served):
    http = served
    a, _ = _series()
    chat = {"messages": [{"role": "user", "content": [{"type": "text", "text": "look <ts><ts/> now"}, {"timeseries": a.tolist()}]}],
            "max_tokens": 4, "ignore_eos": True, "logprobs": True, "top_logprobs": 5}
    r = http.post("/v1/chat/completions", json=chat)
    assert r.status_code == 200, r.text
    content = r.json()["choices"][0]["logprobs"]["content"]
    assert len(content) == 4
    for e in content:
        assert set(e) == {"token", "logprob", "bytes", "top_logprobs"} and len(e["top_logprobs"]) == 5 and e["logprob"] <= 0
        assert e["top_logprobs"][0]["logprob"] >= e["logprob"] and bytes(e["bytes"]).decode() == e["token"]
    assert "logprobs" not in http.post("/v1/chat/completions", json=dict(chat, logprobs=False, top_logprobs=None)).json()["choices"][0]
    comp = {"prompt": "x <ts><ts/> y", "multi_modal_data": {"timeseries": [a.tolist()]}, "max_tokens": 3, "ignore_eos": True, "logprobs": 2}
    r = http.post("/v1/completions", json=comp)
    assert r.status_code == 200, r.text
    lp = r.json()["choices"][0]["logprobs"]
    assert len(lp["tokens"]) == len(lp["token_logprobs"]) == len(lp["top_logprobs"]) == len(lp["text_offset"]) == 3
    assert all(len(t) <= 2 for t in lp["top_logprobs"]) and lp["text_offset"][0] == 0
    # refusals: streaming with logprobs, out-of-range values
    assert http.post("/v1/chat/completions", json=dict(chat, stream=True)).status_code == 400
    assert http.post("/v1/completions", json=dict(comp, stream=True)).status_code == 400
    assert http.post("/v1/chat/completions", json=dict(chat, top_logprobs=21)).status_code == 400
    assert http.post("/v1/chat/completions", json=dict(chat, logprobs=False, top_logprobs=2)).status_code == 400
    assert http.post("/v1/completions", json=dict(comp, logprobs=-1)).status_code == 400
