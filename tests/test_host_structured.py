"""Structured outputs on CPU: the regex compiler against Python's ``re`` (accept / reject identical on a corpus of patterns x random and
adversarial strings), the constructs it refuses, trimming, the state cap, the token bytes of SimpleTokenizer and of a byte-level BPE
tokenizer, SamplingParams / server parsing and its 400s, and generate() / LLM / the server end to end through a torch restatement of
the three kernels (tests/structured_double.py)."""
import itertools
import random
import re

import numpy as np
import pytest
import torch

from chatts_b200 import structured as so
from tests.structured_double import StructuredDouble, mask_build_reference, unpack_bits
from tests.test_host_model import _build


@pytest.fixture
def cabi_double(cabi_double, monkeypatch):
    from chatts_b200 import _cabi
    dbl = StructuredDouble()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: dbl)
    return dbl


# ------------------------------------------------------------------------------------------------------------------ compiler
PATTERNS = [r"\d{1,3}(\.\d+)?", r"(yes|no)", r"col: \d+(; col: \d+)*", r"a*b+c?", r"[a-c]{2,4}", r"(ab|a)*b", r"[^abc]+", r".{2}x",
            r"\w+@\w+\.com", r"(a|b)*abb", r"x{3}", r"x{2,}", r"x{,2}", r"a{}", r"a{,}", r"\s*\S+", r"[\d\-]+", r"(?:foo|bar)baz",
            r"^abc$", r"a+?b", r"[]a]+", r"[a-]+", r"\.\*\+", r"(a?){3}", r"((a|b)c)*", r"[\w.]+", r"\D\W", r"[^\n]*", r"a|", r"()",
            r"(|a)b", r"[0-9a-fA-F]{1,4}", r"[\b]x", r"a{2}b{0,3}", r"(a|ab)(c|bcd)(d*)", r"[\s\d]+\?", r"\(\d+\)", r"a.c|[.]"]
ALPHABET = b"abcdxy0159.;:-? @\n\t_()]\x80\xc3\xff"


def _strings(pattern, n=2000, seed=0):
    rng = random.Random(hash(pattern) ^ seed)
    out = [bytes(rng.choice(ALPHABET) for _ in range(rng.randint(0, 10))) for _ in range(n)]
    out += [bytes(s) for k in range(5) for s in itertools.product(b"abc1.", repeat=k)]
    # adversarial: strings the pattern matches (from its own alphabet), then each cut short, extended and with one byte changed
    lits = [c.encode() for c in re.findall(r"[a-z0-9.;: ()?-]", pattern)] or [b"a"]
    for _ in range(300):
        s = b"".join(rng.choice(lits) for _ in range(rng.randint(0, 8)))
        out += [s, s[:-1], s + b"a", s[:1] + b"\n" + s[1:]]
    return out


@pytest.mark.parametrize("pattern", PATTERNS)
def test_regex_accepts_exactly_what_python_re_fullmatch_accepts(pattern):
    dfa = so.compile_regex(pattern)
    rx = re.compile(pattern.encode())
    bad = [s for s in _strings(pattern) if dfa.fullmatch(s) != bool(rx.fullmatch(s))]
    assert not bad, bad[:5]


def test_utf8_literals_match_as_their_bytes():
    dfa = so.compile_regex("(größer|kleiner) als é+")
    for text in ("größer als é", "kleiner als ééé", "größer als", "groesser als é", "größer als e"):
        assert dfa.fullmatch(text.encode()) == bool(re.fullmatch("(größer|kleiner) als é+", text)), text


@pytest.mark.parametrize("pattern,word", [(r"(a)\1", "backreference"), (r"(?=a)b", "lookahead"), (r"(?<!a)b", "lookbehind"),
                                          (r"a^b", "anchor"), (r"a$b", "anchor"), (r"\bfoo", "anchor"), (r"[é]", "non-ASCII"),
                                          (r"(?P<x>a)", "named group"), (r"(?i)a", "inline flags"), (r"a*+", "possessive"),
                                          (r"*a", "nothing to repeat"), (r"(a", "missing"), (r"a)", "unbalanced"), (r"[a", "unterminated"),
                                          (r"\x41", "escape"), (r"a{3,2}", "min repeat"), (r"[^\s\S]", "matches no string"),
                                          (r"a{1001}", "exceeds"), (r"\p{L}", "escape")])
def test_unsupported_constructs_raise_naming_them(pattern, word):
    with pytest.raises(ValueError, match=word):
        so.compile_regex(pattern)


@pytest.mark.parametrize("pattern", PATTERNS + [r"a[^\s\S]|b", r"(x[^\s\S])*y|z", r"c(a[^\s\S]|b)*d"])
def test_trimming_leaves_no_dead_state(pattern):
    dfa = so.compile_regex(pattern)
    live = set(np.nonzero(dfa.accept)[0].tolist())
    changed = True
    while changed:
        changed = False
        for s in range(dfa.num_states):
            if s not in live and any(int(t) in live for t in dfa.trans[s] if t >= 0):
                live.add(s)
                changed = True
    assert live == set(range(dfa.num_states))
    assert (dfa.trans < dfa.num_states).all() and (dfa.trans >= -1).all()


def test_state_cap():
    assert so.MAX_STATES == 4096
    so.compile_regex(r"(a|b)*a(a|b){10}")                          # 2^11 states: under the cap
    with pytest.raises(ValueError, match="4096"):
        so.compile_regex(r"(a|b)*a(a|b){12}")                      # 2^13
    with pytest.raises(ValueError, match="4096"):
        so.compile_choice(tuple(f"{i:05d}-choice" for i in range(1000)))


def test_choice_trie():
    dfa = so.compile_choice(("yes", "no", "nö", ""))
    for s in ("yes", "no", "nö", ""):
        assert dfa.fullmatch(s.encode())
    for s in ("ye", "yess", "n", "non"):
        assert not dfa.fullmatch(s.encode())
    assert dfa.num_states == 1 + 3 + 2 + 2                        # root, y-e-s, n-o, ö (2 bytes)


# ------------------------------------------------------------------------------------------------------------------ token bytes
def test_token_bytes_simple_tokenizer():
    from chatts_b200 import SimpleTokenizer
    off, data = so.token_bytes(SimpleTokenizer(990, 999, 998), 1000)
    assert off.shape == (1001,) and off.dtype == np.int64 and data.dtype == np.uint8
    for t in (0, 65, 255):
        assert bytes(data[off[t]:off[t + 1]]) == bytes([t])
    assert all(off[t] == off[t + 1] for t in (256, 990, 998, 999))
    off2, _ = so.token_bytes(None, 300)
    assert off2[256] == off2[300] == 256


def _bpe():
    tk = pytest.importorskip("tokenizers")
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    alphabet = pre_tokenizers.ByteLevel.alphabet()
    vocab = {c: i for i, c in enumerate(sorted(alphabet))}
    merges = [("Ġ", "y"), ("Ġy", "e"), ("Ġye", "s"), ("n", "o"), ("Ã", "©")]
    for a, b in merges:
        vocab[a + b] = len(vocab)
    tok = Tokenizer(models.BPE(vocab=vocab, merges=merges))
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tok.decoder = decoders.ByteLevel()
    tok.add_special_tokens(["<|end|>"])
    assert tk
    return tok


def test_token_bytes_byte_level_bpe():
    tok = _bpe()
    V = tok.get_vocab_size() + 7                                    # embedding rows past the tokenizer
    off, data = so.token_bytes(tok, V)
    piece = lambda t: bytes(data[off[t]:off[t + 1]])
    assert piece(tok.token_to_id("Ġyes")) == b" yes" and piece(tok.token_to_id("no")) == b"no"
    assert piece(tok.token_to_id("Ã©")) == "é".encode()
    assert piece(tok.token_to_id("Ċ")) == b"\n" and piece(tok.token_to_id("a")) == b"a"
    assert piece(tok.token_to_id("<|end|>")) == b""                # special token: no bytes
    assert all(piece(t) == b"" for t in range(tok.get_vocab_size(), V))
    # every encoded text is the concatenation of its tokens' bytes
    for text in ("no yes", "é no\n", "a b"):
        assert b"".join(piece(t) for t in tok.encode(text).ids) == text.encode()
    tf = pytest.importorskip("transformers")
    hf = tf.PreTrainedTokenizerFast(tokenizer_object=tok)
    off2, data2 = so.token_bytes(hf, V)
    assert np.array_equal(off, off2) and np.array_equal(data, data2)


def test_mask_reference_walks_token_bytes():
    dfa = so.compile_choice(("yes", "no"))
    off = np.array([0, 1, 3, 4, 6, 6], dtype=np.int64)              # "y", "es", "n", "no", stop id (no bytes)
    data = np.frombuffer(b"yesnno", dtype=np.uint8)
    bits = unpack_bits(mask_build_reference(dfa.trans, dfa.accept, off, data, [4]), 5)
    assert bits[0].tolist() == [True, False, True, True, False]    # start: y, n, no; stop only where accepting
    s_y = dfa.walk(b"y")
    assert bits[s_y].tolist() == [False, True, False, False, False]
    assert bits[dfa.walk(b"no")].tolist() == [False, False, False, False, True]


# ------------------------------------------------------------------------------------------------------------------ params
def test_structured_outputs_params_and_sampling_params():
    from chatts_b200.vllm_compat import SamplingParams, StructuredOutputsParams
    assert SamplingParams().structured_outputs is None
    sp = SamplingParams(structured_outputs={"choice": ["a", "b"]})
    assert sp.structured_outputs == StructuredOutputsParams(choice=["a", "b"])
    assert SamplingParams(structured_outputs=StructuredOutputsParams()).structured_outputs is None
    for bad in ({"json": {"type": "object"}}, {"grammar": "root ::= x"}, {"json_object": True}):
        with pytest.raises(ValueError, match="not supported"):
            SamplingParams(structured_outputs=bad)
    for bad in ({"choice": ["a"], "regex": "a"}, {"choice": []}, {"choice": "ab"}, {"choice": [1]}, {"regex": 3}, {"foo": 1}):
        with pytest.raises(ValueError):
            SamplingParams(structured_outputs=bad)
    with pytest.raises(ValueError, match="ignore_eos"):
        SamplingParams(structured_outputs={"regex": "a"}, ignore_eos=True)


def test_server_body_parsing():
    from chatts_b200.server import _sampling_from_body
    assert "structured_outputs" not in _sampling_from_body({})
    assert _sampling_from_body({"structured_outputs": {"choice": ["x", "y"]}})["structured_outputs"] == {"choice": ["x", "y"]}
    assert _sampling_from_body({"guided_choice": ["x"]}, chat=True)["structured_outputs"] == {"choice": ["x"]}
    assert _sampling_from_body({"guided_regex": r"\d+"})["structured_outputs"] == {"regex": r"\d+"}
    assert "structured_outputs" not in _sampling_from_body({"response_format": {"type": "json_object"}})
    for bad in ({"structured_outputs": {"regex": "(a"}}, {"structured_outputs": {"json": {}}}, {"structured_outputs": "x"},
                {"structured_outputs": {"choice": ["a"]}, "guided_regex": "a"}, {"guided_regex": "a", "ignore_eos": True},
                {"structured_outputs": {"choice": ["a"], "regex": "a"}}):
        with pytest.raises(ValueError):
            _sampling_from_body(bad)


# ------------------------------------------------------------------------------------------------------------------ end to end
def _enc(proc, texts):
    return proc(text=texts, timeseries=[], padding=True, return_tensors="pt")


def _outputs(ids, S, eos):
    out = []
    for row in ids[:, S:].tolist():
        cut = row.index(eos) if eos in row else len(row)
        out.append((bytes(row[:cut]).decode("utf-8", "replace"), eos in row))
    return out


@pytest.mark.parametrize("sample", [False, True])
def test_generate_choice_and_regex(cabi_double, sample):
    cfg, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["which one?", "answer please", "x", "the number"])
    S = enc["input_ids"].shape[1]
    kw = dict(do_sample=True, temperature=1.0, seed=7) if sample else {}
    choices = ["increase", "decrease", "steady"]
    ids = model.generate(**enc, max_new_tokens=12, structured_outputs={"choice": choices}, **kw)
    for text, stopped in _outputs(ids, S, cfg.eos_token_id):
        assert stopped and text in choices
    for pat in (r"\d{1,3}(\.\d+)?", r"(yes|no)", r"col: \d+(; col: \d+)*"):
        ids = model.generate(**enc, max_new_tokens=24, structured_outputs=so.StructuredOutputsParams(regex=pat), **kw)
        for text, stopped in _outputs(ids, S, cfg.eos_token_id):
            assert re.fullmatch(pat, text) if stopped else re.fullmatch(pat, text + "0") or re.match(pat, text), (pat, text)
    assert model.pool.available() == model.pool.num_pages


def test_generate_single_string_and_cut_by_length(cabi_double):
    cfg, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["go"])
    S = enc["input_ids"].shape[1]
    ids = model.generate(**enc, max_new_tokens=10, structured_outputs={"regex": "col: 42"})
    assert ids[0, S:].tolist() == list(b"col: 42") + [cfg.eos_token_id]
    ids = model.generate(**enc, max_new_tokens=4, structured_outputs={"regex": "col: 42"})
    assert ids[0, S:].tolist() == list(b"col:")


def test_generate_logprobs_describe_the_masked_distribution(cabi_double):
    cfg, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["a", "bb"])
    S = enc["input_ids"].shape[1]
    ids = model.generate(**enc, max_new_tokens=6, structured_outputs={"choice": ["yes", "no"]}, logprobs=5)
    res = model.last_logprobs
    dfa = so.compile_choice(("yes", "no"))
    for b in range(2):
        state = 0
        for j, t in enumerate(ids[b, S:].tolist()):
            allowed = {t2 for t2 in range(256) if dfa.walk(bytes([t2]), state) >= 0}
            if dfa.accept[state]:
                allowed.add(cfg.eos_token_id)
            assert np.isfinite(res.logprobs[b, j])
            assert set(int(i) for i in res.top_ids[b, j] if i >= 0) <= allowed
            assert np.isfinite(res.top_logprobs[b, j][res.top_ids[b, j] >= 0]).all()
            if t == cfg.eos_token_id:
                break
            state = dfa.walk(bytes([t]), state)


def test_generate_refusals(cabi_double):
    _, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["a"])
    n = model.pool.available()
    with pytest.raises(ValueError, match="ignore_eos"):
        model.generate(**enc, max_new_tokens=2, structured_outputs={"choice": ["a"]}, ignore_eos=True)
    with pytest.raises(ValueError):
        model.generate(**enc, max_new_tokens=2, structured_outputs={"regex": "(?=a)"})
    model.tp_size = 2
    with pytest.raises(ValueError, match="single-GPU"):
        model.generate(**enc, max_new_tokens=2, structured_outputs={"choice": ["a"]})
    model.tp_size = 1
    assert model.pool.available() == n


def test_unconstrained_call_unchanged_by_a_constrained_one(cabi_double):
    _, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["same prompt", "other"])
    before = model.generate(**enc, max_new_tokens=8)
    model.generate(**enc, max_new_tokens=8, structured_outputs={"regex": r"[a-z]+"})
    assert torch.equal(model.generate(**enc, max_new_tokens=8), before)


def test_llm_and_server_end_to_end(cabi_double):
    from starlette.testclient import TestClient
    from chatts_b200.server import create_app
    from chatts_b200.vllm_compat import LLM, SamplingParams
    _, _, model, _ = _build(cabi_double)
    llm = LLM(model=model)
    outs = llm.generate(["pick", "choose"], SamplingParams(max_tokens=12, structured_outputs={"choice": ["up", "down"]}, n=2,
                                                           temperature=0.8, seed=3))
    for o in outs:
        for c in o.outputs:
            assert c.text in ("up", "down") and c.finish_reason == "stop"
    o = llm.generate(["n"], SamplingParams(max_tokens=3, structured_outputs={"regex": r"\d{5}"}))[0].outputs[0]
    assert re.fullmatch(r"\d{3}", o.text) and o.finish_reason == "length"
    app = create_app(llm, batch_window_ms=5.0)
    with TestClient(app) as http:
        r = http.post("/v1/completions", json={"prompt": "q", "max_tokens": 10, "structured_outputs": {"choice": ["yes", "no"]}})
        assert r.status_code == 200 and r.json()["choices"][0]["text"] in ("yes", "no")
        r = http.post("/v1/chat/completions", json={"messages": [{"role": "user", "content": "q"}], "max_tokens": 10,
                                                    "guided_regex": r"[0-9]{2}"})
        assert r.status_code == 200 and re.fullmatch(r"[0-9]{2}", r.json()["choices"][0]["message"]["content"])
        assert http.post("/v1/completions", json={"prompt": "q", "guided_regex": "a(?=b)"}).status_code == 400
        assert http.post("/v1/completions", json={"prompt": "q", "structured_outputs": {"json": {}}}).status_code == 400
    app.state.engine.close()
    app = create_app(llm, scheduler="continuous")
    with TestClient(app) as http:
        r = http.post("/v1/completions", json={"prompt": "q", "max_tokens": 4, "guided_choice": ["a"]})
        assert r.status_code == 400 and "continuous" in r.text
    app.state.engine.close()


def test_automaton_cache(cabi_double):
    _, _, model, proc = _build(cabi_double)
    enc = _enc(proc, ["a"])
    model.generate(**enc, max_new_tokens=2, structured_outputs={"choice": ["x", "y"]})
    a = next(iter(model._struct_cache.automata.values()))
    model.generate(**enc, max_new_tokens=2, structured_outputs={"choice": ["x", "y"]})
    assert len(model._struct_cache.automata) == 1 and next(iter(model._struct_cache.automata.values())) is a
    model.generate(**enc, max_new_tokens=2, structured_outputs={"choice": ["x", "y"]}, eos_token_id=[998, 997])
    assert len(model._struct_cache.automata) == 2
