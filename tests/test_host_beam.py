"""Beam search on CPU: the restatement of csrc/beam.cu (tests/beam_double.py) against transformers' generate(num_beams=...) on a tiny
fp32 Qwen2ForCausalLM over a grid of num_beams, length_penalty, early_stopping, EOS ids and num_return_sequences; ChatTSForCausalLM's
generate(num_beams=...) through the C-ABI double against transformers on the same weights; every refusal, leaving the pool as it was;
num_beams=1 bitwise equal to the plain call; and the page plan after every step (one writer per page, full pages immutable)."""
import itertools

import numpy as np
import pytest
import torch

from tests.beam_double import BeamDouble, beam_search, fork_reference, select_reference  # noqa: F401
from tests.test_oracle_decoder import _hf_model

PAD = 7


@pytest.fixture
def cabi_double(cabi_double, monkeypatch):
    from chatts_b200 import _cabi
    dbl = BeamDouble()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: dbl)
    return dbl


_HF = {}


def _hf():
    if "m" not in _HF:
        _HF["m"] = _hf_model(torch.float32)
    return _HF["m"]


def _ours(m, prompt, B, nb, max_new, eos, lp, es, nrs):
    S = prompt.shape[1]

    def next_lp(seqs):
        rows = torch.cat([prompt.repeat_interleave(nb, 0), torch.tensor(seqs, dtype=torch.long).view(B * nb, -1)], 1)
        with torch.no_grad():
            lg = m(rows, attention_mask=torch.ones_like(rows)).logits[:, -1].float()
        return torch.log_softmax(lg, -1).numpy()
    return beam_search(next_lp, S, B, nb, m.config.vocab_size, max_new, eos, lp, es, nrs)


def _hf_run(m, prompt, nb, max_new, eos, lp, es, nrs):
    with torch.no_grad():
        o = m.generate(prompt, attention_mask=torch.ones_like(prompt), num_beams=nb, length_penalty=lp, early_stopping=es,
                       num_return_sequences=nrs, max_new_tokens=max_new, eos_token_id=list(eos) if eos else None, pad_token_id=PAD,
                       do_sample=False, return_dict_in_generate=True, output_scores=True)
    return o.sequences, o.sequences_scores


def _assert_same(hf_seq, hf_scores, hyps, scores, S):
    flat = [h for per in hyps for h in per]
    n = max(len(h) for h in flat)
    assert hf_seq.shape[1] == S + n, (hf_seq.shape, S, n)
    for r, h in enumerate(flat):
        assert hf_seq[r, S:S + len(h)].tolist() == h, (r, hf_seq[r, S:].tolist(), h)
        assert (hf_seq[r, S + len(h):] == PAD).all()
    # 1e-5, or about two fp32 ulps where length_penalty < 0 multiplies the summed log-probs up to a few hundred
    np.testing.assert_allclose(scores, hf_scores.float().numpy(), rtol=2.5e-7, atol=1e-5)


def _eos_ids(m, prompt, nb, max_new, kind):
    """EOS ids that the search meets: the best step-0 token ("step0"), or tokens of the best sequence of a run without EOS."""
    if kind == "none":
        return ()
    seq, _ = _hf_run(m, prompt, nb, max_new, (), 1.0, False, 1)
    gen = seq[0, prompt.shape[1]:].tolist()
    if kind == "step0":
        return (gen[0],)
    return (gen[2],) if kind == "one" else (gen[2], gen[4])


GRID = [(nb, lp, es, kind) for nb, lp, es, kind in itertools.product([2, 3, 4, 5, 6], [-1.0, 0.0, 1.0, 2.0], [True, False, "never"],
                                                                     ["one", "two"])]


@pytest.mark.parametrize("nb,lp,es,kind", GRID + [(4, 1.0, False, "none"), (3, 2.0, "never", "none"), (3, 1.0, True, "step0"),
                                                  (5, -1.0, False, "step0")])
def test_restatement_matches_transformers(nb, lp, es, kind):
    m = _hf()
    g = torch.Generator().manual_seed(nb * 31 + int(lp * 7) + len(str(es)))
    B, S, max_new = 2, 6, 9
    prompt = torch.randint(10, m.config.vocab_size, (B, S), generator=g)
    eos = _eos_ids(m, prompt[:1], nb, max_new, kind)
    nrs = 1 + (int(lp) + len(kind) + len(str(es))) % nb
    hf_seq, hf_scores = _hf_run(m, prompt, nb, max_new, eos, lp, es, nrs)
    hyps, scores, _, _ = _ours(m, prompt, B, nb, max_new, eos, lp, es, nrs)
    _assert_same(hf_seq, hf_scores, hyps, scores, S)


# ------------------------------------------------------------------------------------------------------------------ the model
def _chatts(cabi_double, max_batch=8, cached=False, page=16):
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig.tiny()
    sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=torch.float32, std=0.05)
    model = ChatTSForCausalLM(cfg, sd, device="cpu", dtype=torch.float32, max_batch=max_batch, max_seq_len=512, page_size=page,
                              use_cuda_graph=False, enable_prefix_caching=cached)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    return cfg, sd, model, proc


def _hf_from(cfg, sd):
    from transformers import Qwen2Config, Qwen2ForCausalLM
    c = Qwen2Config(hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size, num_hidden_layers=cfg.num_hidden_layers,
                    num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads, vocab_size=cfg.vocab_size,
                    rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta, max_position_embeddings=cfg.max_position_embeddings,
                    tie_word_embeddings=False, attn_implementation="eager")
    m = Qwen2ForCausalLM(c).eval()
    m.load_state_dict({k: v for k, v in sd.items() if not k.startswith("ts_encoder.")}, strict=True)
    return m


@pytest.mark.parametrize("nb,lp,es,nrs,page", [(3, 1.0, False, 2, 16), (4, 2.0, True, 4, 4), (2, -1.0, "never", 1, 5), (5, 0.0, False, 3, 16)])
def test_chatts_generate_matches_transformers(cabi_double, nb, lp, es, nrs, page):
    cfg, sd, model, proc = _chatts(cabi_double, max_batch=16, page=page)
    enc = proc(text=["the series rose", "then it fell!!!"], timeseries=[], padding=True, return_tensors="pt")
    S = enc["input_ids"].shape[1]
    hf = _hf_from(cfg, sd)
    seq, _ = _hf_run(hf, enc["input_ids"][:1], nb, 10, (), 1.0, False, 1)
    eos = (seq[0, S + 3].item(),)
    hf_seq, hf_scores = _hf_run(hf, enc["input_ids"], nb, 10, eos, lp, es, nrs)
    free = model.pool.available()
    out = model.generate(**enc, max_new_tokens=10, num_beams=nb, length_penalty=lp, early_stopping=es, num_return_sequences=nrs,
                         eos_token_id=list(eos), pad_token_id=PAD)
    assert out.shape == hf_seq.shape and out.tolist() == hf_seq.tolist(), (out[:, S:], hf_seq[:, S:])
    np.testing.assert_allclose(model.last_beam_scores.numpy(), hf_scores.float().numpy(), rtol=2.5e-7, atol=1e-5)
    assert model.last_beam_scores.dtype == torch.float32 and model.pool.available() == free


REFUSALS = [
    (dict(do_sample=True), "do_sample=False"),
    (dict(num_beam_groups=2), "group"),
    (dict(diversity_penalty=0.5), "diverse"),
    (dict(repetition_penalty=1.1), "repetition_penalty"),
    (dict(logprobs=2), "logprobs"),
    (dict(prompt_logprobs=1), "prompt_logprobs"),
    (dict(structured_outputs={"choice": ["a"]}), "structured_outputs"),
    (dict(streamer=object()), "streamer"),
    (dict(num_return_sequences=5), "num_return_sequences"),
    (dict(num_beams=7, eos_token_id=[1, 2]), "at most 6"),
    (dict(num_beams=3, early_stopping="sometimes"), "early_stopping"),
]


@pytest.mark.parametrize("kw,match", REFUSALS)
def test_refusals_take_nothing(cabi_double, kw, match):
    _, _, model, proc = _chatts(cabi_double)
    enc = proc(text=["abc", "defg"], timeseries=[], padding=True, return_tensors="pt")
    free = model.pool.available()
    kw = dict(dict(num_beams=4), **kw)
    with pytest.raises(ValueError, match=match):
        model.generate(**enc, max_new_tokens=4, **kw)
    assert model.pool.available() == free


def test_refusals_from_defaults_tp_and_rows(cabi_double):
    _, _, model, proc = _chatts(cabi_double, max_batch=8)
    enc = proc(text=["abc", "defg", "xy"], timeseries=[], padding=True, return_tensors="pt")
    free = model.pool.available()
    with pytest.raises(ValueError, match="max_batch"):
        model.generate(**enc, max_new_tokens=4, num_beams=3)                  # 9 rows > 8
    model.generation_defaults = dict(do_sample=True, temperature=0.7)
    with pytest.raises(ValueError, match="do_sample=False"):
        model.generate(**enc, max_new_tokens=4, num_beams=2)
    model.generation_defaults = dict(repetition_penalty=1.05)
    with pytest.raises(ValueError, match="repetition_penalty"):
        model.generate(**enc, max_new_tokens=4, num_beams=2)
    model.generation_defaults = None
    model.tp_size = 2
    with pytest.raises(ValueError, match="single-GPU"):
        model.generate(**enc, max_new_tokens=4, num_beams=2)
    model.tp_size = 1
    assert model.pool.available() == free
    taken = model.pool.alloc(free - 3)
    with pytest.raises(RuntimeError, match="KV cache exhausted"):                # does not fit: takes nothing
        model.generate(**enc, max_new_tokens=4, num_beams=2)
    assert model.pool.available() == 3
    model.pool.release(taken)


def test_num_beams_one_is_the_plain_call(cabi_double):
    _, _, model, proc = _chatts(cabi_double)
    enc = proc(text=["one prompt here", "and another"], timeseries=[], padding=True, return_tensors="pt")
    a = model.generate(**enc, max_new_tokens=6)
    b = model.generate(**enc, max_new_tokens=6, num_beams=1, num_return_sequences=1)
    assert torch.equal(a, b) and model.last_beam_scores is None


class _Recorder(BeamDouble):
    """Checks the page plan after every selection + fork: each row's tail is written by that row only, spares are in no table, and the
    contents of every full page a table references never change afterwards."""

    def __init__(self):
        super().__init__()
        self.frozen, self.steps = {}, 0

    def beam_select(self, *a, **k):
        super().beam_select(*a, **k)
        names = ("batch", "num_beams", "keep", "vocab", "cand_ids", "cand_logprobs", "eos_ids", "len_den", "max_new", "early_stopping",
                 "length_penalty", "run_scores", "fin_scores", "fin_info", "prompt_flags", "step_ptr", "bp_tokens", "bp_parents",
                 "cur_ids", "positions", "seq_lens", "slot_map", "page_table", "page_table_old", "own_pages", "spare_pages", "page_size",
                 "fork")
        self.last = dict(zip(names, a), **k)

    def beam_fork_kv(self, kv, fork, rows):
        super().beam_fork_kv(kv, fork, rows)
        L = self.last
        ps, pt, pos = L["page_size"], L["page_table"], L["positions"]
        tails = [int(pt[r, int(pos[r]) // ps]) for r in range(rows)]
        assert len(set(tails)) == rows, tails                                   # no page is the tail of two rows
        full = {int(pt[r, c]) for r in range(rows) for c in range(int(pos[r]) // ps)}
        spares = {int(p) for p in L["spare_pages"]}
        assert not (full & set(tails)) and not (spares & (full | set(tails)))
        for p in full:
            snap = kv[:, :, p].clone()
            if p in self.frozen:
                assert torch.equal(self.frozen[p], snap), p                    # a full page never changes
            else:
                self.frozen[p] = snap
        self.steps += 1


@pytest.mark.parametrize("page,nb,cached", [(4, 3, False), (5, 4, True), (16, 2, False)])
def test_page_plan_every_step(cabi_double, monkeypatch, page, nb, cached):
    from chatts_b200 import _cabi
    rec = _Recorder()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: rec)
    _, _, model, proc = _chatts(rec, page=page, cached=cached)
    enc = proc(text=["a prompt of some length", "short"], timeseries=[], padding=True, return_tensors="pt")
    free = model.pool.available()
    out = model.generate(**enc, max_new_tokens=12, num_beams=nb, ignore_eos=True, num_return_sequences=nb)
    assert rec.steps == 12 and out.shape[0] == 2 * nb
    assert model.pool.available() == free
    if cached:                                      # a second call hits the prompt pages the first indexed, and gives the same output
        rec.frozen = {}                             # pages return to the pool between calls
        again = model.generate(**enc, max_new_tokens=12, num_beams=nb, ignore_eos=True, num_return_sequences=nb)
        assert torch.equal(out, again) and model.last_cached_positions.sum() > 0
        assert model.pool.available() == free
