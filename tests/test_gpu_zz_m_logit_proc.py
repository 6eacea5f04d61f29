"""Logits processors of generate() and the continuous engine on the GPU (tiny model, SimpleTokenizer): neutral values bitwise equal to a
call without them; logit_bias={eos: 100} with min_new_tokens=k gives exactly k tokens and then EOS, and every token lies in
allowed_token_ids, greedy and seeded sampled at batch 1 and 4; with logprobs on, every greedily chosen token has rank 1 in the processed
distribution; the engine gives a penalised request the tokens of a stand-alone generate() and leaves neutral neighbours bitwise as they
are, and a slot reused by requests with different processor fields keeps nothing of the previous one; every page returns to the pool."""
import pytest
import torch

from tests.test_gpu_zz_h_prefix_cache import _model, _proc

pytestmark = pytest.mark.gpu
PROMPTS = ["did the series go up?", "answer with a label", "x", "what is the value at the peak?"]
ALLOWED = list(range(97, 123)) + [32]


def _setup(dt=torch.bfloat16):
    model = _model("tiny", dt, False)
    return model, _proc(model.config)


def _enc(proc, texts):
    return proc(text=texts, timeseries=[], padding=True, return_tensors="pt")


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_neutral_values_are_the_plain_call(dt):
    model, proc = _setup(dt)
    enc = _enc(proc, PROMPTS)
    a = model.generate(**enc, max_new_tokens=12, ignore_eos=True)
    b = model.generate(**enc, max_new_tokens=12, ignore_eos=True, presence_penalty=0.0, frequency_penalty=0.0, logit_bias={},
                       allowed_token_ids=None, min_new_tokens=0)
    assert torch.equal(a, b) and model.pool.available() == model.pool.num_pages


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("sample", [None, 7])
@pytest.mark.parametrize("k", [1, 5])
def test_eos_bias_with_min_new_tokens(B, sample, k):
    model, proc = _setup()
    enc = _enc(proc, PROMPTS[:B])
    S = enc["input_ids"].shape[1]
    eos = model.config.eos_token_id
    kw = {} if sample is None else dict(do_sample=True, temperature=1.0, top_p=0.95, seed=sample)
    ids = model.generate(**enc, max_new_tokens=16, logit_bias={eos: 100.0}, min_new_tokens=k, **kw)
    assert ids.shape[1] == S + k + 1
    for row in ids[:, S:].tolist():
        assert eos not in row[:k] and row[k] == eos, row
    assert model.pool.available() == model.pool.num_pages


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("sample", [None, 3])
def test_allowed_token_ids(B, sample):
    model, proc = _setup()
    enc = _enc(proc, PROMPTS[:B])
    S = enc["input_ids"].shape[1]
    kw = {} if sample is None else dict(do_sample=True, temperature=1.0, top_k=50, seed=sample)
    ids = model.generate(**enc, max_new_tokens=20, ignore_eos=True, allowed_token_ids=ALLOWED, presence_penalty=0.5, **kw)
    assert set(ids[:, S:].reshape(-1).tolist()) <= set(ALLOWED)
    assert model.pool.available() == model.pool.num_pages


def test_logprobs_describe_the_processed_logits():
    model, proc = _setup()
    enc = _enc(proc, PROMPTS)
    S = enc["input_ids"].shape[1]
    ids = model.generate(**enc, max_new_tokens=12, ignore_eos=True, logprobs=5, frequency_penalty=1.5, presence_penalty=0.5,
                         logit_bias={101: 4.0}, repetition_penalty=1.2)
    lp = model.last_logprobs
    n = ids.shape[1] - S
    assert (lp.ranks[:, :n] == 1).all()
    assert (lp.top_ids[:, :n, 0] == ids[:, S:].numpy()).all()


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_continuous_engine(dt):
    from chatts_b200.engine import ContinuousEngine
    model, proc = _setup(dt)
    pen = dict(presence_penalty=0.8, frequency_penalty=0.4, repetition_penalty=1.3, logit_bias={101: 3.0}, min_tokens=4)
    alone = []
    for p in PROMPTS:
        enc = _enc(proc, [p])
        S = enc["input_ids"].shape[1]
        alone.append(model.generate(**enc, max_new_tokens=14, ignore_eos=True,
                                    **{("min_new_tokens" if k == "min_tokens" else k): v for k, v in pen.items()})[0, S:].tolist())

    def run(penalised):
        eng = ContinuousEngine(model, slots=4, steps_per_round=3)
        rids = [eng.add_request(_enc(proc, [p])["input_ids"][0], max_new_tokens=14, ignore_eos=True, **(pen if i in penalised else {}))
                for i, p in enumerate(PROMPTS)]
        done = {r.rid: r.tokens for r in eng.run()}
        eng.close()
        return [done[r] for r in rids]
    plain, mixed = run(()), run((1, 3))
    assert mixed[1] == alone[1] and mixed[3] == alone[3]
    assert mixed[0] == plain[0] and mixed[2] == plain[2]                    # neutral neighbours: unchanged
    assert mixed[1] != plain[1]
    assert model.pool.available() == model.pool.num_pages


def test_continuous_engine_slot_reuse():
    from chatts_b200.engine import ContinuousEngine
    model, proc = _setup()
    eos = model.config.eos_token_id
    reqs = [(PROMPTS[0], dict(min_tokens=3, presence_penalty=0.5, logit_bias={101: 2.0}, allowed_token_ids=ALLOWED + [eos])),
            (PROMPTS[1], dict(ignore_eos=True, logit_bias={eos: 100.0}, min_tokens=3)),
            (PROMPTS[2], dict(frequency_penalty=0.7, min_tokens=2)),
            (PROMPTS[3], dict())]
    want = []
    for p, kw in reqs:
        enc = _enc(proc, [p])
        S = enc["input_ids"].shape[1]
        want.append(model.generate(**enc, max_new_tokens=6, **{("min_new_tokens" if k == "min_tokens" else k): v
                                                                for k, v in kw.items()})[0, S:].tolist())
    assert want[1] == [eos] * 6
    eng = ContinuousEngine(model, slots=1, steps_per_round=2)
    rids = [eng.add_request(_enc(proc, [p])["input_ids"][0], max_new_tokens=6, **kw) for p, kw in reqs]
    done = {r.rid: r.tokens for r in eng.run()}
    eng.close()
    for rid, w in zip(rids, want):
        toks = done[rid]
        assert toks == w[:len(toks)] and (len(toks) == 6 or toks[-1] == eos), (toks, w)
    assert model.pool.available() == model.pool.num_pages
