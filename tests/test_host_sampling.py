"""Sampled decoding (temperature / top-k / top-p) on CPU: the statement cts_sample_advance follows (tests/cabi_double.py
``sample_reference``: threshold sets by bisection over the 16-bit logit key, inverse CDF in index order, counter-based
uniform) against transformers' own logits warpers, and generate(do_sample=True) through the
double: reproducible per seed, top_k=1 == greedy, every token inside the kept set."""
import numpy as np
import pytest
import torch

from tests.cabi_double import TorchDouble
from tests.test_host_model import PROMPTS, _build, _series

DT = torch.bfloat16


@pytest.mark.parametrize("top_k,top_p,temp", [(0, 0.9, 0.7), (20, 1.0, 1.0), (50, 0.8, 0.2), (0, 1.0, 1.3), (5, 0.5, 1.0)])
def test_kept_set_matches_transformers_warpers(top_k, top_p, temp):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    g = torch.Generator().manual_seed(top_k + int(100 * top_p))
    row = (torch.randn(1000, generator=g) * 3).to(DT)
    tok, cdf, target, kept = TorchDouble.sample_reference(row, temp, top_k, top_p, seed=11, step=3, b=1)
    sc = TemperatureLogitsWarper(temp)(None, row.float()[None])
    if top_k:
        sc = TopKLogitsWarper(top_k)(None, sc)
    if top_p < 1.0:
        sc = TopPLogitsWarper(top_p)(None, sc)
    hf_kept = torch.isfinite(sc[0]).numpy()
    # identical up to ties of the 16-bit logits at the threshold (we keep all of them; HF keeps them by sort position)
    extra = kept & ~hf_kept
    assert not (hf_kept & ~kept).any()
    if extra.any():
        thr = row.float().numpy()[kept].min()
        assert (row.float().numpy()[extra] == thr).all()
    assert kept[tok] and 0 <= target <= cdf[-1]
    # the draw follows the renormalised kept distribution: empirical frequencies over many (seed, step) pairs
    p = np.diff(np.concatenate([[0.0], cdf])) / cdf[-1]
    idx = np.nonzero(kept)[0]
    draws = np.array([TorchDouble.sample_reference(row, temp, top_k, top_p, seed=s, step=s % 7, b=s % 3)[0] for s in range(400)])
    assert kept[draws].all()
    top = idx[np.argmax(p[idx])]
    assert abs((draws == top).mean() - p[top]) < 4 * np.sqrt(p[top] * (1 - p[top]) / 400) + 0.02


def test_uniform_stream_is_uniform_and_reproducible():
    u = np.array([(TorchDouble._splitmix64(7 ^ TorchDouble._splitmix64((s << 32) | b)) >> 40) / 2 ** 24 for s in range(200) for b in range(8)])
    assert 0 <= u.min() and u.max() < 1 and abs(u.mean() - 0.5) < 0.03 and abs(np.var(u) - 1 / 12) < 0.01
    assert len(set(u.tolist())) > 1590


def test_generate_samples_through_the_kernel(cabi_double):
    cfg, sd, model, proc = _build(cabi_double, split=1)
    enc = proc(text=PROMPTS, timeseries=list(_series()), padding=True, return_tensors="pt")
    kw = dict(max_new_tokens=10, do_sample=True, temperature=0.8, top_p=0.9, top_k=40, ignore_eos=True)
    a = model.generate(**enc, seed=5, **kw)
    b = model.generate(**enc, seed=5, **kw)
    c = model.generate(**enc, seed=6, **kw)
    assert torch.equal(a, b) and not torch.equal(a, c)                      # (seed, step, row) fixes every draw
    assert len(model.pool.free) == model.pool.num_pages
    # top_k = 1 is greedy decoding (up to exact ties of the 16-bit logits, which the kept set retains: use a row without ties)
    row = torch.arange(1000, dtype=torch.float32).mul(0.01).to(DT)
    row[417] = 50.0
    assert TorchDouble.sample_reference(row, 1.0, 1, 1.0, seed=3, step=0, b=0)[0] == 417


def test_repetition_penalty_matches_transformers_processor(cabi_double):
    """generate(repetition_penalty=...) == greedy decoding through transformers' RepetitionPenaltyLogitsProcessor on the same logits:
    the double's apply/mark statement against the library class, then the generate() plumbing (prompt ids marked once, every new
    token marked, the penalty applied before every argmax)."""
    import numpy as np
    from transformers import RepetitionPenaltyLogitsProcessor
    from tests.cabi_double import TorchDouble
    g = torch.Generator().manual_seed(3)
    V, B = 1000, 3
    logits = (torch.randn(B, V, generator=g) * 3).to(torch.bfloat16)
    ids = torch.randint(0, V, (B, 17), generator=g)
    want = RepetitionPenaltyLogitsProcessor(penalty=1.3)(ids, logits.clone().float()).to(torch.bfloat16)
    dbl = TorchDouble()
    seen = torch.zeros(B, (V + 31) // 32, dtype=torch.int32)
    dbl.rep_penalty_mark(ids.reshape(-1).to(torch.int32), torch.arange(B).repeat_interleave(17).to(torch.int32), seen, V)
    got = logits.clone()
    dbl.rep_penalty_apply(got, B, seen, 1.3)
    assert torch.equal(got, want)

    from tests.test_host_model import _build, _series
    cfg, sd, model, proc = _build(cabi_double)
    enc = proc(text=["A <ts><ts/> ? " + "ab" * 6], timeseries=[_series()[0]], return_tensors="pt")
    S = enc["input_ids"].shape[1]
    plain = model.generate(**enc, max_new_tokens=12, ignore_eos=True)[0, S:].tolist()
    pen = model.generate(**enc, max_new_tokens=12, ignore_eos=True, repetition_penalty=1.8)[0, S:].tolist()
    assert model.generate(**enc, max_new_tokens=12, ignore_eos=True, repetition_penalty=1.0)[0, S:].tolist() == plain
    # reference loop: the model's own next-token logits, penalised by the HF processor over (prompt + generated) before the argmax
    proc_hf = RepetitionPenaltyLogitsProcessor(penalty=1.8)
    hist = enc["input_ids"].clone()
    ref = []
    for _ in range(12):
        run = model.generate(input_ids=hist, attention_mask=torch.ones_like(hist), timeseries=enc["timeseries"], max_new_tokens=1, ignore_eos=True)
        # logits of this step: recompute through forward (same kernels) and penalise
        lg = model.forward(hist, torch.ones_like(hist), enc["timeseries"]).logits[:, 0].float()
        tok = int(proc_hf(hist, lg.clone()).to(torch.bfloat16).float().argmax(-1))
        ref.append(tok)
        hist = torch.cat([hist, torch.tensor([[tok]])], 1)
    assert pen == ref and pen != plain
