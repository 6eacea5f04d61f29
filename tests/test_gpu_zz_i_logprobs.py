"""Log probabilities of generate() and ContinuousEngine on the GPU: tokens are bit-identical with logprobs on and off on every single-GPU
decode path; every returned logprob, rank and top-k entry is log_softmax of the logits the token was picked from (captured by
tests/gpu_util.py:decode_run) within the kernel tolerance; prompt logprobs are log_softmax of forward(logits_to_keep=0) at the mapped
positions, in insert and overwrite mode with a left-padded batch; a prompt-logprob call does not use the prefix cache but indexes its
pages; the engine serves mixed requests."""
import numpy as np
import pytest
import torch

from tests.gpu_util import decode_run, record
from tests.test_gpu_zz_h_prefix_cache import _model, _proc, _series

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
TOL = 1e-5
STEPS = 5
K = 5


def _enc(cfg, proc, with_ts=True):
    if with_ts:
        return proc(text=["the series <ts><ts/> went up or down?", "compare <ts><ts/> and <ts><ts/> please"],
                    timeseries=[_series(1), _series(2, 96), _series(3, 64)], padding=True, return_tensors="pt")
    return proc(text=["a b c d e f", "g h"], timeseries=[], padding=True, return_tensors="pt")


def _lp_of(logits):
    """log_softmax in float64 (torch's fp32 log_softmax on the CPU is itself up to ~2e-5 off at a 152k vocabulary)."""
    return torch.log_softmax(logits.double(), -1)


def _check_decode(res, run, B):
    lgs = torch.cat([run.prefill[None], run.logits])                         # [STEPS + 1, B, V]
    toks = run.tokens.long()
    worst = 0.0
    for j in range(STEPS + 1):
        lp = _lp_of(lgs[j])
        for b in range(B):
            t = int(toks[b, j])
            worst = max(worst, abs(float(res.logprobs[b, j]) - float(lp[b, t])))
            assert int(res.ranks[b, j]) == 1 + int((lgs[j, b] > lgs[j, b, t]).sum())
            vals = lp[b, torch.from_numpy(res.top_ids[b, j].astype(np.int64))]
            assert np.allclose(res.top_logprobs[b, j], vals.numpy(), atol=TOL, rtol=0)
            order = sorted(range(lgs.shape[2]), key=lambda i: (-float(lgs[j, b, i]), i))[:K]
            assert res.top_ids[b, j].tolist() == order
    assert worst <= TOL, worst
    return worst


CASES = ([(kind, dt, "default") for kind in ("tiny", "small128", "l14b") for dt in (BF, FP)]
         + [("tiny", BF, p) for p in ("native", "eager", "fp8", "w4_mma")])


@pytest.mark.parametrize("kind,dt,path", CASES, ids=lambda v: v if isinstance(v, str) else str(v).split(".")[-1])
def test_decode_logprobs_match_the_logits(kind, dt, path, monkeypatch):
    monkeypatch.setenv("CTS_W4_KERNEL", "mma")
    monkeypatch.setenv("CTS_NATIVE_STEP", "1" if path == "native" else "0")
    if path == "w4_mma":                                  # the decode-parity model whose every K suits the mma W4 kernel
        from tests.test_gpu_zz_g_decode_parity import _model as _parity_model
        model = _parity_model("tiny_w4", dt, path, 4, 16)[3]
    else:
        model = _model(kind, dt, False)
    if path == "eager":
        model.use_cuda_graph = False
    elif path == "fp8":
        model.quantize_fp8()
    cfg = model.config
    enc = _enc(cfg, _proc(cfg), with_ts=kind != "l14b")
    B = enc["input_ids"].shape[0]
    off = model.generate(**enc, max_new_tokens=STEPS + 1, ignore_eos=True)
    on = model.generate(**enc, max_new_tokens=STEPS + 1, ignore_eos=True, logprobs=K)
    assert torch.equal(off, on)
    res = model.last_logprobs
    run = decode_run(model, enc, STEPS)
    S = enc["input_ids"].shape[1]
    assert torch.equal(run.tokens.long(), on[:, S:])
    worst = _check_decode(res, run, B)
    record("decode_logprobs", kind=kind, dtype=str(dt).split(".")[-1], path=path, max_abs_err=worst)


@pytest.mark.parametrize("mode", ["insert", "overwrite"])
@pytest.mark.parametrize("dt", [BF, FP], ids=["bf16", "fp16"])
@pytest.mark.parametrize("kind", ["tiny", "small128"])
def test_prompt_logprobs_match_forward(kind, dt, mode, monkeypatch):
    monkeypatch.setenv("CTS_TS_MERGE_MODE", mode)
    model = _model(kind, dt, False)
    cfg = model.config
    enc = _enc(cfg, _proc(cfg))
    full = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"], logits_to_keep=0).logits
    model.generate(**enc, max_new_tokens=2, ignore_eos=True, prompt_logprobs=K)
    res = model.last_logprobs
    _, _, _, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
    ids, am = enc["input_ids"].numpy(), enc["attention_mask"].numpy()
    worst, n, ts = 0.0, 0, cfg.ts_token_start_index
    for r in range(ids.shape[0]):
        kept = np.nonzero(am[r])[0]
        assert len(res.prompt[r]) == kept.shape[0] and res.prompt[r][0] is None
        cu0 = int(lay.cu_seqlens[r])
        merged = {int(c): j - cu0 for j, c in enumerate(lay.src_col) if cu0 <= j < int(lay.cu_seqlens[r + 1]) and c >= 0}
        lg = full[r].float().cpu()
        lp = _lp_of(lg)
        for e, c in enumerate(kept[1:], start=1):
            ent, tok = res.prompt[r][e], int(ids[r, c])
            if mode == "overwrite" and tok in (ts, ts + 1):
                assert ent is None
                continue
            j = merged[int(c)] - 1
            worst = max(worst, abs(ent.logprob - float(lp[j, tok])))
            assert ent.token_id == tok and ent.rank == 1 + int((lg[j] > lg[j, tok]).sum())
            order = sorted(range(lg.shape[1]), key=lambda i: (-float(lg[j, i]), i))[:K]
            assert ent.top_ids == order
            n += 1
    assert n > 0 and worst <= TOL, worst
    record("prompt_logprobs", kind=kind, dtype=str(dt).split(".")[-1], mode=mode, entries=n, max_abs_err=worst)


def test_prompt_logprobs_with_prefix_caching():
    model = _model("tiny", BF, True)
    cfg = model.config
    enc = _proc(cfg)(text=["a question about <ts><ts/> that is long enough to fill pages " * 2], timeseries=[_series(4), _series(5)],
                     return_tensors="pt")
    base = model.generate(**enc, max_new_tokens=3, ignore_eos=True)
    ref = model.generate(**enc, max_new_tokens=3, ignore_eos=True, prompt_logprobs=2)
    assert int(model.last_cached_positions[0]) == 0 and torch.equal(ref, base)
    full = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"], logits_to_keep=0).logits[0]
    ent = model.last_logprobs.prompt[0][1]
    assert abs(ent.logprob - float(_lp_of(full[0].cpu())[ent.token_id])) <= TOL
    again = model.generate(**enc, max_new_tokens=3, ignore_eos=True)
    assert int(model.last_cached_positions[0]) > 0 and torch.equal(again, base)


def test_continuous_engine_mixed_requests():
    from chatts_b200.engine import ContinuousEngine
    model = _model("tiny", BF, False)
    cfg = model.config
    proc = _proc(cfg)
    texts, ks = ["a b c d", "the series <ts><ts/> ?", "x y", "more words here"], [None, 3, 0, 20]
    series = {1: [_series(7)]}
    eng = ContinuousEngine(model, slots=4, steps_per_round=3)
    encs = []
    for i, (t, k) in enumerate(zip(texts, ks)):
        e = proc(text=[t], timeseries=series.get(i, []), return_tensors="pt")
        encs.append(e)
        eng.add_request(e["input_ids"][0], e.get("timeseries"), max_new_tokens=7, ignore_eos=True, logprobs=k)
    done = eng.run()
    eng.close()
    worst = 0.0
    for r, e, k in zip(done, encs, ks):
        out = model.generate(**e, max_new_tokens=7, ignore_eos=True, logprobs=k)
        assert r.tokens == out[0, -7:].tolist()
        if k is None:
            assert r.token_logprobs == []
            continue
        res = model.last_logprobs
        for j, (lp, rank, ids, vals) in enumerate(r.token_logprobs):
            worst = max(worst, abs(lp - float(res.logprobs[0, j])))
            assert len(ids) == k and len(vals) == k
    # the engine decodes 4 slots where generate() decodes 1: the logits may differ in their last bits (5.2e-4 measured on an H100)
    record("engine_logprobs", max_abs_diff_vs_generate=worst)
    assert worst <= 5e-3, worst
