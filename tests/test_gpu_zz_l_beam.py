"""generate(num_beams=...) on the GPU (tiny model, bf16 and fp16, with and without CUDA graphs): after the search, every beam row's KV rows
in its page table equal the rows a fresh prefill of that row's tokens writes (the check that catches a wrong fork); every returned score
is the length-penalised sum of the oracle's teacher-forced log-probs of its tokens; the returned sequences are those of the beam search
restated in tests/beam_double.py driven by the oracle's logits, on prompts with an EOS id whose every selection margin exceeds the measured
error of the GPU's log-probs (asserted, not skipped); a cold call with prefix caching on gives the output of the call with it off; and
every page goes back to the pool."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from chatts_b200 import beam as beammod
from oracle import decoder as od
from tests.beam_double import beam_search
from tests.gpu_util import record, rel_err
from tests.test_gpu_zz_h_prefix_cache import _model, _proc, _weights

pytestmark = pytest.mark.gpu
PROMPTS = ["did the series go up or down?", "what is the value at the peak"]        # equal lengths: no padding
KV_BOUND = {torch.bfloat16: 2.5e-2, torch.float16: 4e-3}       # decode-written vs prefill-written rows (two evaluation orders)
SCORE_TOL = {torch.bfloat16: 5e-2, torch.float16: 1e-2}        # per generated token, against the same-dtype oracle


def _run(dt, graphs, cached, nb=4, new=14, page=16):
    model = _model("tiny", dt, cached, page=page, max_batch=8)
    model.use_cuda_graph = graphs
    proc = _proc(model.config)
    enc = proc(text=PROMPTS, timeseries=[], padding=True, return_tensors="pt")
    seen = {}
    sel = model.ctx.beam_select

    def spy(*a, **k):
        seen["bp"] = (a[16], a[17])
        return sel(*a, **k)
    model.ctx.beam_select = spy
    free = model.pool.available()
    out = model.generate(**enc, max_new_tokens=new, num_beams=nb, num_return_sequences=nb, ignore_eos=True)
    model.ctx.beam_select = sel
    assert model.pool.available() == free
    return model, enc, out, seen


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "eager"])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_beam_kv_rows_and_scores(dt, graphs):
    nb, new = 4, 14
    model, enc, out, seen = _run(dt, graphs, False, nb, new)
    B, S = enc["input_ids"].shape
    R, ps = B * nb, model.page_size
    st = model._steps[R]
    table, pos = st.page_table.cpu().numpy(), st.positions.cpu().numpy()
    bp_tok, bp_par = (t.cpu().numpy() for t in seen["bp"])
    steps = int(pos[0]) - S + 1
    worst = 0.0
    for r in range(R):
        hist = beammod.hypothesis(bp_tok, bp_par, (steps - 1, bp_par[steps - 1, r], bp_tok[steps - 1, r], 1))
        ids = torch.tensor([enc["input_ids"][r // nb].tolist() + hist[:-1]])
        n = ids.shape[1]
        assert n == int(pos[r])
        _, _, counts, lay = model._prepare_inputs(ids, None, None)
        pts, held = model._alloc_pages(lay.lens, 0)
        try:
            model._prefill(lay, counts, None, pts)
            torch.cuda.synchronize()
            idx = np.arange(n)
            fresh = model.kv[:, :, torch.from_numpy(pts[0, idx // ps].astype(np.int64)), :, torch.from_numpy(idx % ps)]
            mine = model.kv[:, :, torch.from_numpy(table[r, idx // ps].astype(np.int64)), :, torch.from_numpy(idx % ps)]
            worst = max(worst, rel_err(mine, fresh))
        finally:
            model.pool.release(held)
    record("beam_kv_rows", dtype=str(dt).split(".")[-1], graphs=graphs, rel_err=worst, bound=KV_BOUND[dt])
    assert worst <= KV_BOUND[dt], worst
    # scores: length-penalised (1.0) sum of the oracle's teacher-forced log-probs
    cfg = model.config
    sd = _weights("tiny", dt)[1]
    scores = model.last_beam_scores.numpy()
    err = 0.0
    for i in range(out.shape[0]):
        gen = [t for t in out[i, S:].tolist()]
        while gen and gen[-1] == cfg.pad_token_id:
            gen.pop()
        full = out[i, :S + len(gen)]
        h = od.forward_hidden(sd["model.embed_tokens.weight"][full], sd, cfg.to_dict(), od.State(cfg.num_hidden_layers))
        lp = F.log_softmax(od.logits(h, sd).float(), -1)
        tgt = full[S:]
        total = float(lp[torch.arange(S - 1, S - 1 + len(gen)), tgt].sum()) / len(gen)
        err = max(err, abs(total - float(scores[i])))
    record("beam_scores_vs_oracle", dtype=str(dt).split(".")[-1], graphs=graphs, max_abs_err=err, bound=SCORE_TOL[dt])
    assert err <= SCORE_TOL[dt], err
    assert torch.isfinite(model.last_beam_scores).all() and (np.diff(scores.reshape(B, nb), axis=1) <= 0).all()


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_prefix_caching_gives_the_same_beams(dt):
    _, _, off, _ = _run(dt, True, False)
    model, enc, on, _ = _run(dt, True, True)
    assert torch.equal(off, on)                                            # a cold call with caching on is the uncached call
    # a warm call computes only the suffix (cts_attn_prefill_paged), whose logits differ from a full prefill in the last bits, so its
    # beams are not compared bit for bit; it must hit the prompt pages the first call indexed and hand every page back
    again = model.generate(**enc, max_new_tokens=14, num_beams=4, num_return_sequences=4, ignore_eos=True)
    assert int(np.sum(model.last_cached_positions)) > 0 and again.shape[0] == on.shape[0]
    assert model.pool.available() == model.pool.num_pages                  # free or evictable: nothing held


# prompts whose every selection margin clears the error the GPU's log-probs carry (fp16: bf16 logits of this model tie exactly among
# the best candidates, so no bf16 prompt can have a margin); each ends some hypotheses at the EOS id
ORACLE_CASES = [  # text, num_beams, early_stopping, length_penalty, max_new_tokens, EOS id
    ("uyayopsi?bil", 2, True, 1.0, 6, 313),
]


def _oracle_log_probs(cfg, sd, prompt):
    def f(seqs):
        rows = []
        for sq in seqs:
            ids = torch.tensor(prompt + list(sq))
            h = od.forward_hidden(sd["model.embed_tokens.weight"][ids], sd, cfg.to_dict(), od.State(cfg.num_hidden_layers))
            rows.append(F.log_softmax(od.logits(h[-1:], sd).float(), -1)[0])
        return torch.stack(rows).numpy()
    return f


@pytest.mark.parametrize("sync_every", [1, 16])
@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "eager"])
@pytest.mark.parametrize("text,nb,es,lp,new,eos", ORACLE_CASES)
def test_sequences_match_the_oracle_driven_search(text, nb, es, lp, new, eos, graphs, sync_every):
    dt = torch.float16
    model = _model("tiny", dt, False, max_batch=8)
    model.use_cuda_graph = graphs
    cfg, sd = _weights("tiny", dt)
    enc = _proc(cfg)(text=[text], timeseries=[], return_tensors="pt")
    prompt, S = enc["input_ids"][0].tolist(), enc["input_ids"].shape[1]
    seen, logits = {}, []
    sel, lpk = model.ctx.beam_select, model.ctx.logprobs

    def spy_select(*a, **k):
        seen["bp"] = (a[16], a[17])
        return sel(*a, **k)

    def spy_logprobs(lg, rows, *a, **k):
        logits.append(lg[:rows].float().cpu().clone())              # the logits each step's candidates come from
        return lpk(lg, rows, *a, **k)
    model.ctx.beam_select, model.ctx.logprobs = spy_select, spy_logprobs
    try:
        out = model.generate(**enc, max_new_tokens=new, num_beams=nb, num_return_sequences=nb, eos_token_id=[eos], early_stopping=es,
                             length_penalty=lp, sync_every=sync_every)
    finally:
        model.ctx.beam_select, model.ctx.logprobs = sel, lpk
    assert model.pool.available() == model.pool.num_pages
    if sync_every == 1:
        assert len(logits) < new                                    # the done flags end the search early
    # the error of the GPU's log-probs: every step, every row, against the oracle on the same tokens
    oracle = _oracle_log_probs(cfg, sd, prompt)
    bp_tok, bp_par = (t.cpu().numpy() for t in seen["bp"])
    tol = 0.0
    for s, lg in enumerate(logits):
        hist = [beammod.hypothesis(bp_tok, bp_par, (s - 1, bp_par[s - 1, r], bp_tok[s - 1, r], 1)) if s else [] for r in range(nb)]
        tol = max(tol, float(np.abs(F.log_softmax(lg, -1).numpy() - oracle(hist)).max()))
    tol += 1e-6                                                     # cts_logprobs against torch's log_softmax of the same logits
    hyps, scores, _, margin = beam_search(lambda seqs: (oracle(seqs), tol), S, 1, nb, cfg.vocab_size, new, (eos,), lp, es, nb)
    record("beam_oracle_margin", graphs=graphs, sync_every=sync_every, logprob_err=tol, margin=margin)
    assert margin > 1, (margin, tol)
    assert any(h and h[-1] == eos for h in hyps[0])
    n = max(len(h) for h in hyps[0])
    assert out.shape == (nb, S + n)
    for i, h in enumerate(hyps[0]):
        assert out[i, S:S + len(h)].tolist() == h and (out[i, S + len(h):] == cfg.pad_token_id).all(), (i, out[i, S:], h)
        L = len(h)
        assert abs(float(model.last_beam_scores[i]) - float(scores[i])) <= L * tol / L ** lp + 1e-6
