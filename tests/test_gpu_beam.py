"""The beam-search kernels (csrc/beam.cu) bit for bit against their restatement (tests/beam_double.py): cts_beam_select over several steps
of random candidate sets with planted ties, EOS ids inside and outside the top num_beams, all three early_stopping modes and negative
length penalties; cts_beam_fork_kv on random caches with swaps, 3-cycles and tails at offsets 0, 1 and page_size - 1, every other byte
of the cache unchanged."""
import numpy as np
import pytest
import torch

from chatts_b200 import beam as beammod
from tests.beam_double import fork_reference, select_reference
from tests.gpu_util import ctx

pytestmark = pytest.mark.gpu
ES = {0: False, 1: True, 2: "never"}


def _state(rng, B, nb, keep, page, max_pages, max_new, plen):
    R = B * nb
    pages = rng.permutation(10_000)[: R * (max_pages + 2)].astype(np.int32)
    table = np.zeros((R, max_pages), dtype=np.int32)
    own = pages[: R * max_pages].reshape(R, max_pages).copy()
    spare = pages[R * max_pages: R * max_pages + R].copy()
    p0 = plen // page
    for b in range(B):
        shared = rng.integers(0, 10_000, p0)
        for j in range(nb):
            table[b * nb + j, :p0] = shared
            table[b * nb + j, p0] = own[b * nb + j, p0]
    run = np.zeros(R, dtype=np.float32)
    run.reshape(B, nb)[:, 1:] = -1e9
    flags = np.zeros((B, 2), dtype=np.int32)
    flags[:, 0] = 1
    return dict(run=run, fin_scores=np.full(R, -1e9, dtype=np.float32), fin_info=np.zeros((R, 4), dtype=np.int32), flags=flags,
                step=np.zeros(2, dtype=np.int32), bp_tok=np.zeros((max_new, R), dtype=np.int32), bp_par=np.zeros((max_new, R), dtype=np.int32),
                cur=np.zeros(R, dtype=np.int32), pos=np.full(R, plen - 1, dtype=np.int32), sl=np.full(R, plen, dtype=np.int32),
                slot=np.zeros(R, dtype=np.int32), table=table, own=own, spare=spare, fork=np.zeros((R, 3), dtype=np.int32))


def _candidates(rng, R, keep, V, eos, quant):
    ids = np.stack([rng.choice(V, keep, replace=False) for _ in range(R)]).astype(np.int32)
    for r in range(R):                                             # EOS among the candidates of some rows, at varying ranks
        if eos and rng.random() < 0.5 and not np.isin(eos, ids[r]).any():
            ids[r, rng.integers(0, keep)] = rng.choice(eos)
    assert all(len(set(row)) == keep for row in ids.tolist())      # distinct per row, as cts_logprobs gives them
    lp = -np.abs(rng.standard_normal((R, keep))).astype(np.float32) * 3
    lp = (np.round(lp * quant) / quant).astype(np.float32)        # coarse values: ties across and within rows
    order = np.lexsort((ids, -lp), axis=1)
    return np.take_along_axis(ids, order, 1), np.take_along_axis(lp, order, 1)


CASES = [  # name, B, nb, n_eos, es, lp, page, V, max_new, plen
    ("small-b1-es0", 1, 2, 1, 0, 1.0, 4, 50, 7, 5),
    ("small-b3-es1", 3, 3, 2, 1, -1.0, 4, 64, 9, 8),
    ("small-b2-never", 2, 4, 1, 2, 2.0, 5, 40, 8, 3),
    ("small-b2-never-neg", 2, 3, 0, 2, -0.5, 3, 30, 6, 7),
    ("b8-5beams", 8, 5, 1, 0, 0.0, 16, 152064, 20, 37),
    ("b4-6beams-2eos", 4, 6, 2, 1, 1.0, 64, 152064, 30, 64),
    ("b16-2beams", 16, 2, 1, 2, -1.0, 64, 1000, 12, 100),
]


@pytest.mark.parametrize("name,B,nb,n_eos,es,lp,page,V,max_new,plen", CASES, ids=[c[0] for c in CASES])
def test_select_matches_restatement(name, B, nb, n_eos, es, lp, page, V, max_new, plen):
    c = ctx()
    rng = np.random.default_rng(len(name) * 7 + B)
    keep = beammod.beams_to_keep(nb, n_eos)
    max_pages = (plen + max_new) // page + 2
    R = B * nb
    eos = rng.choice(V, n_eos, replace=False).astype(np.int32).tolist()
    host = _state(rng, B, nb, keep, page, max_pages, max_new, plen)
    d = {k: torch.from_numpy(v.copy()).cuda() for k, v in host.items()}
    den = beammod.len_den(max_new, lp)
    den_d, eos_d = torch.from_numpy(den).cuda(), torch.tensor(eos, dtype=torch.int32).cuda()
    old = torch.zeros_like(d["table"])
    for step in range(max_new):
        ids, lps = _candidates(rng, R, keep, V, eos, quant=4 if step % 2 else 64)
        ids_d, lps_d = torch.from_numpy(ids).cuda(), torch.from_numpy(lps).cuda()
        c.beam_select(B, nb, keep, V, ids_d, lps_d, eos_d, den_d, max_new, ES[es], lp, d["run"], d["fin_scores"], d["fin_info"], d["flags"],
                      d["step"], d["bp_tok"], d["bp_par"], d["cur"], d["pos"], d["sl"], d["slot"], d["table"], old, d["own"], d["spare"],
                      page, d["fork"])
        h = host
        select_reference(B, nb, keep, V, ids, lps, eos, den, max_new, es, lp, h["run"], h["fin_scores"], h["fin_info"], h["flags"], h["step"],
                         h["bp_tok"], h["bp_par"], h["cur"], h["pos"], h["sl"], h["slot"], h["table"], h["own"], h["spare"], page, h["fork"])
        torch.cuda.synchronize()
        for k, v in host.items():
            got = d[k].cpu().numpy()
            assert np.array_equal(got.view(np.int32) if got.dtype == np.float32 else got,
                                  v.view(np.int32) if v.dtype == np.float32 else v), (name, step, k, got, v)


FORKS = [  # name, L, nkv, page, d, pattern
    ("small-swap", 2, 2, 16, 64, "swap"),
    ("small-cycle3", 2, 2, 16, 64, "cycle3"),
    ("small-offsets", 1, 2, 8, 16, "offsets"),
    ("14b-all-fork", 48, 8, 64, 128, "cycle3"),
]


@pytest.mark.parametrize("name,L,nkv,page,d,pattern", FORKS, ids=[f[0] for f in FORKS])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_fork_kv_copies_only_the_tail_rows(name, L, nkv, page, d, pattern, dt):
    c = ctx()
    rows = 30 if name.startswith("14b") else 9
    P = 3 * rows + 4
    g = torch.Generator().manual_seed(3)
    kv = torch.randn(L, 2, P, nkv, page, d, generator=g).to(dt)
    tails = torch.randperm(P, generator=g)[:2 * rows].tolist()
    old, spare = tails[:rows], tails[rows:]
    if pattern == "swap":
        parent = [1, 0, 3, 2, 4, 6, 5, 8, 7][:rows]
    elif pattern == "cycle3":
        parent = [(r // 3) * 3 + (r + 1) % 3 for r in range(rows)]
    else:
        parent = [(r + 1) % rows for r in range(rows)]
    offs = [(0, 1, page - 1)[r % 3] for r in range(rows)]
    fork = torch.tensor([[old[parent[r]], spare[r], offs[r]] if parent[r] != r else [0, 0, 0] for r in range(rows)], dtype=torch.int32)
    orig, ref = kv.clone(), kv.clone()
    fork_reference(ref, fork, rows)
    got = kv.cuda()
    c.beam_fork_kv(got, fork.cuda(), rows)
    torch.cuda.synchronize()
    assert torch.equal(got.cpu().view(torch.int16), ref.view(torch.int16))
    assert not torch.equal(ref.view(torch.int16), orig.view(torch.int16))       # the cases do copy something


def test_argument_errors_small():
    from chatts_b200._cabi import CtsError
    c = ctx()
    z = torch.zeros(64, dtype=torch.int32).cuda()
    f = torch.zeros(64, dtype=torch.float32).cuda()
    kw = dict(eos_ids=z[:1], len_den=f, max_new=4, early_stopping=False, length_penalty=1.0, run_scores=f, fin_scores=f, fin_info=z,
              prompt_flags=z, step_ptr=z, bp_tokens=z, bp_parents=z, cur_ids=z, positions=z, seq_lens=z, slot_map=z,
              page_table=z.view(8, 8), page_table_old=z.view(8, 8), own_pages=z, spare_pages=z, page_size=4, fork=z)
    with pytest.raises(CtsError, match="keep"):
        c.beam_select(1, 2, 3, 100, z, f, **kw)                     # keep < 2 * num_beams
    with pytest.raises(CtsError, match="num_beams"):
        c.beam_select(1, 11, 22, 100, z, f, **kw)
    with pytest.raises(CtsError, match="vocab"):
        c.beam_select(1, 2, 4, 3, z, f, **kw)
    with pytest.raises(CtsError, match="aligned"):
        c.beam_fork_kv(torch.zeros(1, 2, 4, 1, 4, 8, dtype=torch.bfloat16).cuda().view(-1)[1:33].view(1, 2, 1, 1, 4, 4), z, 1)
