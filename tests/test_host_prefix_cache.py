"""Prefix caching on CPU: the page keys (series content, page boundaries, the capped last page, seeds), the caching page pool
(reference counts, LRU eviction, deepest-first release, all-or-nothing allocation), the refusals under tensor parallelism, and the
model / ContinuousEngine / LLM / AsyncEngineArgs / server surfaces through the C-ABI double (tests/prefix_double.py)."""
import numpy as np
import pytest
import torch

from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer, layout
from chatts_b200.prefix_cache import CachingPagePool, chain_seed, page_keys, series_digests
from chatts_b200.weights import synthetic_state_dict
from tests.prefix_double import PrefixDouble

DT = torch.bfloat16


@pytest.fixture
def cabi_double(cabi_double, monkeypatch):
    from chatts_b200 import _cabi
    dbl = PrefixDouble()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: dbl)
    return dbl


def _series(seed, n=96):
    return np.sin(np.arange(n) / (2.0 + seed)) * (1 + seed)


def _lay(ids, cnt, mode="insert"):
    return layout.hf_layout(np.asarray(ids)[None], None, cnt, 100, mode)


# ------------------------------------------------------------------------------------------------------------------------- keys
def test_keys_follow_series_content_and_page_boundaries():
    seed = chain_seed("insert", 4, 0)
    lay = _lay([1, 2, 100, 101, 4, 5, 6, 7, 8], [3])        # <ts> at 2, its 3 patch rows at 3-5: page 0 already holds a row
    assert lay.total == 12
    s1, s2 = series_digests(torch.tensor(_series(1))[None, :, None]), series_digests(torch.tensor(_series(2))[None, :, None])
    k1, k2 = page_keys(lay, s1, [3], seed, 4)[0], page_keys(lay, s2, [3], seed, 4)[0]
    assert len(k1) == 3 and len(set(k1)) == 3                # full pages only, one key each
    assert all(a != b for a, b in zip(k1, k2))               # other series, same ids: no page in common from the first row on
    assert len(page_keys(_lay([1, 2, 100, 101, 4, 5, 6, 7], [3]), s1, [3], seed, 4)[0]) == 2     # 11 positions: 2 full pages
    assert page_keys(lay, s1, [3], seed, 4)[0] == k1                                             # deterministic
    assert page_keys(lay, s1, [3], chain_seed("insert", 4, 1), 4)[0][0] != k1[0]                  # another epoch: another chain


def test_text_prefix_shared_series_pages_not():
    seed = chain_seed("insert", 4, 0)
    ids = [1, 2, 3, 4, 100, 101, 5, 6, 7, 8]                 # <ts> at 4: page 0 = text only, rows at 5-7
    lay = _lay(ids, [3])
    s1, s2 = series_digests(torch.tensor(_series(1))[None, :, None]), series_digests(torch.tensor(_series(2))[None, :, None])
    k1, k2 = page_keys(lay, s1, [3], seed, 4)[0], page_keys(lay, s2, [3], seed, 4)[0]
    assert k1[0] == k2[0] and all(a != b for a, b in zip(k1[1:], k2[1:]))
    # another question after the same series: the pages in front of the first difference are shared, the chain parts at it
    k3 = page_keys(_lay([1, 2, 3, 4, 100, 101, 5, 6, 9, 9], [3]), s1, [3], seed, 4)[0]
    assert k3[:2] == k1[:2] and k3[2] != k1[2]
    # the patch index is part of the content: the same series at another offset is another chain
    k4 = page_keys(_lay([1, 2, 3, 100, 101, 4, 5, 6, 7, 8], [3]), s1, [3], seed, 4)[0]
    assert k4[1] != k1[1]


def test_seed_covers_mode_page_size_and_epoch_and_padding_does_not_matter():
    seeds = {chain_seed(m, p, e) for m in ("insert", "overwrite") for p in (16, 32) for e in (0, 1)}
    assert len(seeds) == 8
    a = torch.tensor(_series(1), dtype=torch.float32)
    padded = torch.cat([a, torch.zeros(40)])
    assert series_digests(a[None, :, None]) == series_digests(padded[None, :, None])
    assert series_digests(a[None, :, None]) != series_digests(a[None, :, None].to(torch.float64))
    b = a.clone()
    b[50] += 1e-3
    assert series_digests(a[None, :, None]) != series_digests(b[None, :, None])


# ------------------------------------------------------------------------------------------------------------------------- pool
def test_pool_refcounts_lru_and_deepest_first_release():
    pool = CachingPagePool(6)
    a = pool.alloc(3)
    for i, p in enumerate(a):
        assert pool.register(f"a{i}", p)
    assert not pool.register("a0", 5) and not pool.register("zz", a[0])
    pool.acquire(pool.lookup(["a0", "a1", "x"]))             # a second holder of the first two pages
    assert [pool.ref[p] for p in a] == [2, 2, 1]
    pool.release(a[:2])
    assert [pool.ref[p] for p in a] == [1, 1, 1] and pool.available() == 3
    pool.release(a)                                          # deepest first: a2, then a1, then a0 become evictable
    assert list(pool.evictable) == [a[2], a[1], a[0]] and pool.available() == 6
    b = pool.alloc(4)                                        # 3 never-cached pages first, then the LRU one: the chain's tail
    assert a[2] in b and a[1] not in b and pool.evictions == 1
    assert pool.lookup(["a0", "a1", "a2"]) == [a[0], a[1]]
    pool.release(b)
    assert pool.available() == 6 and len(pool.free) == 4
    pool.clear()
    assert pool.lookup(["a0"]) == [] and len(pool.free) == 6 and not pool.ref
    with pytest.raises(RuntimeError, match="exhausted"):
        pool.alloc(7)


def _model(cabi_double, cached=True, max_batch=4, max_seq_len=256, **kw):
    from chatts_b200.model import ChatTSForCausalLM
    cfg = ChatTSConfig.tiny()
    sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=DT, std=0.05)
    m = ChatTSForCausalLM(cfg, sd, device="cpu", dtype=DT, max_batch=max_batch, max_seq_len=max_seq_len, page_size=16,
                          use_cuda_graph=False, enable_prefix_caching=cached, **kw)
    return cfg, sd, m, ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)


def _enc(proc, question, seed=1):
    return proc(text=["Look at <ts><ts/> then answer: " + question], timeseries=[_series(seed, 160)], return_tensors="pt")


def test_model_hits_caps_and_all_or_nothing(cabi_double):
    cfg, sd, m, proc = _model(cabi_double, max_batch=2, max_seq_len=256)
    enc = _enc(proc, "what is the trend?")
    _, _, counts, lay = m._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
    n = int(lay.lens[0])
    pts, held, keys, cached = m._alloc_prompt(lay, enc["timeseries"], 4)
    assert cached.tolist() == [0] and len(keys[0]) == n // 16
    m._prefix_register(keys, pts, lay.lens, cached)
    m.pool.release(held)
    assert m.prefix_cache_stats()["cached_pages"] == n // 16
    # the same prompt again: every full page but the one holding the last position
    pts2, held2, _, cached2 = m._alloc_prompt(lay, enc["timeseries"], 4)
    assert int(cached2[0]) == (n - 1) // 16 * 16 and pts2[0, : (n - 1) // 16].tolist() == pts[0, : (n - 1) // 16].tolist()
    other = m.pool.alloc(10)
    free_before, ref_before, lru_before = list(m.pool.free), dict(m.pool.ref), list(m.pool.evictable)
    two = layout.hf_layout(np.concatenate([enc["input_ids"]] * 2), None, np.concatenate([m._host_counts[1].numpy()] * 2),
                           cfg.ts_token_start_index)
    m._host_counts = tuple(torch.cat([h, h]) for h in m._host_counts)
    with pytest.raises(RuntimeError, match="exhausted"):     # 2 x 8 new pages, 12 free or evictable: nothing may be taken
        m._alloc_prompt(two, torch.cat([enc["timeseries"]] * 2), 100)
    assert m.pool.free == free_before and m.pool.ref == ref_before and list(m.pool.evictable) == lru_before
    m.pool.release(other)
    m.pool.release(held2)
    assert m.pool.available() == m.pool.num_pages
    st = m.prefix_cache_stats()
    assert st["queried_positions"] == 2 * n and st["hit_positions"] == int(cached2[0])


def test_generate_warm_equals_cold_and_invalidation(cabi_double):
    cfg, sd, m, proc = _model(cabi_double)
    _, _, ref, _ = _model(cabi_double, cached=False)
    for q in ("what is the trend?", "is there a spike?"):
        enc = _enc(proc, q)
        out = m.generate(**enc, max_new_tokens=4, ignore_eos=True)
        assert torch.equal(out, ref.generate(**enc, max_new_tokens=4, ignore_eos=True))
    assert int(m.last_cached_positions[0]) > 0 and ref.last_cached_positions is None
    ad = {"model.layers.0.self_attn.q_proj.lora_A.weight": torch.randn(4, cfg.hidden_size) * 0.05,
          "model.layers.0.self_attn.q_proj.lora_B.weight": torch.randn(cfg.num_attention_heads * cfg.head_dim, 4) * 0.05}
    m.merge_lora(ad, lora_alpha=8, r=4)
    assert m.prefix_cache_stats()["cached_pages"] == 0
    m.generate(**_enc(proc, "is there a spike?"), max_new_tokens=2, ignore_eos=True)
    assert int(m.last_cached_positions[0]) == 0
    m.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"])       # forward() never uses the cache
    assert m.pool.available() == m.pool.num_pages


def test_continuous_engine_shares_and_releases(cabi_double):
    from chatts_b200.engine import ContinuousEngine
    cfg, sd, m, proc = _model(cabi_double)
    eng = ContinuousEngine(m, slots=4, steps_per_round=2, max_prefill_batch=2)
    rids = []
    for i, q in enumerate(["a?", "bb?", "ccc?", "dddd?"]):
        enc = _enc(proc, q)
        rids.append(eng.add_request(enc["input_ids"][0], enc["timeseries"], max_new_tokens=3, ignore_eos=True))
        if i == 1:
            eng.step()
    eng.run()
    done = {r.rid: r for r in eng.finished}
    eng.close()
    assert [done[r].cached_positions > 0 for r in rids] == [False, False, True, True]
    assert m.pool.available() == m.pool.num_pages and not any(m.pool.ref.values())


def test_refusals_under_tensor_parallelism(monkeypatch):
    from chatts_b200 import vllm_compat
    from chatts_b200.model import ChatTSForCausalLM
    with pytest.raises(ValueError, match="single-GPU"):
        ChatTSForCausalLM(ChatTSConfig.tiny(), {}, tp_size=2, enable_prefix_caching=True)
    import torch.multiprocessing as mp
    monkeypatch.setattr(mp, "get_context", lambda *a, **k: pytest.fail("a worker was spawned"))
    with pytest.raises(ValueError, match="single-GPU"):
        vllm_compat.LLM(config=ChatTSConfig.tiny(), tensor_parallel_size=2, enable_prefix_caching=True)


def test_llm_async_args_and_server_surfaces(cabi_double):
    from chatts_b200 import server, vllm_compat
    cfg, sd, m, proc = _model(cabi_double)
    llm = vllm_compat.LLM(model=m, enable_prefix_caching=True)
    req = lambda q: {"prompt": "Look at <ts><ts/> then answer: " + q, "multi_modal_data": {"timeseries": [_series(1, 160)]}}
    sp = vllm_compat.SamplingParams(max_tokens=3, temperature=0.0)
    a = llm.generate(req("what is the trend?"), sp)[0]
    b = llm.generate(req("is there a spike?"), sp)[0]
    assert a.num_cached_tokens == 0 and b.num_cached_tokens > 0 and b.num_cached_tokens % 16 == 0
    _, _, plain, _ = _model(cabi_double, cached=False)
    assert vllm_compat.LLM(model=plain).generate(req("x"), sp)[0].num_cached_tokens == 0
    with pytest.raises(ValueError, match="enable_prefix_caching"):
        vllm_compat.LLM(model=plain, enable_prefix_caching=True)
    assert vllm_compat.AsyncEngineArgs().enable_prefix_caching is False
    assert vllm_compat.AsyncEngineArgs(enable_prefix_caching=True).enable_prefix_caching is True
    assert server.parse_args(["--enable-prefix-caching"]).enable_prefix_caching is True
    assert server.parse_args([]).enable_prefix_caching is False
