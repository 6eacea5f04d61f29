"""FP8 weights (ChatTSForCausalLM.quantize_fp8): cts_gemm_fp8 (csrc/gemm_fp8.cu: e4m3 codes converted in registers, mma.sync, fp32
split-K partials scaled per row) against an fp32 matmul of W' = fp32(code) * s, every e4m3 code through every fragment position exactly,
cts_fp8_dequant bit for bit against the host statement, and the whole model after quantize_fp8() against the oracle on W'."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import decoder as od
from oracle import merge as om
from oracle import ts_encoder as ote
from tests.gpu_util import ctx, parity_gate, record

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FINITE = [c for c in range(256) if c not in (0x7F, 0xFF)]          # the 254 finite e4m3fn codes (+-0 and the subnormals included)


def _rand_codes(n, k, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(0, 256, (n, k), generator=g, dtype=torch.uint8)
    q[(q == 0x7F) | (q == 0xFF)] = 0
    s = (torch.rand(n, generator=g) + 0.5) * 1e-4
    return q.cuda(), s.cuda()


@pytest.mark.parametrize("t", [8, 16, 32])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_fp8_every_code_exact_at_every_fragment_position(dtype, t):
    """One-hot activations: partial[0][t][n] = s_n * e4m3(q[n][k_t]) with a single non-zero product, so the kernel's result must equal
    fp32(code) * s_n EXACTLY.  The codes cycle so that each of the 254 finite codes sits at every (row % 16, k % 16) of the m16n8k16
    fragments (1024 rows x 64 K: 256 instances per position)."""
    from chatts_b200.weights import pack_fp8_mma
    c = ctx()
    n, k = 1024, 64
    r, col = torch.arange(n)[:, None], torch.arange(k)[None, :]
    idx = ((r // 16) * (k // 16) + col // 16 + 7 * (r % 16) + 3 * (col % 16)) % 254
    q = torch.tensor(FINITE, dtype=torch.uint8)[idx]
    for pos in range(256):                                     # every code at every fragment position
        rr, cc = pos // 16, pos % 16
        assert len(set(q[rr::16, cc::16].flatten().tolist())) == 254
    s = (torch.rand(n, generator=torch.Generator().manual_seed(1)) + 0.5) * 3e-3
    qw, sc = pack_fp8_mma(q).cuda(), s.cuda()
    want = q.view(torch.float8_e4m3fn).float() * s[:, None]               # [n, k]
    bad = 0
    for k0 in range(0, k, t):                                  # token i = unit vector k0 + i
        x = torch.zeros(t, k, dtype=dtype)
        x[torch.arange(t), k0 + torch.arange(t)] = 1
        out = torch.full((1, t, n), float("nan"), device="cuda")
        c.gemm_fp8(x.cuda(), qw, sc, k, out, 1, t=t)
        torch.cuda.synchronize()
        bad += int((out[0].cpu() != want[:, k0:k0 + t].t()).sum())
    record("gemm_fp8_every_code", dtype=str(dtype), t=t, mismatches=bad)
    assert bad == 0


# (n, k, t, split): tiny (K = 704), ChatTS-14B (qkv 7168 x 5120, o 5120 x 5120, gate_up 27648 x 5120, down 5120 x 13824), ChatTS-8B
# (qkv 6144 x 4096, o 4096 x 4096, gate_up 24576 x 4096, down 4096 x 12288), TP shards (qkv N = 896 at TP8, down K = 1728 / 3456 / 6912),
# ragged n (200, 528); t in {1, 5, 8, 17, 32}; split from 1 to the largest allowed (k / 64)
SHAPES = [(512, 704, 5, 1), (256, 704, 17, 11), (1408, 256, 32, 4), (256, 256, 1, 4),
          (7168, 5120, 1, 4), (5120, 5120, 8, 7), (27648, 5120, 32, 1), (27648, 5120, 5, 3), (5120, 13824, 17, 11),
          (6144, 4096, 8, 5), (4096, 4096, 32, 64), (24576, 4096, 1, 2), (4096, 12288, 5, 8),
          (896, 5120, 1, 16), (5120, 1728, 8, 27), (5120, 3456, 32, 6), (5120, 6912, 1, 13),
          (200, 768, 17, 3), (528, 1536, 32, 24), (200, 128, 1, 2)]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n,k,t,split", SHAPES)
def test_fp8_partials_match_an_fp32_matmul(n, k, t, split, dtype):
    """Each partial against an fp32 matmul of W' = fp32(code) * s over ITS K range (cut at multiples of 64), bound 2e-5 of the largest
    magnitude; outputs NaN-prefilled so an unwritten element shows."""
    from chatts_b200.weights import pack_fp8_mma
    c = ctx()
    q, s = _rand_codes(n, k, seed=n + k + t)
    qw = pack_fp8_mma(q)
    x = (torch.randn(t, k, generator=torch.Generator().manual_seed(3)) * 0.5).to(dtype).cuda()
    got = torch.full((split, t, n), float("nan"), device="cuda")
    c.gemm_fp8(x, qw, s, k, got, split, t=t)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(got).all())
    kb = k // 64
    w32, x32 = q.view(torch.float8_e4m3fn).float() * s[:, None], x.float()
    want = torch.stack([x32[:, kb * i // split * 64:kb * (i + 1) // split * 64] @ w32[:, kb * i // split * 64:kb * (i + 1) // split * 64].t()
                        for i in range(split)])
    err = float((got - want).abs().max() / want.abs().max())
    record("gemm_fp8", n=n, k=k, t=t, split=split, dtype=str(dtype), rel_err=err)
    assert err <= 2e-5


def test_fp8_suggested_split_is_in_range():
    c = ctx()
    for n, k in ((7168, 5120), (5120, 5120), (27648, 5120), (5120, 13824), (896, 5120), (5120, 1728), (512, 704), (256, 128)):
        for t in (1, 8, 32):
            assert 1 <= c.gemm_fp8_suggest_split(n, k, t) <= max(1, k // 64)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n,k", [(200, 704), (896, 5120), (5120, 1728), (27648, 5120)])
def test_fp8_dequant_is_bit_identical_to_the_host_statement(n, k, dtype):
    from chatts_b200.weights import dequantize_fp8, pack_fp8_mma
    c = ctx()
    q, s = _rand_codes(n, k, seed=7 + n)
    s = s * 300.0                                              # scales around 3e-2: values far from the subnormal range of fp16
    out = torch.full((n + 3, k + 64), float("nan"), device="cuda", dtype=dtype)         # padded rows and leading dimension stay untouched
    c.fp8_dequant(pack_fp8_mma(q), s, k, out[:, :])
    torch.cuda.synchronize()
    want = dequantize_fp8(q, s, dtype)
    assert torch.equal(out[:n, :k], want)
    assert bool(torch.isnan(out[:, k:]).all()) and bool(torch.isnan(out[n:]).all())


# ---------------------------------------------------------------------------------------------------------------- whole model
def _fp8_state_dict(model, sd, dtype):
    """The checkpoint with every decoder projection replaced by the model's own W' = fp32(code) * s, read back from its packed codes and
    split into the checkpoint's q / k / v and gate / up tensors: (in the model dtype, in fp32)."""
    from chatts_b200.weights import unpack_fp8_mma
    H, I, d, nh, nkv = model.H, model.I, model.d, model.nh, model.nkv
    same, f32 = dict(sd), {k: v.float() for k, v in sd.items()}
    for l in range(model.L):
        w = {}
        for kind, (n, k) in (("qkv", (model._n_qkv, H)), ("o", (H, nh * d)), ("gu", (2 * I, H)), ("d", (H, I))):
            qw, sc, _ = model.fp8[kind][l]
            w[kind] = unpack_fp8_mma(qw, n, k).cpu().view(torch.float8_e4m3fn).float() * sc.cpu()[:, None]
        q_, k_, v_ = w["qkv"].split([nh * d, nkv * d, nkv * d])
        gu = w["gu"].view(-1, 2, 64, H)
        parts = {"self_attn.q_proj": q_, "self_attn.k_proj": k_, "self_attn.v_proj": v_, "self_attn.o_proj": w["o"],
                 "mlp.gate_proj": gu[:, 0].reshape(I, H), "mlp.up_proj": gu[:, 1].reshape(I, H), "mlp.down_proj": w["d"]}
        for name, t in parts.items():
            same[f"model.layers.{l}.{name}.weight"], f32[f"model.layers.{l}.{name}.weight"] = t.to(dtype).contiguous(), t.contiguous()
    return same, f32


def _model(dtype, qwen3, seed):
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    cfg = ChatTSConfig.tiny()
    if qwen3:
        cfg.qk_norm, cfg.attention_bias = True, False
    sd = synthetic_state_dict(cfg, seed=seed, device="cpu", dtype=dtype, std=0.05)
    model = ChatTSForCausalLM(cfg, sd, dtype=dtype, max_batch=4, max_seq_len=512, page_size=16)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    return cfg, sd, model, proc


def _series():
    x = np.arange(256)
    ts1 = np.sin(x / 10) * 5.0
    ts1[100:] -= 10.0
    return ts1


def _oracle_embed(cfg, w, enc, dtype, fp32):
    ts_w = {k[len("ts_encoder."):]: v for k, v in w.items() if k.startswith("ts_encoder.")}
    x = enc["timeseries"].to(dtype)
    feats, pc = ote.forward(x.float() if fp32 else x, cfg.ts, ts_w)
    return om.hf_merge(enc["input_ids"], enc["attention_mask"], w["model.embed_tokens.weight"], feats, pc.tolist(), cfg.ts_token_start_index)[0]


@pytest.mark.parametrize("qwen3", [False, True], ids=["qwen2", "qwen3"])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_fp8_model_logits_against_the_oracle_on_the_quantised_weights(dt, qwen3):
    """After quantize_fp8(): the prefill's next-token logits (dequantised weights through cts_gemm) and the first decode step's logits
    (cts_gemm_fp8) against the oracle run on W' in the model dtype and in fp32, through the comparative gate of test_gpu_model; the
    freed 16-bit bytes show in torch.cuda.memory_allocated()."""
    cfg, sd, model, proc = _model(dt, qwen3, seed=1235)
    before = torch.cuda.memory_allocated()
    proj_bytes = sum(w.numel() * w.element_size() for ws in (model.wqkv, model.wo, model.wgu, model.wd) for w in ws)
    model.quantize_fp8()
    after = torch.cuda.memory_allocated()
    kept = sum(qw.numel() + sc.numel() * 4 for kind in ("qkv", "o", "gu", "d") for qw, sc, _ in model.fp8[kind])
    kept += model.fp8["scratch"].numel() * model.fp8["scratch"].element_size()
    record("fp8_model_memory", dtype=str(dt), freed_16bit=proj_bytes, codes_scales_scratch=kept, drop=before - after)
    if model.device.type == "cuda":                            # (the kernel-source runs on the host have no device allocator)
        assert before - after >= proj_bytes - kept
    assert all(w is None for ws in (model.wqkv, model.wo, model.wgu, model.wd) for w in ws)
    enc = proc(text=["Describe <ts><ts/> please, in detail, with numbers and dates: " + "x" * 20], timeseries=[_series()], return_tensors="pt")
    lg = model.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0]
    same, f32 = _fp8_state_dict(model, sd, dt)
    # the prefill runs cts_gemm on the dequantised scratch copy: exactly the 16-bit model whose weights are W' in the model dtype
    from chatts_b200.model import ChatTSForCausalLM
    ref16 = ChatTSForCausalLM(cfg, same, dtype=dt, max_batch=4, max_seq_len=512, page_size=16)
    lg16 = ref16.forward(enc["input_ids"], enc["attention_mask"], enc["timeseries"]).logits[:, 0]
    assert torch.equal(lg, lg16), float((lg.float() - lg16.float()).abs().max())
    del ref16
    refs, states, embs = [], [], []
    for fp32, w in ((False, same), (True, f32)):
        emb = _oracle_embed(cfg, w, enc, dt, fp32)
        st = od.State(cfg.num_hidden_layers)
        refs.append(od.logits(od.forward_hidden(emb, w, cfg.to_dict(), st)[-1:], w))
        states.append(st)
    fixed = 1.57e-2 if dt == torch.bfloat16 else 1.6e-3
    parity_gate("fp8_next_token_logits", lg, refs[0], refs[1], dt, fixed, qwen3=int(qwen3))
    # first decode step: the token the prefill picked, through the FP8 decode GEMM
    tok = int(lg[0].float().argmax())
    dec = _first_step_logits(model, enc)
    drefs = []
    for w, st in ((same, states[0]), (f32, states[1])):
        e = w["model.embed_tokens.weight"][tok][None, :]
        drefs.append(od.logits(od.forward_hidden(e, w, cfg.to_dict(), st), w))
    # the decode GEMM multiplies by W' exactly (fp32 code * scale), the same-dtype oracle by W' rounded to the model dtype: the fixed bound
    # against that oracle gets headroom, the comparative bound against the fp32 oracle is the same as for the prefill
    parity_gate("fp8_first_decode_step_logits", dec, drefs[0][0], drefs[1][0], dt, 2e-2 if dt == torch.bfloat16 else 3e-3, qwen3=int(qwen3))


def _first_step_logits(model, enc):
    ids_cpu, am_cpu, counts, lay = model._prepare_inputs(enc["input_ids"], enc["attention_mask"], enc["timeseries"])
    B = ids_cpu.shape[0]
    pts, held = model._alloc_pages(lay.lens, 4)
    try:
        logits = model._prefill(lay, counts, enc["timeseries"], pts)
        st = model._decode_state(B, 4)
        lens32 = torch.from_numpy(lay.lens.astype(np.int32))
        st.page_table.copy_(torch.from_numpy(pts)); st.positions.copy_(lens32 - 1); st.seq_lens.copy_(lens32); st.step_ptr.zero_()
        model.ctx.greedy_advance(logits, B, st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.page_table, model.page_size)
        model._decode_step(st, sample=False)
        torch.cuda.synchronize()
        return st.full_logits[0].float().cpu().clone()
    finally:
        model.pool.release(held)


def test_fp8_generate_greedy_matches_the_oracle_with_cuda_graphs():
    """Teacher-forced check as test_gpu_model.test_generate_greedy_matches_oracle, decode steps replayed from CUDA graphs: every
    produced token is the oracle's argmax on W' or within bf16 noise of it."""
    dt = torch.bfloat16
    cfg, sd, model, proc = _model(dt, False, seed=1236)
    model.quantize_fp8()
    model.use_cuda_graph = True
    x = np.arange(256)
    enc = proc(text=["A <ts><ts/> and B <ts><ts/> ?", "Only text, no series, but a longer prompt to left-pad the other one"],
               timeseries=[_series(), (x * 0.05)[:100]], padding=True, return_tensors="pt")
    new = 40
    ids = model.generate(**enc, max_new_tokens=new, ignore_eos=True)
    S = enc["input_ids"].shape[1]
    assert ids.shape == (2, S + new) and torch.equal(ids[:, :S], enc["input_ids"])
    assert model._steps[2].graph is not None
    same, _ = _fp8_state_dict(model, sd, dt)
    ts_w = {k[len("ts_encoder."):]: v for k, v in same.items() if k.startswith("ts_encoder.")}
    feats, pc = ote.forward(enc["timeseries"].to(dt), cfg.ts, ts_w)
    embeds = om.hf_merge(enc["input_ids"], enc["attention_mask"], same["model.embed_tokens.weight"], feats, pc.tolist(), cfg.ts_token_start_index)
    worst_gap, exact = 0.0, 0
    for b, e in enumerate(embeds):
        st = od.State(cfg.num_hidden_layers)
        lg = od.logits(od.forward_hidden(e, same, cfg.to_dict(), st)[-1:], same)[0].float()
        for tok in ids[b, S:].tolist():
            worst_gap = max(worst_gap, float((lg.max() - lg[tok]) / lg.abs().max()))
            exact += int(int(lg.argmax()) == tok)
            lg = od.logits(od.forward_hidden(same["model.embed_tokens.weight"][tok][None, :], same, cfg.to_dict(), st), same)[0].float()
    record("fp8_generate_greedy", teacher_forced_exact=exact, teacher_forced_total=2 * new, worst_gap_rel=worst_gap)
    assert worst_gap < 1e-2
    assert exact >= int(0.9 * 2 * new)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="tensor parallelism needs two GPUs")
def test_fp8_tensor_parallel_matches_the_single_gpu_fp8_model():
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29653", os.path.join(ROOT, "tools", "tp_check.py"), "--fp8"], capture_output=True, text=True,
                       timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "fp8=1" in r.stdout
