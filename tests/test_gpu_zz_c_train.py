"""The part of the LoRA fine-tune step (row A9) that was written after the round-1 GPU budget was spent: the attention LSE flag, the attention
backward (HMMA), AdamW + clip, adapter packing and the whole-step tests against oracle/lora.py -- compiled for sm_90a,
orchestration parity-checked on CPU through the double (tools/dryrun_train_gpu_tests.py runs this file's logic on CPU).  The kernels validated earlier are in tests/test_gpu_train_kernels.py.  The zz files
sort last on purpose (a sticky CUDA error here cannot poison validated tests); none of the kernels exercised here spins on a
flag."""
import math

import numpy as np
import pytest
import torch

from tests.cabi_double import TorchDouble
from tests.gpu_util import ctx, record, rel_err

DT = torch.bfloat16
DBL = TorchDouble()


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rn(g, *shape, std=1.0, dtype=DT):
    return (torch.randn(*shape, generator=g) * std).to(dtype)


pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ optimiser + packing
def test_adamw_and_clip_match_torch():
    c = ctx()
    g = _g(1)
    n = 100003
    p0 = torch.randn(n, generator=g)
    par = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([par], lr=3e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    p, m, v = p0.cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    ws, out = torch.zeros(c.grad_norm_ws_floats(), device="cuda"), torch.zeros(2, device="cuda")
    for step in range(1, 4):
        gr = torch.randn(n, generator=g) * 0.01
        par.grad = gr.clone()
        tn = torch.nn.utils.clip_grad_norm_([par], 1.0)
        opt.step()
        gd = gr.cuda()
        c.grad_norm_clip(gd, 1.0, ws, out)
        c.adamw(p, gd, m, v, 3e-3, 0.9, 0.95, 1e-8, 0.1, step, grad_scale=out[1:2])
        torch.cuda.synchronize()
        assert abs(float(out[0]) - float(tn)) < 1e-5 * float(tn)
        assert torch.allclose(p.cpu(), par.detach(), atol=2e-6, rtol=1e-5), step
    c.grad_norm_clip(gd, 0.0, ws, out)
    assert float(out[1]) == 1.0


def test_lora_pack_matches_double():
    from chatts_b200._cabi import PACK_DESC_LONGS
    c = ctx()
    g = _g(2)
    r, K, N, R = 8, 256, 384, 24
    master = torch.randn(3 * r * K + 128 * r * 3, generator=g)
    one, sb = int(np.float32(1.0).view(np.uint32)), int(np.float32(2.0).view(np.uint32))
    offA, offAt, offB, offBt = 0, R * K, 2 * R * K, 2 * R * K + N * R
    desc = [[0, r, K, offA, K, 8, 0, 0, offAt, R, one, 0],                        # A of member 1 -> rows 8..15
            [3 * r * K, 128, r, offB, R, 128, 0, 8, offBt, N, sb, 0],              # B of member 1 -> rows 128..255, cols 8..15
            [3 * r * K + 128 * r, 128, r, offB, R, 0, 1, 16, offBt, N, sb, 0]]     # interleaved "gate" rows, cols 16..23
    assert all(len(d) == PACK_DESC_LONGS for d in desc)
    dt = torch.tensor(desc, dtype=torch.int64).reshape(-1)
    ref = torch.zeros(2 * R * K + 2 * N * R, dtype=DT)
    DBL.lora_pack(master, dt, 3, 128 * r * 8, ref)
    work = torch.zeros_like(ref).cuda()
    c.lora_pack(master.cuda(), dt.cuda(), 3, max(r * K, 128 * r), work)
    torch.cuda.synchronize()
    assert torch.equal(work.cpu(), ref)


# ------------------------------------------------------------------------------------------------ attention: LSE + backward
def _attn_inputs(d, lens, nh=4, nkv=2, dtype=DT):
    T = sum(lens)
    g = _g(T + d)
    q, k, v, do = _rn(g, T, nh * d, dtype=dtype), _rn(g, T, nkv * d, dtype=dtype), _rn(g, T, nkv * d, dtype=dtype), _rn(g, T, nh * d, dtype=dtype)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)
    return T, q, k, v, do, cu


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("lens", [[1], [5, 64, 65], [130, 17, 200, 1], [577]])
def test_prefill_lse_matches_prefill_and_logsumexp(d, lens):
    c = ctx()
    nh, nkv = 4, 2
    T, q, k, v, _, cu = _attn_inputs(d, lens)
    sc = 1.0 / math.sqrt(d)
    a, b = torch.empty(T, nh * d, device="cuda", dtype=DT), torch.empty(T, nh * d, device="cuda", dtype=DT)
    lse = torch.full((T, nh), float("nan"), device="cuda")
    c.attn_prefill(q.cuda(), k.cuda(), v.cuda(), cu.cuda(), len(lens), max(lens), nh, nkv, d, sc, a)
    c.attn_prefill_lse(q.cuda(), k.cuda(), v.cuda(), cu.cuda(), len(lens), max(lens), nh, nkv, d, sc, b, lse)
    torch.cuda.synchronize()
    ro, rl = torch.empty(T, nh * d, dtype=DT), torch.empty(T, nh)
    DBL.attn_prefill_lse(q, k, v, cu, len(lens), max(lens), nh, nkv, d, sc, ro, rl)
    e = float((lse.cpu() - rl).abs().max())
    record("attn_prefill_lse", d=d, lens=str(lens), lse_abs_err=e)
    assert torch.equal(a, b)                                   # same kernel, one extra store
    assert e < 2e-3


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("lens", [[1], [5, 64, 65], [130, 17, 200, 1], [577], [64, 128]])
def test_attention_backward(d, lens):
    c = ctx()
    nh, nkv = 4, 2
    T, q, k, v, do, cu = _attn_inputs(d, lens)
    sc = 1.0 / math.sqrt(d)
    qd, kd, vd, dod, cud = q.cuda(), k.cuda(), v.cuda(), do.cuda(), cu.cuda()
    o, lse = torch.empty(T, nh * d, device="cuda", dtype=DT), torch.empty(T, nh, device="cuda")
    c.attn_prefill_lse(qd, kd, vd, cud, len(lens), max(lens), nh, nkv, d, sc, o, lse)
    dq, dk, dv = (torch.full((T, n_ * d), float("nan"), device="cuda", dtype=DT) for n_ in (nh, nkv, nkv))
    ws = torch.empty(T, nh, device="cuda")
    c.attn_bwd(qd, kd, vd, o, dod, lse, cud, len(lens), max(lens), nh, nkv, d, sc, ws, dq, dk, dv)
    torch.cuda.synchronize()
    rq, rk, rv = torch.empty(T, nh * d, dtype=DT), torch.empty(T, nkv * d, dtype=DT), torch.empty(T, nkv * d, dtype=DT)
    DBL.attn_bwd(q, k, v, None, do, None, cu, len(lens), max(lens), nh, nkv, d, sc, None, rq, rk, rv)
    # a length-1 sequence has dQ = dK = 0 exactly (one key: P = 1, dP = delta); the kernels leave rounding noise of ~1e-7 there, so
    # the denominator gets an absolute floor
    err = lambda a, r: float((a.float().cpu() - r.float()).abs().max() / r.float().abs().max().clamp_min(1e-4))
    eq, ek, ev = err(dq, rq), err(dk, rk), err(dv, rv)
    record("attn_bwd", d=d, lens=str(lens), dq=eq, dk=ek, dv=ev)
    for t_ in (dq, dk, dv):
        assert torch.isfinite(t_.float()).all()
    assert eq < 2e-2 and ek < 2e-2 and ev < 2e-2, (eq, ek, ev)
    # deterministic: no atomics in the attention backward
    dq2, dk2, dv2 = (torch.empty_like(t_) for t_ in (dq, dk, dv))
    c.attn_bwd(qd, kd, vd, o, dod, lse, cud, len(lens), max(lens), nh, nkv, d, sc, ws, dq2, dk2, dv2)
    torch.cuda.synchronize()
    assert torch.equal(dq, dq2) and torch.equal(dk, dk2) and torch.equal(dv, dv2)


def test_attention_backward_gqa_group_of_8_fp16():
    c = ctx()
    d, nh, nkv, lens = 128, 8, 1, [100, 260]
    T, q, k, v, do, cu = _attn_inputs(d, lens, nh, nkv, torch.float16)
    sc = 1.0 / math.sqrt(d)
    qd, kd, vd, dod, cud = q.cuda(), k.cuda(), v.cuda(), do.cuda(), cu.cuda()
    o, lse = torch.empty(T, nh * d, device="cuda", dtype=torch.float16), torch.empty(T, nh, device="cuda")
    c.attn_prefill_lse(qd, kd, vd, cud, 2, max(lens), nh, nkv, d, sc, o, lse)
    dq, dk, dv = (torch.empty(T, n_ * d, device="cuda", dtype=torch.float16) for n_ in (nh, nkv, nkv))
    c.attn_bwd(qd, kd, vd, o, dod, lse, cud, 2, max(lens), nh, nkv, d, sc, torch.empty(T, nh, device="cuda"), dq, dk, dv)
    torch.cuda.synchronize()
    rq, rk, rv = (torch.empty(T, n_ * d, dtype=torch.float16) for n_ in (nh, nkv, nkv))
    DBL.attn_bwd(q, k, v, None, do, None, cu, 2, max(lens), nh, nkv, d, sc, None, rq, rk, rv)
    assert rel_err(dq, rq) < 1e-2 and rel_err(dk, rk) < 1e-2 and rel_err(dv, rv) < 1e-2


# ------------------------------------------------------------------------------------------------ the whole step
def _trainer_case(qwen3, head_dim=64):
    from chatts_b200 import ChatTSConfig, ChatTSProcessor, SimpleTokenizer
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    from tests.test_host_train import RECORDS

    kw = {} if head_dim == 64 else dict(head_dim=128, hidden_size=512, num_attention_heads=4, num_key_value_heads=2,
                                        ts=dict(patch_size=16, num_layers=3, hidden_size=512, num_features=2, max_sequence_length=512,
                                                use_position_embedding=True, use_position_idx=False, embedding_dim=16))
    cfg = ChatTSConfig.tiny(**kw)
    if qwen3:
        cfg.qk_norm, cfg.attention_bias = True, False
    sd = synthetic_state_dict(cfg, seed=1234, device="cpu", dtype=DT, std=0.05)
    model = ChatTSForCausalLM(cfg, sd, dtype=DT, max_batch=8, max_seq_len=512, page_size=16)
    proc = ChatTSProcessor(SimpleTokenizer(cfg.ts_token_start_index, cfg.pad_token_id, cfg.eos_token_id), cfg)
    return cfg, sd, model, proc, RECORDS


@pytest.mark.parametrize("qwen3,head_dim", [(False, 64), (True, 64), (True, 128)])
def test_train_step_matches_oracle(qwen3, head_dim):
    from chatts_b200.train import LoraTrainer, encode_records
    from oracle import lora as ol
    from tests.test_host_train import _oracle_inputs

    cfg, sd, model, proc, records = _trainer_case(qwen3, head_dim)
    r, alpha = 8, 16
    tr = LoraTrainer(model, r=r, lora_alpha=alpha, seed=3, init_b_std=0.05, max_grad_norm=0.0)
    ad = ol.init_adapters(cfg.to_dict(), r, seed=3, b_std=0.05)
    batch = encode_records(proc, records, eos_token_id=cfg.eos_token_id)
    tr.zero_grad()
    bt = tr.forward_backward(**batch)
    torch.cuda.synchronize()
    embeds, labels = _oracle_inputs(cfg, sd, batch)
    w = {k: v for k, v in sd.items() if not k.startswith("ts_encoder.")}
    loss, g = ol.grads(embeds, labels, w, ad, alpha / r, cfg.to_dict())
    got_loss = float(tr.loss_out[0])
    got = tr.grads()
    worst = max(rel_err(got[n], ref) for n, ref in g.items())
    flat_ref = torch.cat([g[n].reshape(-1) for n in tr.index])
    cos = float(torch.nn.functional.cosine_similarity(tr.g.cpu(), flat_ref, dim=0))
    record("train_step_vs_oracle", qwen3=qwen3, head_dim=head_dim, loss=got_loss, loss_ref=loss, worst_grad_rel=worst, cosine=cos,
           tokens=bt.T, labels=bt.n_counted)
    assert abs(got_loss - loss) < 2e-2 * abs(loss), (got_loss, loss)
    assert worst < 8e-2 and cos > 0.998, (worst, cos)


def test_training_reduces_loss_and_merge_roundtrip(tmp_path):
    from chatts_b200.train import LoraTrainer, encode_records

    cfg, sd, model, proc, records = _trainer_case(True)
    batch = encode_records(proc, records, eos_token_id=cfg.eos_token_id)
    tr = LoraTrainer(model, r=16, lora_alpha=32, seed=0, lr=5e-3, max_grad_norm=1.0)
    l0 = float(tr.eval_loss(batch)[0])
    losses = [float(tr.train_step(batch)[0]) for _ in range(4)]
    record("train_loss_curve", l0=l0, losses=str(losses), grad_norm=float(tr.norm_out[0]))
    assert abs(losses[0] - l0) < 1e-3 * l0 and losses[-1] < losses[0] - 0.05, losses
    lt = float(tr.eval_loss(batch)[0])
    tr.save_adapter(str(tmp_path / "ad"))
    assert model.merge_lora(str(tmp_path / "ad")) == cfg.num_hidden_layers * 7
    lm = float(LoraTrainer(model, r=16, lora_alpha=32, seed=0).eval_loss(batch)[0])
    assert abs(lm - lt) < 3e-2 * lt, (lm, lt)


def _id_batch(cfg, samples, seed, n_series=2, series_len=256, prefix=20, prompt=24, answer=40):
    """Token-id level records (BASELINE cfg5 shape, scaled down in length): prefix ids + <ts><ts/> per series, prompt, answer."""
    from chatts_b200.processor import sp_encoding
    rng = np.random.default_rng(seed)
    hi = min(cfg.vocab_size, cfg.ts_token_start_index) - 10          # stay clear of <ts>, <ts/>, eos, pad
    ids, lab, series = [], [], []
    for b in range(samples):
        row = []
        for k in range(n_series):
            row += rng.integers(0, hi, prefix).tolist() + [cfg.ts_token_start_index, cfg.ts_token_start_index + 1]
            t = np.arange(series_len - 16 * ((b + k) % 3))                      # ragged lengths: 256 / 240 / 224 points
            series.append(sp_encoding(np.sin(t / (5.0 + k)) * (1 + b) + 0.01 * t)[0])
        row += rng.integers(0, hi, prompt).tolist()
        ans = rng.integers(0, hi, answer).tolist()
        ids.append(row + ans)
        lab.append([-100] * len(row) + ans)
    L = max(e.shape[0] for e in series)
    ts = np.zeros((len(series), L, 1))
    for i, e in enumerate(series):
        ts[i, : e.shape[0]] = e
    ids = torch.tensor(ids, dtype=torch.long)
    return {"input_ids": ids, "attention_mask": torch.ones_like(ids), "labels": torch.tensor(lab, dtype=torch.long),
            "timeseries": torch.from_numpy(ts).to(torch.float32)}


@pytest.mark.parametrize("full_dims", [False, True])
def test_gradient_is_the_directional_derivative_of_the_loss(full_dims):
    """Size-independent property of the whole backward (no oracle needed, so it also runs at the ChatTS-8B layer shape of
    BASELINE config 5): along D = grad/|grad| in adapter space, (L(p + eD) - L(p - eD)) / 2e == <grad L, D> = |grad|.  Also: the
    gradient of a batch is the sum of its micro-batches' gradients (token-mean over the union), and every adapter tensor
    receives a finite, non-zero gradient."""
    from chatts_b200 import ChatTSConfig
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.train import LoraTrainer

    if full_dims:
        cfg = ChatTSConfig.chatts_8b()
        cfg.num_hidden_layers = 2                                  # 8B layer shapes (H 4096, I 12288, 32/8 heads x 128, V 151936), 2 layers
        model = ChatTSForCausalLM.from_synthetic(cfg, seed=7, max_batch=1, max_seq_len=512, page_size=64, use_cuda_graph=False)
        samples = 6
    else:
        cfg = ChatTSConfig.tiny(qk_norm=True, attention_bias=False)
        from chatts_b200.weights import synthetic_state_dict
        sd = synthetic_state_dict(cfg, seed=7, device="cpu", dtype=DT, std=0.05)
        model = ChatTSForCausalLM(cfg, sd, dtype=DT, max_batch=1, max_seq_len=512, page_size=16, use_cuda_graph=False)
        samples = 4
    tr = LoraTrainer(model, r=16, lora_alpha=32, seed=2, init_b_std=0.02, max_grad_norm=0.0)
    batch = _id_batch(cfg, samples, seed=5)
    tr.zero_grad()
    tr.forward_backward(**batch)
    g = tr.g.clone()
    assert torch.isfinite(g).all()
    for name in tr.index:
        assert float(tr.grad(name).abs().max()) > 0, name
    # micro-batches: same gradient as the whole batch when normalised by the same label count
    total = LoraTrainer.count_labels(batch)
    half = samples // 2
    n_ser = 2
    parts = [{k: (v[:half] if k != "timeseries" else v[: half * n_ser]) for k, v in batch.items()},
             {k: (v[half:] if k != "timeseries" else v[half * n_ser:]) for k, v in batch.items()}]
    tr.zero_grad()
    for p in parts:
        tr.forward_backward(**p, denominator=total, accumulate_loss=True)
    e_acc = rel_err(tr.g, g)
    # directional derivative along a random unit direction, step sized for a loss change well above bf16 noise
    # along the gradient itself (a random direction in a 10^5..10^7-dimensional space has a slope too small to see through
    # the bf16 noise of the loss): slope = ||g||, step sized for a predicted loss change of 0.03 per side
    D = g / g.norm()
    slope = float((g * D).sum())
    p0 = tr.p.clone()
    eps = 0.03 / max(abs(slope), 1e-6)
    losses = []
    for sgn in (+1.0, -1.0):
        tr.p.copy_(p0 + sgn * eps * D)
        tr.pack()
        losses.append(float(tr.eval_loss(batch)[0]))
    tr.p.copy_(p0)
    tr.pack()
    fd = (losses[0] - losses[1]) / (2 * eps)
    record("train_directional_derivative", full_dims=full_dims, slope=slope, finite_difference=fd, eps=eps, accumulation_rel_err=e_acc,
           loss_plus=losses[0], loss_minus=losses[1])
    assert e_acc < 3e-2, e_acc
    assert abs(fd - slope) < 0.15 * abs(slope) + 1e-4, (fd, slope)


@pytest.mark.parametrize("t,m,r,il", [(37, 256, 8, 0), (5000, 704, 16, 0), (300, 128, 16, 1), (300, 128, 16, 2), (9000, 64, 16, 0),
                                      (100, 4096, 16, 0), (513, 200, 24, 0)])
def test_lora_wgrad_tensor_core_variant(t, m, r, il, monkeypatch):
    """lora_wgrad_mma.cu (CTS_WGRAD_MMA=1): ldmatrix.trans + mma.sync version of the weight gradient against the restatement
    and against the validated FMA kernel."""
    c = ctx()
    g = _g(t + m + r)
    ld = 2 * m if il else m + 64
    col0 = 0 if il else 32
    p, q = _rn(g, t, ld, std=0.5), _rn(g, t, 3 * r + 8, std=0.5)
    for so_m, so_r, name in ((r, 1, "dB"), (1, m, "dA")):
        base = torch.randn(m * r, generator=g)
        ref = base.clone()
        DBL.lora_wgrad(p, col0, il, m, q, r, r, t, 0.5, ref, so_m, so_r)
        got = {}
        for flag in ("0", "1"):
            monkeypatch.setenv("CTS_WGRAD_MMA", flag)
            out = base.clone().cuda()
            c.lora_wgrad(p.cuda(), col0, il, m, q.cuda(), r, r, t, 0.5, out, so_m, so_r)
            torch.cuda.synchronize()
            got[flag] = out
        e, cross = rel_err(got["1"], ref), rel_err(got["1"], got["0"])
        record("lora_wgrad_mma", t=t, m=m, r=r, il=il, layout=name, err=e, vs_fma=cross)
        assert e < 2e-4 and cross < 2e-4, (name, e, cross)
