"""CPU: kernel SOURCE executed without a GPU.  tests/cuda_on_cpu compiles a few files of chatts_b200/csrc with g++ against a small
"CUDA on CPU" shim (CUDA threads = fibers, __syncthreads / shuffles / atomics provided, blocks one after the other) and the
product's own ctypes wrappers drive them on host memory:

  * tools/shim_gpu_tests.py runs the GPU test cases of the sampling kernel, AdamW + clip, adapter packing, the attention backward
    (attention_bwd.cu: wmma through a fragment shim) and -- in a HYBRID context where the wgmma GEMMs and the attention forward are
    answered by the torch double -- the whole LoRA training step against the oracle, plus, as
    calibration of the shim itself, the elementwise / cross-entropy / weight-gradient tests that pass on the GPU
    (the CPU suite runs the --quick subset; the full selection is 56 cases in about 4 minutes);
  * the low-latency all-reduce (allreduce_ll.cu) runs with its ranks as PROCESSES sharing the symmetric regions: real concurrency
    between ranks, torn 16-byte units, consecutive calls without any barrier in between.

Only kernels without tensor cores / TMA / clusters can run this way.  Not a memory-model check (x86 is stronger than PTX)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_pending_and_validated_kernels_pass_their_gpu_tests_on_the_shim():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), "--quick"], capture_output=True, text=True, timeout=850,
                       cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    import re
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    # sampling, training (incl. one whole step), validated elementwise kernels, cluster-fused decode GEMMs, validated GEMMs, wgmma
    # attention backward, prefill attention, W4A16 mma GEMM
    assert len(passed) == 8 and min(passed) >= 1 and sum(passed) >= 118 and "failed" not in r.stdout, tail
    native = r.stdout.split("entry points running from kernel source:")[1].split("\n")[0].split()
    assert {"sample_advance", "attn_bwd", "adamw", "grad_norm_clip", "lora_pack", "lora_wgrad", "ce_loss_grad", "rmsnorm_bwd", "swiglu_bwd",
            "qkv_rope_bwd", "gemm", "gemm_decode_fused", "attn_prefill", "attn_prefill_lse", "attn_decode", "decoder_step", "reduce_residual_rmsnorm",
            "gemm_w4", "gemm_w4_mma"} <= set(native), native


def _expected(parts, split, resid, dt):
    acc = torch.zeros_like(parts[0][0])
    for p in parts:
        loc = p[0].clone()
        for s in range(1, split):
            loc = loc + p[s]
        acc = acc + loc
    return (resid.float() + acc.to(dt).float()).to(dt)


@pytest.mark.parametrize("W,T,h,split,dt", [(2, 3, 256, 2, torch.bfloat16), (4, 2, 512, 1, torch.float16), (2, 1, 128, 3, torch.bfloat16),
                                            (2, 2, 1024, 2, torch.bfloat16), (4, 3, 1024, 1, torch.bfloat16)])
def test_ll_allreduce_kernel_with_ranks_as_processes(W, T, h, split, dt):
    from tests.cuda_on_cpu.shim import shim_context
    c = shim_context()
    # h / W >= 256 columns: the kernel splits every owner's chunk over several CTAs per token, which wait for each other's statistics
    # (not a cluster) -> the shim runs the whole grid concurrently
    c.lib.shim_concurrent_grid(1 if h // W >= 256 else 0)
    tmax, calls = 4, [0, 1, 0, 0, 1]                         # buffer set per call (one repeated set: allowed, see the protocol test)
    nbytes = c.peer_ll_region_bytes(W, tmax, h)
    g = torch.Generator().manual_seed(W * 100 + h)
    share = lambda t: t.share_memory_()
    regions = [[share(torch.zeros((nbytes + 3) // 4, dtype=torch.int32)) for _ in range(W)] for _ in range(2)]
    ptrs = [share(torch.tensor([r.data_ptr() for r in regions[b]], dtype=torch.int64)) for b in range(2)]
    state = [share(torch.zeros(2, dtype=torch.int32)) for _ in range(W)]
    h0 = (torch.randn(T, h, generator=g) * 0.5).to(dt)
    nw = (1.0 + 0.1 * torch.randn(h, generator=g)).to(dt)
    parts = [[share((torch.randn(split, T, h, generator=g) * 0.3)) for _ in range(W)] for _ in calls]
    # every rank keeps its own h (updated in place by every call) and logs h / norm_out of every call for the parent to check
    resid = [share(h0.clone()) for _ in range(W)]
    xn = [share(torch.zeros(T, h, dtype=dt)) for _ in range(W)]
    log_h = [share(torch.zeros(len(calls), T, h, dtype=dt)) for _ in range(W)]
    log_n = [share(torch.zeros(len(calls), T, h, dtype=dt)) for _ in range(W)]
    pids = []
    for r in range(W):
        pid = os.fork()
        if pid == 0:                                         # rank r: all calls back to back, no synchronisation but the protocol's
            try:
                import signal
                signal.alarm(120)
                for n, which in enumerate(calls):
                    c.peer_allreduce_ll(parts[n][r], split, ptrs[which], nbytes, state[r], r, W, tmax, resid[r], resid[r], nw, 1e-6, xn[r], T)
                    log_h[r][n].copy_(resid[r])
                    log_n[r][n].copy_(xn[r])
                os._exit(0)
            except BaseException:
                import traceback
                traceback.print_exc()
                os._exit(1)
        pids.append(pid)
    codes = [os.waitpid(p, 0)[1] for p in pids]
    c.lib.shim_concurrent_grid(0)
    assert codes == [0] * W, codes
    cur = h0.clone()
    for n in range(len(calls)):
        cur = _expected(parts[n], split, cur, dt)
        x = cur.float()
        want = nw.float() * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)).to(dt).float()
        for r in range(W):
            assert torch.equal(log_h[r][n], cur), f"call {n}: h of rank {r} differs from the rank-ordered sum"
            assert torch.equal(log_n[r][n], log_n[0][n]), f"call {n}: norm_out differs between ranks 0 and {r}"
        assert float((log_n[0][n].float() - want).abs().max() / want.abs().max()) < 1.2e-2
    assert [int(s[0]) for s in state] == [len(calls)] * W    # the epoch advanced once per call on every rank


# ---------------------------------------------------------------------------------------------------------------------------
# gemm_decode_fused.cu through the shim: the TMA -> wgmma mainloop is replaced (inside the kernel, #ifdef CTS_HOST_SHIM) by
# the fp32 partial tile it produces; from the cluster barrier on the kernel runs AS WRITTEN: the K splits of a tile as the CTAs of
# one cluster (threads here), the distributed-shared-memory reduction in split order, the three tails, the fused RMSNorm operand,
# and the in-kernel all-reduce with ranks as processes.  Reference: the torch double's statement of the two-launch path.  The
# partial sums are accumulated in a different order than torch's matmul, so outputs may differ by one ulp of the model dtype.
# ---------------------------------------------------------------------------------------------------------------------------
DT = torch.bfloat16


def _rn(g, *shape, std=1.0):
    return (torch.randn(*shape, generator=g) * std).to(DT)


def _close(a, r, ulps=2.0):
    a, r = a.float(), r.float()
    return float((a - r).abs().max()) <= ulps * 2 ** -8 * float(r.abs().max()) + 1e-6


@pytest.fixture(scope="module")
def shim_ctx():
    from tests.cuda_on_cpu.shim import shim_context
    return shim_context()


@pytest.mark.parametrize("t,n,k,s", [(1, 256, 512, 2), (8, 640, 1024, 7), (32, 384, 704, 4), (17, 200, 640, 3)])
def test_fused_residual_tail_and_tile_statistics(shim_ctx, t, n, k, s):
    from tests.cabi_double import TorchDouble
    g = torch.Generator().manual_seed(t + n + k)
    x, w, h0 = _rn(g, t, k, std=0.5), _rn(g, n, k, std=0.05), _rn(g, t, n, std=0.5)
    tiles = (n + 127) // 128
    out, ssq = h0.clone(), torch.full((t, tiles), float("nan"))
    shim_ctx.gemm_decode_fused(x, w, 0, s, t, h=out, ssq_out=ssq)
    ref, rssq = h0.clone(), torch.zeros(t, tiles)
    TorchDouble().gemm_decode_fused(x, w, 0, s, t, h=ref, ssq_out=rssq)
    assert _close(out, ref)
    pad = torch.zeros(t, tiles * 128)
    pad[:, :n] = out.float() ** 2
    assert torch.allclose(ssq, pad.view(t, tiles, 128).sum(-1), rtol=1e-5, atol=1e-6)      # the statistic of what was actually written


@pytest.mark.parametrize("t,inter,k,s", [(1, 128, 256, 1), (8, 704, 512, 2), (32, 192, 640, 5)])
def test_fused_swiglu_tail(shim_ctx, t, inter, k, s):
    from tests.cabi_double import TorchDouble
    g = torch.Generator().manual_seed(t + inter)
    x, w = _rn(g, t, k, std=0.5), _rn(g, 2 * inter, k, std=0.05)
    out, ref = torch.full((t, inter), float("nan"), dtype=DT), torch.empty(t, inter, dtype=DT)
    shim_ctx.gemm_decode_fused(x, w, 1, s, t, act=out)
    TorchDouble().gemm_decode_fused(x, w, 1, s, t, act=ref)
    assert _close(out, ref, ulps=3.0)


@pytest.mark.parametrize("d,nh,nkv,qk,bias", [(128, 4, 2, False, True), (128, 2, 1, True, False), (64, 4, 2, False, True), (64, 5, 1, True, False)])
@pytest.mark.parametrize("t,s", [(1, 5), (9, 3)])
def test_fused_qkv_rope_tail(shim_ctx, d, nh, nkv, qk, bias, t, s):
    from tests.cabi_double import TorchDouble
    g = torch.Generator().manual_seed(d + nh + t)
    H, page, pages = 512, 16, 4
    N = (nh + 2 * nkv) * d
    x, w = _rn(g, t, H, std=0.5), _rn(g, N, H, std=0.05)
    b = _rn(g, N, std=0.2) if bias else None
    qn = (torch.rand(d, generator=g) + 0.5).to(DT) if qk else None
    kn = (torch.rand(d, generator=g) + 0.5).to(DT) if qk else None
    pos = torch.randint(0, 100, (t,), generator=g).to(torch.int32)
    ang = torch.rand(128, d // 2, generator=g) * 6.28
    cos, sin = ang.cos().to(DT), ang.sin().to(DT)
    slot = torch.randperm(pages * page, generator=g)[:t].to(torch.int32)
    if t > 2:
        slot[1] = -1
    outs = []
    for c in (shim_ctx, TorchDouble()):
        q = torch.full((t, nh * d), float("nan"), dtype=DT)
        kc, vc = torch.zeros(pages, nkv, page, d, dtype=DT), torch.zeros(pages, nkv, page, d, dtype=DT)
        c.gemm_decode_fused(x, w, 2, s, t, bias=b, positions=pos, cos=cos, sin=sin, slot_map=slot, q_out=q, k_cache=kc, v_cache=vc, q_norm=qn,
                            k_norm=kn, eps=1e-6, nh=nh, nkv=nkv, head_dim=d, page_size=page)
        outs.append((q, kc, vc))
    for a, r in zip(outs[0], outs[1]):
        assert _close(a, r, ulps=4.0)
    assert bool((outs[0][1] != 0).any()) and bool((outs[0][2] != 0).any())               # the KV pages were written


def test_fused_rmsnorm_operand(shim_ctx):
    """NORM_IN: the token operand is RMSNorm(h) built from the per-tile sums of squares of the previous RESIDUAL call."""
    from tests.cabi_double import TorchDouble
    g = torch.Generator().manual_seed(5)
    t, H, inter = 6, 256, 192
    h = _rn(g, t, H, std=0.7)
    nw = (1.0 + 0.1 * torch.randn(H, generator=g)).to(DT)
    w = _rn(g, 2 * inter, H, std=0.05)
    ssq = (h.float() ** 2).view(t, H // 128, 128).sum(-1)
    out, ref = torch.empty(t, inter, dtype=DT), torch.empty(t, inter, dtype=DT)
    shim_ctx.gemm_decode_fused(None, w, 1, 2, t, act=out, norm_h=h, norm_w=nw, ssq_in=ssq, norm_eps=1e-6)
    TorchDouble().gemm_decode_fused(None, w, 1, 2, t, act=ref, norm_h=h, norm_w=nw, ssq_in=ssq, norm_eps=1e-6)
    assert _close(out, ref, ulps=3.0)


@pytest.mark.parametrize("W,T,N,Kr,S", [(2, 3, 256, 128, 1), (2, 7, 512, 320, 2), (4, 5, 512, 256, 3)])
def test_fused_gemm_allreduce_tail_with_ranks_as_processes(shim_ctx, W, T, N, Kr, S):
    """The tensor-parallel tail of CTS_FUSED_RESIDUAL: every rank's cluster scatters its (tile, token) partial to the tile's owner, the
    owner adds in rank order + residual and broadcasts h and the tile statistic.  Ranks = processes sharing the regions, the CTAs of
    a cluster = threads, CUDA threads = fibers; three calls back to back over alternating buffer sets."""
    c = shim_ctx
    tmax = 8
    nbytes = tmax * N * 12 + tmax * (N // 128) * 8 + 64
    g = torch.Generator().manual_seed(W * 10 + T)
    share = lambda x: x.share_memory_()
    regions = [[share(torch.zeros((nbytes + 3) // 4, dtype=torch.int32)) for _ in range(W)] for _ in range(2)]
    ptrs = [share(torch.tensor([r.data_ptr() for r in regions[b]], dtype=torch.int64)) for b in range(2)]
    state = [share(torch.zeros(2, dtype=torch.int32)) for _ in range(W)]
    calls = [0, 1, 0]
    h0 = _rn(g, T, N, std=0.5)
    xs = [[share(_rn(g, T, Kr, std=0.5)) for _ in range(W)] for _ in calls]
    ws = [[share(_rn(g, N, Kr, std=0.05)) for _ in range(W)] for _ in calls]
    hs = [share(h0.clone()) for _ in range(W)]
    ssq = [share(torch.zeros(T, N // 128)) for _ in range(W)]
    log_h = [share(torch.zeros(len(calls), T, N, dtype=DT)) for _ in range(W)]
    log_s = [share(torch.zeros(len(calls), T, N // 128)) for _ in range(W)]
    pids = []
    for r in range(W):
        pid = os.fork()
        if pid == 0:
            try:
                import signal
                signal.alarm(150)
                for n, which in enumerate(calls):
                    c.gemm_decode_fused(xs[n][r], ws[n][r], 0, S, T, h=hs[r], ssq_out=ssq[r], peer=(ptrs[which], nbytes, state[r], r, W, tmax))
                    log_h[r][n].copy_(hs[r])
                    log_s[r][n].copy_(ssq[r])
                os._exit(0)
            except BaseException:
                import traceback
                traceback.print_exc()
                os._exit(1)
        pids.append(pid)
    codes = [os.waitpid(p, 0)[1] for p in pids]
    assert codes == [0] * W, codes
    cur = h0.clone()
    for n in range(len(calls)):
        acc = sum(xs[n][r].float() @ ws[n][r].float().t() for r in range(W))
        cur_ref = (cur.float() + acc.to(DT).float()).to(DT)
        for r in range(W):
            assert torch.equal(log_h[r][n], log_h[0][n]) and torch.equal(log_s[r][n], log_s[0][n]), f"call {n}: rank {r} differs from rank 0"
        assert _close(log_h[0][n], cur_ref, ulps=3.0), f"call {n}"
        assert torch.allclose(log_s[0][n], (log_h[0][n].float() ** 2).view(T, N // 128, 128).sum(-1), rtol=1e-5)
        cur = log_h[0][n].clone()                            # follow the kernel's own h (an ulp may differ from the reference chain)
    assert [int(s_[0]) for s_ in state] == [len(calls)] * W


# the all-reduce-inside-the-GEMM variant is an opt-in path: it runs here only with
# CTS_SLOW_TESTS=1, to keep the default CPU suite within a few minutes on a busy machine
_TP_VARIANTS = ["CTS_PEER_LL=1"] + (["CTS_PEER_LL=1 CTS_DECODE_FUSED=2"] if os.environ.get("CTS_SLOW_TESTS") == "1" else [])


@pytest.mark.parametrize("variant", _TP_VARIANTS)
def test_tensor_parallel_model_with_ranks_as_processes(variant):
    """tools/shim_tp_check.py: the tensor-parallel MODEL (2 ranks = 2 processes under torchrun, gloo for the host-side collectives, the
    symmetric buffers as shared memory behind cts_ipc_*), every kernel from source -- with the low-latency all-reduce kernel, and with the
    all-reduce inside the decode GEMMs (5 launches per layer).  Logits against the single-rank model, greedy agreement, identical tokens
    on both ranks."""
    import socket
    env = dict(os.environ, TP_CHECK_NEW="8")
    env.update(kv.split("=") for kv in variant.split())
    with socket.socket() as sk:                              # a port that is free right now
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tools", "shim_tp_check.py")], capture_output=True, text=True, timeout=600,
                       cwd=ROOT, env=env)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert "identical tokens on all ranks: True" in out and "greedy agreement [8, 8]/8" in out, out[-2000:]


@pytest.mark.skipif(os.environ.get("CTS_SLOW_TESTS") != "1", reason="the guard of bench.py's opt-in --probe (opt-in decode variants, off by default); CTS_SLOW_TESTS=1 runs it")
def test_numeric_guard_of_the_decode_variant_probe_runs_from_source():
    """tools/probe_decode_variant.py (the child bench.py runs before it adopts fusion level 2): default path and variant on the same weights,
    teacher-forced, logits compared at every step -- executed here through the shim with a toy configuration."""
    code = r'''
import sys
sys.path.insert(0, "tools")
import shim_gpu_tests                                    # host patches + shim context
import torch
import chatts_b200.model as mm
from chatts_b200 import ChatTSConfig
import probe_decode_variant as P
fs = mm.ChatTSForCausalLM.from_synthetic.__func__
mm.ChatTSForCausalLM.from_synthetic = classmethod(lambda cls, config=None, seed=1234, device="cpu", dtype=torch.bfloat16, gen_device=None, **kw: fs(cls, config, seed, "cpu", dtype, "cpu", **kw))
c = ChatTSConfig.chatts_14b()
c.hidden_size, c.intermediate_size, c.num_attention_heads, c.num_key_value_heads, c.head_dim = 512, 1024, 4, 2, 128
c.ts["hidden_size"] = 512                                  # the TS encoder projects into the decoder width
import json
print(json.dumps(P.compare(2, [2], 2, 2, cfg=c)))
'''
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    d = json.loads([ln for ln in r.stdout.split("\n") if ln.startswith("{")][-1])
    assert d["finite"] and d["steps"] == 3 and d["max_rel"] <= 1e-2, d
