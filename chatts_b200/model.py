"""ChatTSForCausalLM on H100: TS encoder -> merge at ``<ts>`` -> Qwen2 decoder -> lm_head, behind the
``generate()`` surface the reference's callers use (README.md:88-103, demo/demo_hf.ipynb cells 3-5,
chatts/utils/inference_tsmllm_deepspeed.py:89-106).

Replaces, for this path only: the checkpoint's remote-code ``Qwen2TSForCausalLM`` (HF surface) and
``chatts.vllm.chatts_vllm.Qwen2TSForCausalLM`` (chatts_vllm.py:452-625).  All arithmetic runs in the sm_90a
kernels of libchatts_b200.so; torch provides device memory, streams, CUDA-graph capture and
torch.distributed.  There is no CPU or eager-torch fallback: constructing the model without an H100 raises.

Decode is a single CUDA graph per batch size: embedding gather -> [split-K wgmma GEMM -> fused
reduce(+bias+RoPE+KV write | +residual+RMSNorm | SwiGLU)] x layers -> paged flash-decode -> lm_head -> argmax
-> device-side advance (next id, position, KV slot), so a step replays with no host round trip.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _cabi, layout, prefix_cache
from . import beam as beammod
from . import logprobs as lpmod
from .token_pipeline import TokenPipeline, generate_processors, resolve_generate
from .trace import span
from ._cabi import EPI_NONE, EPI_PARTIAL_F32, EPI_RESIDUAL, EPI_SWIGLU_IL
from .config import ChatTSConfig
from .ts_encoder import TimeSeriesEmbedding
from .weights import load_checkpoint, shard_tensor, synthetic_state_dict


@dataclass
class CausalLMOutput:
    logits: torch.Tensor


def rope_tables(cfg, n_pos, dtype, device):
    """cos/sin exactly as transformers computes them (modeling_qwen2.py:88-113): fp32 inv_freq, fp32 outer
    product, fp32 cos/sin, THEN cast to the model dtype.  Computed once on the host at load time (not on the
    hot path) so the table is bit-identical to the reference's; [n_pos, head_dim/2] because emb = cat(f, f)."""
    d = cfg.head_dim
    inv_freq = 1.0 / (float(cfg.rope_theta) ** (torch.arange(0, d, 2, dtype=torch.int64).to(torch.float32) / d))
    pos = torch.arange(n_pos, dtype=torch.float32)
    freqs = (inv_freq[:, None] @ pos[None, :]).transpose(0, 1)
    return freqs.cos().to(dtype).to(device).contiguous(), freqs.sin().to(dtype).to(device).contiguous()


class PagePool:
    """Free-list allocator over the pages of the KV cache ([num_pages, nkv, page_size, d] per layer and K/V)."""

    def __init__(self, num_pages):
        self.free = list(range(num_pages - 1, -1, -1))
        self.num_pages = num_pages

    def alloc(self, n):
        if n > len(self.free):
            raise RuntimeError(f"KV cache exhausted: need {n} pages, {len(self.free)} free of {self.num_pages}")
        return [self.free.pop() for _ in range(n)]

    def release(self, pages):
        self.free.extend(reversed(pages))

    def available(self):
        return len(self.free)


def _check_quantization(quantization):
    if quantization not in (None, "fp8"):
        raise ValueError(f"quantization={quantization!r}: supported are None (the checkpoint's 16-bit weights) and 'fp8'")


class _Step:
    """Static buffers of one decode configuration (batch size) + its captured CUDA graphs."""
    pass


class ChatTSForCausalLM:
    def __init__(self, config, state_dict, device="cuda", dtype=torch.bfloat16, tp_rank=0, tp_size=1,
                 max_batch=32, max_seq_len=2048, page_size=64, use_cuda_graph=True, comm=None,
                 use_peer_allreduce=True, graph_with_tp=True, use_chain=None, use_native_step=None, use_fused_decode=None, use_peer_ll=None,
                 enable_prefix_caching=False):
        if enable_prefix_caching and tp_size > 1:
            raise ValueError("enable_prefix_caching is single-GPU only (tensor_parallel_size must be 1)")
        if not torch.cuda.is_available():
            raise _cabi.CtsError("chatts_b200 needs an H100 (sm_90a) GPU; there is no CPU fallback")
        self.config, self.dtype = config, dtype
        self.device = torch.device(device if str(device) != "cuda" else f"cuda:{torch.cuda.current_device()}")
        self.tp_rank, self.tp_size, self.comm = tp_rank, tp_size, comm
        self.ctx = _cabi.get_context(self.device)
        cfg = config
        assert cfg.num_key_value_heads % tp_size == 0 and cfg.num_attention_heads % tp_size == 0
        self.nh, self.nkv, self.d = cfg.num_attention_heads // tp_size, cfg.num_key_value_heads // tp_size, cfg.head_dim
        self.H, self.I = cfg.hidden_size, cfg.intermediate_size // tp_size
        self.V = cfg.vocab_size // tp_size if tp_size > 1 else cfg.vocab_size
        self.L = cfg.num_hidden_layers
        self.eps = float(cfg.rms_norm_eps)
        self.page_size, self.max_batch, self.max_seq_len = page_size, max_batch, max_seq_len
        self.max_pages = (max_seq_len + page_size - 1) // page_size
        self.use_cuda_graph = use_cuda_graph
        self.graph_with_tp = graph_with_tp
        import os as _os
        self.use_chain = bool(int(_os.environ.get("CTS_DECODE_CHAIN", "0"))) if use_chain is None else bool(use_chain)
        # the whole decode step enqueued by one C call (cts_decoder_step) instead of ~440 ctypes calls: identical launches; off by
        # default (CTS_NATIVE_STEP=1 / use_native_step=True)
        self.use_native_step = bool(int(_os.environ.get("CTS_NATIVE_STEP", "0"))) if use_native_step is None else bool(use_native_step)
        # decode GEMMs with the split-K reduction and the projection tail fused in through a thread-block cluster
        # (csrc/gemm_decode_fused.cu: 9 -> 7 dependent stages per layer); off by default
        #   1: projections fused with their tails, plain RMSNorm launches between them (7 stages, bit-identical to the default path)
        #   2: the RMSNorms too -- the residual projections emit per-tile sums of squares, the next projection builds its normalised
        #      token operand itself (5 stages; single GPU only)
        self.use_fused_decode = int(_os.environ.get("CTS_DECODE_FUSED", "0")) if use_fused_decode is None else int(use_fused_decode)
        # tensor parallelism: low-latency two-shot all-reduce (cts_peer_allreduce_ll) instead of the one-shot push kernel
        # (the default: same logits, same tokens on every rank; CTS_PEER_LL=0 selects the one-shot kernel)
        self.use_peer_ll = (_os.environ.get("CTS_PEER_LL", "1") == "1") if use_peer_ll is None else bool(use_peer_ll)
        # row-parallel exchange of prefill-sized steps: "rs_ag" (default: fp32 reduce-scatter + 16-bit all-gather of the result), "fp32"
        # (one fp32 all-reduce, rounds 1-2), "16bit" (all-reduce in the model dtype: vLLM's semantics, fastest, re-rounds the running sum)
        self.tp_prefill_exchange = _os.environ.get("CTS_TP_PREFILL_EXCHANGE", "rs_ag")
        self._nccl = False
        if tp_size > 1 and torch.distributed.is_available() and torch.distributed.is_initialized():
            try:
                self._nccl = str(torch.distributed.get_backend(comm)) == "nccl"   # comm None = the default group; gloo (CPU tests) has no reduce_scatter: fp32 all-reduce there
            except Exception:
                self._nccl = False
        # bytes of the NEXT GEMM's weight a decode GEMM prefetches into L2 once its own stream is requested.  OFF by default: the
        # prefetched lines do not survive the current GEMM's stream through L2, so the bytes are read twice.  CTS_NEXT_PREFETCH_MB=<n> turns it on for experiments.
        self.next_prefetch_bytes = int(float(_os.environ.get("CTS_NEXT_PREFETCH_MB", "0")) * (1 << 20))
        self.w4 = None               # W4A16 decode weights (csrc/gemm_w4.cu): set by attach_w4 / quantize_w4_synthetic / from_pretrained(GPTQ)
        self.fp8 = None              # FP8 projection weights (csrc/gemm_fp8.cu): set by quantize_fp8
        self._load(state_dict)
        # every position the page table can address has a row in the rotary tables (max_pages * page_size >= max_seq_len), capped by
        # the model's max_position_embeddings; _alloc_pages rejects sequences beyond it (no silent out-of-bounds cos/sin read)
        n_pos = min(cfg.max_position_embeddings, max(self.max_pages * page_size, 16))
        self.cos, self.sin = rope_tables(cfg, n_pos, dtype, self.device)
        self.n_pos = n_pos
        num_pages = max_batch * self.max_pages
        self.kv = torch.zeros(self.L, 2, num_pages, self.nkv, page_size, self.d, device=self.device, dtype=dtype)
        # prefix caching (chatts_b200/prefix_cache.py): generate() and ContinuousEngine reuse the KV pages of a prompt prefix an earlier
        # prefill wrote; forward() never does.  Off: the plain free list, and every prefill computes every position.
        self.enable_prefix_caching = bool(enable_prefix_caching)
        self.pool = prefix_cache.CachingPagePool(num_pages) if self.enable_prefix_caching else PagePool(num_pages)
        self._prefix_epoch = 0
        self._prefix_queried = self._prefix_hits = 0
        self._steps = {}
        self.peer, self.peer_tokens = None, 0
        if tp_size > 1 and use_peer_allreduce:
            from .tp import PeerBuffers
            self.peer_tokens = max(max_batch, 64)
            self.peer = PeerBuffers(self.ctx, tp_rank, tp_size, self.peer_tokens, self.H, group=comm)

    # ------------------------------------------------------------------------------------------ loading
    def _load(self, sd):
        cfg, dev, dt = self.config, self.device, self.dtype

        def take(name):
            t = sd[name]
            t = shard_tensor(name, t, cfg, self.tp_rank, self.tp_size)
            return t.to(dev, dt).contiguous()

        self.embed = take("model.embed_tokens.weight")
        self.final_norm = take("model.norm.weight")
        self.lm_head = take("lm_head.weight") if "lm_head.weight" in sd else (
            shard_tensor("lm_head.weight", sd["model.embed_tokens.weight"], cfg, self.tp_rank, self.tp_size).to(dev, dt).contiguous())
        self.ln1, self.ln2, self.wqkv, self.bqkv, self.wo, self.wgu, self.wd = [], [], [], [], [], [], []
        self.qn, self.kn = [], []
        for l in range(self.L):
            p = f"model.layers.{l}."
            self.ln1.append(take(p + "input_layernorm.weight"))
            self.ln2.append(take(p + "post_attention_layernorm.weight"))
            self.wqkv.append(torch.cat([take(p + f"self_attn.{n}_proj.weight") for n in "qkv"], 0).contiguous())
            if (p + "self_attn.q_proj.bias") in sd:
                self.bqkv.append(torch.cat([take(p + f"self_attn.{n}_proj.bias") for n in "qkv"], 0).contiguous())
            else:
                self.bqkv.append(None)
            has_qkn = (p + "self_attn.q_norm.weight") in sd          # Qwen3 / ChatTS-8B
            self.qn.append(take(p + "self_attn.q_norm.weight") if has_qkn else None)
            self.kn.append(take(p + "self_attn.k_norm.weight") if has_qkn else None)
            self.wo.append(take(p + "self_attn.o_proj.weight"))
            # gate/up INTERLEAVED per 128-row tile (64 gate rows, then the 64 matching up rows): SwiGLU becomes local to
            # one MMA tile (CTS_EPI_SWIGLU_IL in the persistent prefill GEMM; cts_reduce_swiglu(interleaved) at decode)
            g, u = take(p + "mlp.gate_proj.weight"), take(p + "mlp.up_proj.weight")
            assert g.shape[0] % 64 == 0, "intermediate_size (per rank) must be a multiple of 64"
            self.wgu.append(torch.stack([g.view(-1, 64, g.shape[1]), u.view(-1, 64, u.shape[1])], 1).reshape(2 * g.shape[0], g.shape[1]).contiguous())
            del g, u
            self.wd.append(take(p + "mlp.down_proj.weight"))
        ts_w = {k: v for k, v in sd.items() if k.startswith("ts_encoder.")}
        self.ts_encoder = TimeSeriesEmbedding(cfg.ts, ts_w, device=dev, dtype=dt) if ts_w else None

    @classmethod
    def from_synthetic(cls, config=None, seed=1234, device="cuda", dtype=torch.bfloat16, gen_device=None, quantization=None, **kw):
        """Random-init weights at the config's shapes (no checkpoint exists offline).  ``gen_device='cpu'`` gives
        values identical to the CPU oracle's; the default generates on the GPU (14B in seconds).  quantization="fp8": quantize_fp8()."""
        _check_quantization(quantization)
        config = config or ChatTSConfig.chatts_14b()
        sd = synthetic_state_dict(config, seed=seed, device=gen_device or device, dtype=dtype)
        model = cls(config, sd, device=device, dtype=dtype, **kw)
        del sd
        return model.quantize_fp8() if quantization == "fp8" else model

    @classmethod
    def from_pretrained(cls, path, device_map=None, torch_dtype=None, trust_remote_code=True, device=None, quantization=None, **kw):
        """AutoModelForCausalLM.from_pretrained surface (README.md:88): config.json + safetensors shards.  quantization="fp8": the
        decoder projections are quantised to FP8 at load time (quantize_fp8); None keeps the checkpoint's dtype."""
        _check_quantization(quantization)
        cfg = ChatTSConfig.from_json(path)
        dt = {"float16": torch.float16, "bfloat16": torch.bfloat16, torch.float16: torch.float16,
              torch.bfloat16: torch.bfloat16, None: getattr(torch, cfg.torch_dtype, torch.bfloat16)}[torch_dtype]
        dev = device if device is not None else (f"cuda:{device_map}" if isinstance(device_map, int) else (device_map or "cuda"))
        sd = load_checkpoint(path, device="cpu")
        w4_packed, w4_gs = None, 0
        if any(k.endswith(".qweight") for k in sd):                # GPTQ-Int4 checkpoint (README.md:52,262-263)
            if quantization is not None:
                raise ValueError(f"quantization={quantization!r} applies to 16-bit checkpoints; {path} is already GPTQ-quantised")
            import json as _json
            import os as _os
            from .weights import dequantize_gptq, gptq_w4_pack
            cj = _os.path.join(path, "config.json") if _os.path.isdir(path) else path
            qc = _json.load(open(cj)).get("quantization_config", {})
            # decode streams the 4-bit codes (csrc/gemm_w4.cu); prefill runs on a dequantised copy holding the same values (the scales
            # rounded to the model dtype, which is what the kernel multiplies with).  Act-order checkpoints, tensor parallelism and
            # CTS_W4=0 keep the dequantised weights only.
            if _os.environ.get("CTS_W4", "1") != "0" and kw.get("tp_size", 1) == 1:
                w4_packed, w4_gs = gptq_w4_pack(sd, qc, dtype=dt)
            sd = dequantize_gptq(sd, qc, dtype=dt, scale_dtype=dt if w4_packed is not None else None)
        model = cls(cfg, sd, device=dev, dtype=dt, **kw)
        del sd
        if w4_packed is not None:
            model.attach_w4(w4_packed, w4_gs)
        if quantization == "fp8":
            model.quantize_fp8()
        # generation_config.json: the defaults HF's generate() applies when the caller passes none (README.md:102 calls
        # model.generate(**inputs, max_new_tokens=300) with no sampling arguments)
        import json as _json2
        import os as _os2
        gc = _os2.path.join(path, "generation_config.json") if _os2.path.isdir(path) else ""
        if gc and _os2.path.exists(gc):
            model.generation_defaults = {k: v for k, v in _json2.load(open(gc)).items()
                                         if k in ("do_sample", "temperature", "top_p", "top_k", "eos_token_id", "pad_token_id", "max_new_tokens",
                                                  "repetition_penalty")}
        return model

    # ------------------------------------------------------------------------------------------ LoRA
    def merge_lora(self, adapter, lora_alpha=None, r=None):
        """PeftModel.from_pretrained(model, adapter).merge_and_unload() (demo/demo_lora.ipynb cells 3-4): fold LoRA adapters
        into the resident weights, W += (alpha / r) * B @ A, for q/k/v/o/gate/up/down_proj.  ``adapter`` is a directory with
        adapter_model.safetensors + adapter_config.json, or a name->tensor dict (PEFT names:
        ``...layers.{i}.self_attn.q_proj.lora_A.weight`` [r, in], ``...lora_B.weight`` [out, r]).  Load-time host logic:
        the merged weights then run through the same kernels."""
        import json
        import os
        import re
        if self.fp8 is not None:
            raise ValueError("merge_lora on an FP8 model: the 16-bit projection weights are gone -- merge the adapter into the 16-bit "
                             "model first, then call quantize_fp8()")
        self._prefix_clear()
        if isinstance(adapter, str):
            cfg_path = os.path.join(adapter, "adapter_config.json")
            if os.path.exists(cfg_path):
                ac = json.load(open(cfg_path))
                lora_alpha = ac.get("lora_alpha", lora_alpha) if lora_alpha is None else lora_alpha
                r = ac.get("r", r) if r is None else r
            from safetensors.torch import load_file
            sd = load_file(os.path.join(adapter, "adapter_model.safetensors"))
        else:
            sd = dict(adapter)
        pairs = {}
        for name, t in sd.items():
            m = re.search(r"layers\.(\d+)\.(?:self_attn|mlp)\.(\w+_proj)\.lora_([AB])(?:\.\w+)?\.weight$", name)
            if m:
                pairs.setdefault((int(m.group(1)), m.group(2)), {})[m.group(3)] = t
        if not pairs:
            raise ValueError("no LoRA tensors (…{q,k,v,o,gate,up,down}_proj.lora_{A,B}.weight) found in the adapter")
        cfg, d = self.config, self.d
        nh_t, nkv_t = cfg.num_attention_heads, cfg.num_key_value_heads
        merged = 0
        for (l, proj), ab in sorted(pairs.items()):
            A, B = ab["A"].to(self.device, torch.float32), ab["B"].to(self.device, torch.float32)
            rank = A.shape[0]
            scale = float(lora_alpha if lora_alpha is not None else rank) / float(r if r is not None else rank)
            delta = (B @ A) * scale                                   # [out, in] in the unsharded HF shape
            delta = shard_tensor(f"model.layers.{l}.{'self_attn' if proj[0] in 'qkvo' else 'mlp'}.{proj}.weight", delta, cfg,
                                 self.tp_rank, self.tp_size)

            def add(w_rows, dlt):
                w_rows.copy_((w_rows.float() + dlt).to(self.dtype))

            if proj == "q_proj":
                add(self.wqkv[l][: self.nh * d], delta)
            elif proj == "k_proj":
                add(self.wqkv[l][self.nh * d:(self.nh + self.nkv) * d], delta)
            elif proj == "v_proj":
                add(self.wqkv[l][(self.nh + self.nkv) * d:], delta)
            elif proj == "o_proj":
                add(self.wo[l], delta)
            elif proj == "down_proj":
                add(self.wd[l], delta)
            elif proj in ("gate_proj", "up_proj"):
                # interleaved layout: tile k holds gate rows [64k, 64k+64) then up rows [64k, 64k+64)
                v = self.wgu[l].view(-1, 2, 64, self.H)
                sel = v[:, 0 if proj == "gate_proj" else 1]
                sel.copy_((sel.float() + delta.view(-1, 64, self.H)).to(self.dtype))
            else:
                continue
            merged += 1
        return merged          # in-place update: captured decode graphs keep reading the same (now merged) buffers

    # ------------------------------------------------------------------------------------------ W4A16 (GPTQ-Int4, README.md:52,262-263)
    def attach_w4(self, packed, group_size):
        """Switch the DECODE step to the 4-bit weight stream.  ``packed``: {HF linear name (e.g. 'model.layers.3.mlp.up_proj'):
        (qw uint8 [out, in/2], scales [out, in/g], zeros uint8 [out, in/g])} in the layout of weights.py:repack_gptq_w4, for all
        seven projections of every layer.  The dense weights stay (prefill and every T > 32 step use them): they must hold the SAME
        values, i.e. weights.py:dequantize_gptq(..., scale_dtype=model dtype) -- HBM keeps both copies.  Fused operands
        are assembled exactly like the dense ones: q|k|v stacked, gate/up interleaved per 64 rows.  Single GPU (a tensor-parallel
        row split would cut groups: down_proj's 13824 / 8 = 1728 inputs are not a multiple of the group size)."""
        if self.fp8 is not None:
            raise ValueError("attach_w4 on an FP8 model: the projections are already quantised")
        if self.tp_size != 1:
            raise ValueError("W4A16 decode weights are single-GPU (tensor parallelism uses the dequantised weights)")
        self._prefix_clear()
        dev = self.device
        gs = int(group_size)
        w4 = dict(group_size=gs, qkv=[], o=[], gu=[], d=[])

        def get(name):
            qw, sc, zp = packed[name]
            return qw.to(dev).contiguous(), sc.to(dev, self.dtype).contiguous(), zp.to(dev).contiguous()

        def il(a, b):                     # gate/up interleaved per 64 output rows, as _load does for the dense weight
            return torch.stack([a.view(-1, 64, a.shape[1]), b.view(-1, 64, b.shape[1])], 1).reshape(2 * a.shape[0], a.shape[1]).contiguous()

        for l in range(self.L):
            p = f"model.layers.{l}."
            q, k, v = (get(p + f"self_attn.{n}_proj") for n in "qkv")
            w4["qkv"].append(tuple(torch.cat([a, b, c], 0).contiguous() for a, b, c in zip(q, k, v)))
            w4["o"].append(get(p + "self_attn.o_proj"))
            g, u = get(p + "mlp.gate_proj"), get(p + "mlp.up_proj")
            w4["gu"].append(tuple(il(a, b) for a, b in zip(g, u)))
            w4["d"].append(get(p + "mlp.down_proj"))
        c = self.ctx
        import os as _os
        # kernel of the decode step: "mma" (default) = csrc/gemm_w4_mma.cu, the codes dequantised in registers from the fragment-major copy
        # built here (the row layout is dropped per layer once it is converted); "tc5" = csrc/gemm_w4.cu (wgmma, bit-identical to the
        # dense GEMM, no faster than it: kept as the checker)
        w4["kernel"] = _os.environ.get("CTS_W4_KERNEL", "mma")
        k_dims = (self.H, self.nh * self.d, self.I)
        if w4["kernel"] == "mma" and not (all(kd % 128 == 0 for kd in k_dims) and (gs == 64 or gs % 128 == 0)):
            w4["kernel"] = "tc5"          # the mma kernel's pipeline stage is 128 K wide (cts_gemm_w4f_args): odd shapes take the wgmma kernel
        if w4["kernel"] == "mma":
            from .weights import repack_w4_mma
            for kind in ("qkv", "o", "gu", "d"):
                for l in range(self.L):
                    qw, sc, zp = w4[kind][l]
                    w4[kind][l] = repack_w4_mma(qw, sc, zp, gs) + (int(qw.shape[0]),)
            w4["splits"] = None           # per batch size: _w4_splits
        else:
            w4["splits"] = dict(qkv=c.gemm_w4_suggest_split(self._n_qkv, self.H), o=c.gemm_w4_suggest_split(self.H, self.nh * self.d),
                                gu=c.gemm_w4_suggest_split(2 * self.I, self.H), d=c.gemm_w4_suggest_split(self.H, self.I))
        self.w4 = w4
        self._steps = {}                  # decode states (workspaces, captured graphs) are rebuilt for the new launches
        return self

    def quantize_w4_synthetic(self, group_size=128, seed=7):
        """Benchmark / test helper (no GPTQ checkpoint exists offline): draw random 4-bit codes, scales and zero points at the model's
        shapes, REPLACE the dense weights by their dequantised values and attach the packed copy -- a W4A16 model whose prefill and
        decode paths see the same weights."""
        from .weights import dequantize_w4, W4_NIBBLE_OF_K  # noqa: F401
        if self.fp8 is not None:
            raise ValueError("quantize_w4_synthetic on an FP8 model: the projections are already quantised")
        self._prefix_clear()
        g = torch.Generator(device=self.device).manual_seed(seed)
        packed = {}

        def make(n_out, n_in):
            qw = torch.randint(0, 256, (n_out, n_in // 2), generator=g, device=self.device, dtype=torch.uint8)
            sc = ((torch.rand(n_out, n_in // group_size, generator=g, device=self.device) * 0.5 + 0.75) * (0.02 * 3.46 / 7.5)).to(self.dtype)
            zp = torch.randint(7, 10, (n_out, n_in // group_size), generator=g, device=self.device, dtype=torch.uint8)
            return qw, sc, zp

        d, H, I = self.d, self.H, self.I
        for l in range(self.L):
            p = f"model.layers.{l}."
            parts = {}
            for name, (n_out, n_in) in (("self_attn.q_proj", (self.nh * d, H)), ("self_attn.k_proj", (self.nkv * d, H)), ("self_attn.v_proj", (self.nkv * d, H)),
                                        ("self_attn.o_proj", (H, self.nh * d)), ("mlp.gate_proj", (I, H)), ("mlp.up_proj", (I, H)), ("mlp.down_proj", (H, I))):
                t = make(n_out, n_in)
                packed[p + name] = t
                parts[name] = dequantize_w4(*t, group_size)
            self.wqkv[l].copy_(torch.cat([parts["self_attn.q_proj"], parts["self_attn.k_proj"], parts["self_attn.v_proj"]], 0))
            self.wo[l].copy_(parts["self_attn.o_proj"])
            gp, up = parts["mlp.gate_proj"], parts["mlp.up_proj"]
            self.wgu[l].copy_(torch.stack([gp.view(-1, 64, H), up.view(-1, 64, H)], 1).reshape(2 * I, H))
            self.wd[l].copy_(parts["mlp.down_proj"])
            del parts
        return self.attach_w4(packed, group_size)

    # ------------------------------------------------------------------------------------------ FP8 weights (vLLM's quantization="fp8")
    def quantize_fp8(self):
        """Quantise the seven projections of every layer (fused q|k|v, gate/up interleaved, o, down) to FP8 in place: e4m3 codes (round
        to nearest even) with one fp32 scale per output feature, s_n = max|W[n, :]| / 448 over the full checkpoint row (under tensor
        parallelism the K-sliced o_proj / down_proj rows take the maximum over the ranks, so every rank holds a slice of the single-GPU
        codes).  The 16-bit projection tensors are freed; embeddings, norms, biases, lm_head, the TS encoder and the KV cache stay in the
        model dtype.  Decode-sized steps stream the codes (cts_gemm_fp8); every other step dequantises each projection into one
        scratch matrix just before its GEMM (cts_fp8_dequant + cts_gemm).  Returns the model."""
        from .weights import pack_fp8_mma, quantize_fp8_rows
        if self.fp8 is not None:
            raise ValueError("quantize_fp8() was already called on this model")
        if self.w4 is not None:
            raise ValueError("quantize_fp8 on a W4A16 model: its projections are already quantised")
        kinds = (("qkv", self.wqkv, False), ("o", self.wo, True), ("gu", self.wgu, False), ("d", self.wd, True))
        names = dict(qkv="self_attn.{q,k,v}_proj", o="self_attn.o_proj", gu="mlp.{gate,up}_proj", d="mlp.down_proj")
        # every refusal before the first tensor is freed
        for kind, ws, _ in kinds:
            if ws[0].shape[1] % 64 != 0:
                raise ValueError(f"quantize_fp8: {names[kind]} has {ws[0].shape[1]} input features per rank; the FP8 kernels need a multiple of 64")
        for l in range(self.L):
            for kind, ws, _ in kinds:
                if not bool(torch.isfinite(ws[l]).all()):
                    raise ValueError(f"quantize_fp8: model.layers.{l}.{names[kind]}.weight holds non-finite values")
        fp8 = dict(qkv=[], o=[], gu=[], d=[])
        biggest = 0
        for l in range(self.L):
            for kind, ws, row_parallel in kinds:
                w = ws[l]
                row_max = w.abs().amax(1).to(torch.float32)
                if row_parallel and self.tp_size > 1:
                    torch.distributed.all_reduce(row_max, op=torch.distributed.ReduceOp.MAX, group=self.comm)
                codes, scales = quantize_fp8_rows(w, row_max, f"model.layers.{l}.{names[kind]}.weight")
                fp8[kind].append((pack_fp8_mma(codes), scales, int(w.shape[1])))
                biggest = max(biggest, w.numel())
                ws[l] = None
                del w, codes
        # one scratch matrix for the dequantised projection of prefill-sized steps (stream order: each GEMM reads it before the next
        # dequantisation overwrites it)
        fp8["scratch"] = torch.empty(biggest, device=self.device, dtype=self.dtype)
        self.fp8 = fp8
        self._prefix_clear()
        self._steps = {}
        if hasattr(self, "_layer_list"):
            del self._layer_list
        if self.device.type == "cuda":
            torch.cuda.empty_cache()
        return self

    def _fp8_dense(self, ent):
        """16-bit row-major copy of one FP8 projection in the scratch matrix (prefill-sized steps)."""
        qw, sc, k = ent
        out = self.fp8["scratch"][: sc.shape[0] * k].view(sc.shape[0], k)
        self.ctx.fp8_dequant(qw, sc, k, out)
        return out

    def _fp8_splits(self, T):
        """Split-K factors of the four projections for an FP8 decode step of T tokens."""
        c = self.ctx
        return dict(qkv=c.gemm_fp8_suggest_split(self._n_qkv, self.H, T), o=c.gemm_fp8_suggest_split(self.H, self.nh * self.d, T),
                    gu=c.gemm_fp8_suggest_split(2 * self.I, self.H, T), d=c.gemm_fp8_suggest_split(self.H, self.I, T))

    @property
    def _n_qkv(self):
        return (self.nh + 2 * self.nkv) * self.d

    # ------------------------------------------------------------------------------------------ layers
    def _splits(self, T):
        c = self.ctx
        import os
        ov = os.environ.get("CTS_SPLITS")          # tuning override "qkv,o,gu,d" (decode-sized T only)
        if ov and T <= 32:
            a = [int(v) for v in ov.split(",")]
            return dict(qkv=a[0], o=a[1], gu=a[2], d=a[3])
        return dict(qkv=c.suggest_split(self._n_qkv, self.H, T), o=c.suggest_split(self.H, self.nh * self.d, T),
                    gu=c.suggest_split(self.I, self.H, T, True), d=c.suggest_split(self.H, self.I, T))

    def _ws_floats(self, T, sp):
        return max(sp["qkv"] * T * self._n_qkv if sp["qkv"] > 1 else 0, sp["o"] * T * self.H if sp["o"] > 1 else 0,
                   sp["gu"] * T * 2 * self.I if T <= 128 else 0, sp["d"] * T * self.H if sp["d"] > 1 else 0, 1)

    def _w4_splits(self, T):
        """Split-K factors of the four projections for a W4A16 decode step of T tokens."""
        w4, c = self.w4, self.ctx
        if w4["splits"] is not None:
            return w4["splits"]
        return dict(qkv=c.gemm_w4_mma_suggest_split(self._n_qkv, self.H, T), o=c.gemm_w4_mma_suggest_split(self.H, self.nh * self.d, T),
                    gu=c.gemm_w4_mma_suggest_split(2 * self.I, self.H, T), d=c.gemm_w4_mma_suggest_split(self.H, self.I, T))

    def _layers(self, st, T, attend):
        """Runs every decoder layer on st.h [T,H] in place; leaves RMSNorm_final(h) in st.xn."""
        c, sp, eps = self.ctx, st.splits, self.eps
        I, H = self.I, self.H
        c.reduce_residual_rmsnorm(None, 0, st.h, None, self.ln1[0], eps, st.xn, t=T)
        fp8 = self.fp8
        fused = self.use_fused_decode and T <= 32 and st.k_lin is None and fp8 is None             # decode states only
        # decode-sized steps: every weight-streaming GEMM names the weight its successor will stream, and prefetches the head of it
        # into L2 once its own last tile is requested (cts_gemm_args.next_*): HBM keeps streaming through the kernel boundaries
        nb = self.next_prefetch_bytes if (T <= 32 and st.k_lin is None and fp8 is None) else 0
        # W4A16: decode-sized steps stream the 4-bit codes (every projection through the split-K partial path with the W4 split factors)
        w4 = self.w4 if (self.w4 is not None and T <= 32 and st.k_lin is None and not fused) else None
        if w4 is not None:
            sp = self._w4_splits(T)
        # FP8: decode-sized steps stream the codes the same way; every other step dequantises each projection just before its GEMM
        f8 = fp8 is not None and T <= 32 and st.k_lin is None
        if f8:
            sp = self._fp8_splits(T)
        dense = {"qkv": self.wqkv, "o": self.wo, "gu": self.wgu, "d": self.wd}

        def W(kind, l):
            """The 16-bit weight of a projection for cts_gemm (FP8 model: dequantised into the scratch matrix now)."""
            return dense[kind][l] if fp8 is None else self._fp8_dense(fp8[kind][l])

        def proj(kind, l, x, split, **kw):
            """fp32 split-K partials of one projection into st.ws: from the packed 4-bit / FP8 weight when attached, else from the dense one."""
            if w4 is not None and w4["kernel"] == "mma":
                qwf, szp, n_out = w4[kind][l]
                c.gemm_w4_mma(x, qwf, szp, n_out, w4["group_size"], st.ws, split, t=T)
            elif w4 is not None:
                qw, sc, zp = w4[kind][l]
                c.gemm_w4(x, qw, sc, zp, w4["group_size"], st.ws, split, t=T)
            elif f8:
                qw, sc, k = fp8[kind][l]
                c.gemm_fp8(x, qw, sc, k, st.ws, split, t=T)
            else:
                c.gemm(x, W(kind, l), st.ws, epilogue=EPI_PARTIAL_F32, split_k=split, t=T, **kw)

        def nxt(w, split):
            return dict(next_w=w, next_split=split, next_bytes=nb) if nb > 0 else {}
        for l in range(self.L):
            kc, vc = self.kv[l, 0], self.kv[l, 1]
            if fused:
                # 7 stages per layer: every projection reduces its K splits inside a cluster and applies its tail in the epilogue
                # (under tensor parallelism the row-parallel o_proj / down_proj keep the peer-memory all-reduce kernel, which sums
                # the local splits itself; the column-parallel QKV and gate_up projections are fused all the same)
                nw = self.ln1[l + 1] if l + 1 < self.L else self.final_norm
                # level 2 under tensor parallelism: the row-parallel projections carry their all-reduce INSIDE the GEMM kernel
                # (gemm_decode_fused peer tail; needs the low-latency regions, use_peer_ll) -- 5 launches per layer, none of them a collective
                tp_deep = self.tp_size > 1 and self.use_peer_ll and self.peer is not None and H % (128 * self.tp_size) == 0
                deep = self.use_fused_decode >= 2 and (self.tp_size == 1 or tp_deep)
                pr = [None, None]
                so, sd = min(sp["o"], 8), min(sp["d"], 8)
                if deep and self.tp_size > 1:
                    # a (tile, token) of the in-kernel all-reduce waits for the same tile's CTAs on the other ranks: keep every rank's
                    # whole grid resident (one CTA per SM suffices) instead of relying on the order CTAs are scheduled in
                    cap = max(1, 148 // max(1, H // 128))
                    so, sd = min(so, cap), min(sd, cap)
                    pr = [(self.peer.partials[w], self.peer.part_bytes, self.peer.state, self.tp_rank, self.tp_size, self.peer.max_batch) for w in (0, 1)]
                rope = dict(bias=self.bqkv[l], positions=st.positions, cos=self.cos, sin=self.sin, slot_map=st.slot_map, q_out=st.q, k_cache=kc,
                            v_cache=vc, q_norm=self.qn[l], k_norm=self.kn[l], eps=eps, nh=self.nh, nkv=self.nkv, head_dim=self.d,
                            page_size=self.page_size)
                if deep:
                    # 5 stages: QKV(norm in, RoPE out) -> attention -> o_proj(+residual, sum of squares out) -> gate_up(norm in, SwiGLU out)
                    # -> down(+residual, sum of squares out); layer 0 takes the xn of the plain RMSNorm above
                    if l == 0:
                        c.gemm_decode_fused(st.xn, self.wqkv[l], _cabi.FUSED_QKV_ROPE, min(sp["qkv"], 8), T, **rope)
                    else:
                        c.gemm_decode_fused(None, self.wqkv[l], _cabi.FUSED_QKV_ROPE, min(sp["qkv"], 8), T, norm_h=st.h, norm_w=self.ln1[l],
                                            ssq_in=st.ssq_b, norm_eps=eps, **rope)
                    attend(l)
                    c.gemm_decode_fused(st.ao, self.wo[l], _cabi.FUSED_RESIDUAL, so, T, h=st.h, ssq_out=st.ssq_a, peer=pr[0])
                    c.gemm_decode_fused(None, self.wgu[l], _cabi.FUSED_SWIGLU, min(sp["gu"], 8), T, act=st.act, norm_h=st.h, norm_w=self.ln2[l],
                                        ssq_in=st.ssq_a, norm_eps=eps)
                    c.gemm_decode_fused(st.act, self.wd[l], _cabi.FUSED_RESIDUAL, sd, T, h=st.h, ssq_out=st.ssq_b, peer=pr[1])
                    if l + 1 == self.L:
                        c.reduce_residual_rmsnorm(None, 0, st.h, None, self.final_norm, eps, st.xn, t=T)
                    continue
                c.gemm_decode_fused(st.xn, self.wqkv[l], _cabi.FUSED_QKV_ROPE, min(sp["qkv"], 8), T, **rope)
                attend(l)
                if self.tp_size > 1:
                    self._tp_row_parallel(st, T, st.ao, self.wo[l], self.ln2[l], 0, sp["o"])
                else:
                    c.gemm_decode_fused(st.ao, self.wo[l], _cabi.FUSED_RESIDUAL, min(sp["o"], 8), T, h=st.h)
                    c.reduce_residual_rmsnorm(None, 0, st.h, None, self.ln2[l], eps, st.xn, t=T)
                c.gemm_decode_fused(st.xn, self.wgu[l], _cabi.FUSED_SWIGLU, min(sp["gu"], 8), T, act=st.act)
                if self.tp_size > 1:
                    self._tp_row_parallel(st, T, st.act, self.wd[l], nw, 1, sp["d"])
                else:
                    c.gemm_decode_fused(st.act, self.wd[l], _cabi.FUSED_RESIDUAL, min(sp["d"], 8), T, h=st.h)
                    c.reduce_residual_rmsnorm(None, 0, st.h, None, nw, eps, st.xn, t=T)
                continue
            # ---- QKV projection + bias + RoPE + KV write
            if sp["qkv"] > 1 or w4 is not None or f8:
                proj("qkv", l, st.xn, sp["qkv"], **nxt(self.wo[l], sp["o"]))
                c.qkv_rope_cache(st.ws, True, sp["qkv"], self.bqkv[l], st.positions, self.cos, self.sin, st.slot_map, st.q, kc, vc,
                                 st.k_lin, st.v_lin, T, self.nh, self.nkv, self.d, self.page_size, self.qn[l], self.kn[l], eps)
            else:
                c.gemm(st.xn, W("qkv", l), st.qkv, bias=self.bqkv[l], epilogue=EPI_NONE, t=T, **nxt(self.wo[l], sp["o"]))
                c.qkv_rope_cache(st.qkv, False, 1, None, st.positions, self.cos, self.sin, st.slot_map, st.q, kc, vc,
                                 st.k_lin, st.v_lin, T, self.nh, self.nkv, self.d, self.page_size, self.qn[l], self.kn[l], eps)
            attend(l)
            # ---- o_proj + residual + post-attention RMSNorm
            if self.tp_size > 1:
                self._tp_row_parallel(st, T, st.ao, fp8["o"][l] if f8 else W("o", l), self.ln2[l], 0, sp["o"], nxt(self.wgu[l], sp["gu"]))
            elif sp["o"] > 1 or w4 is not None or f8:
                proj("o", l, st.ao, sp["o"], **nxt(self.wgu[l], sp["gu"]))
                c.reduce_residual_rmsnorm(st.ws, sp["o"], st.h, st.h, self.ln2[l], eps, st.xn, t=T)
            else:
                c.gemm(st.ao, W("o", l), st.h, residual=st.h, epilogue=EPI_RESIDUAL, t=T, **nxt(self.wgu[l], sp["gu"]))
                c.reduce_residual_rmsnorm(None, 0, st.h, None, self.ln2[l], eps, st.xn, t=T)
            # ---- gate/up + SwiGLU
            if T > 128:
                c.gemm(st.xn, W("gu", l), st.act, epilogue=EPI_SWIGLU_IL, t=T)          # persistent, SwiGLU fused in the tile
            else:
                proj("gu", l, st.xn, sp["gu"], **nxt(self.wd[l], sp["d"]))
                c.reduce_swiglu(st.ws, sp["gu"], T, I, st.act, interleaved=True)
            # ---- down_proj + residual + next layer's input RMSNorm (or the final norm)
            nw = self.ln1[l + 1] if l + 1 < self.L else self.final_norm
            after = nxt(self.wqkv[l + 1], sp["qkv"]) if l + 1 < self.L else nxt(self.lm_head, 1)
            if self.tp_size > 1:
                self._tp_row_parallel(st, T, st.act, fp8["d"][l] if f8 else W("d", l), nw, 1, sp["d"], after)
            elif sp["d"] > 1 or w4 is not None or f8:
                proj("d", l, st.act, sp["d"], **after)
                c.reduce_residual_rmsnorm(st.ws, sp["d"], st.h, st.h, nw, eps, st.xn, t=T)
            else:
                c.gemm(st.act, W("d", l), st.h, residual=st.h, epilogue=EPI_RESIDUAL, t=T, **after)
                c.reduce_residual_rmsnorm(None, 0, st.h, None, nw, eps, st.xn, t=T)

    def _tp_row_parallel(self, st, T, x, w, norm_w, which, split, nxt=None):
        """Row-parallel projection under tensor parallelism: local split-K partials -> sum over splits and ranks ->
        residual + norm.  Decode-sized T: ONE kernel over NVLink peer memory (cts_peer_allreduce_residual_rmsnorm: each
        CTA reduces its token's local split-K partials into the symmetric buffer, signals, pulls the peers' rows; the
        buffers alternate between o_proj (0) and down_proj (1)).  Large prefill T: NCCL (bandwidth-bound) -- fp32 reduce-scatter over token
        shards + all-gather of the rounded result by default, see the branches below.  ``w``: the 16-bit weight, or the (codes, scales, k)
        of an FP8 projection for a decode-sized step (cts_gemm_fp8)."""
        c = self.ctx
        big = split == 1 and not (self.peer is not None and T <= self.peer_tokens)
        if isinstance(w, tuple) and big:
            w = self._fp8_dense(w)
        if big and self.tp_prefill_exchange == "16bit":
            # Opt-in (CTS_TP_PREFILL_EXCHANGE=16bit): every rank rounds its projection to the model dtype and NCCL sums the ranks' outputs
            # in that dtype -- what vLLM's RowParallelLinear does (qwen2.py:100-116 / 168-174) -- half the bytes of the fp32 all-reduce.
            # Not the default: the sum is re-rounded at every ring step, which moves the logits further from the single-GPU model.
            proj = st.tp_proj
            c.gemm(x, w, proj, epilogue=EPI_NONE, t=T)
            torch.distributed.all_reduce(proj[:T], group=self.comm)
            st.h[:T].add_(proj[:T])                               # residual add in the model dtype (one rounding, as the fused tail does)
            c.reduce_residual_rmsnorm(None, 0, st.h, st.h, norm_w, self.eps, st.xn, t=T)
            return
        if big and self.tp_prefill_exchange == "rs_ag" and self._nccl:
            # Default for prefill-sized T: the fp32 sum is kept (reduce-scatter of the fp32 partials over token shards, summed by NCCL in
            # fp32) and only the RESULT travels in the model dtype (all-gather of the rounded shards): three quarters of the bytes of the
            # fp32 all-reduce, the same numbers as the single-GPU path up to the order of the fp32 sum -- h = resid + dtype(sum).
            W = self.tp_size
            ct = -(-T // W)                                       # tokens per shard (the last shard is padded: st.ws / st.tp_proj hold W * ct rows)
            c.gemm(x, w, st.ws, epilogue=EPI_PARTIAL_F32, split_k=1, t=T, **(nxt or {}))
            part = st.ws.view(-1)[: W * ct * self.H]
            torch.distributed.reduce_scatter_tensor(st.tp_shard32, part, group=self.comm)
            st.tp_shard16.copy_(st.tp_shard32)                    # ONE rounding of the projection to the model dtype (cast = plumbing)
            torch.distributed.all_gather_into_tensor(st.tp_proj.view(-1)[: W * ct * self.H], st.tp_shard16, group=self.comm)
            st.h[:T].add_(st.tp_proj[:T])                         # residual add in the model dtype, as the fused tail does
            c.reduce_residual_rmsnorm(None, 0, st.h, st.h, norm_w, self.eps, st.xn, t=T)
            return
        if isinstance(w, tuple):
            c.gemm_fp8(x, w[0], w[1], w[2], st.ws, split, t=T)
        else:
            c.gemm(x, w, st.ws, epilogue=EPI_PARTIAL_F32, split_k=split, t=T, **(nxt or {}))
        if self.peer is not None and T <= self.peer_tokens and self.use_peer_ll:
            c.peer_allreduce_ll(st.ws, split, self.peer.partials[which], self.peer.part_bytes, self.peer.state, self.tp_rank, self.tp_size,
                                self.peer.max_batch, st.h, st.h, norm_w, self.eps, st.xn, T)
            return
        if self.peer is not None and T <= self.peer_tokens:
            c.peer_allreduce_residual_rmsnorm(st.ws, split, self.peer.partials[which], self.peer.flags[which], self.peer.state,
                                              self.tp_rank, self.tp_size, self.peer.max_batch, st.h, st.h, norm_w, self.eps,
                                              st.xn, T)
            return
        part = st.ws[: T * self.H] if split == 1 else st.ws.view(-1)[: split * T * self.H].view(split, T * self.H).sum(0)
        torch.distributed.all_reduce(part, group=self.comm)
        c.reduce_residual_rmsnorm(part, 1, st.h, st.h, norm_w, self.eps, st.xn, t=T)

    def _alloc_step(self, T, decode):
        st = _Step()
        dev, dt = self.device, self.dtype
        st.splits = self._splits(T)
        st.h = torch.empty(T, self.H, device=dev, dtype=dt)
        st.xn = torch.empty(T, self.H, device=dev, dtype=dt)
        st.q = torch.empty(T, self.nh * self.d, device=dev, dtype=dt)
        st.ao = torch.empty(T, self.nh * self.d, device=dev, dtype=dt)
        st.act = torch.empty(T, self.I, device=dev, dtype=dt)
        st.tp_proj = st.tp_shard32 = st.tp_shard16 = None
        tp_pad = 0
        if self.tp_size > 1 and not decode:                     # row-parallel exchange of a prefill: token shards of ceil(T / W) rows
            ct = -(-T // self.tp_size)
            tp_pad = self.tp_size * ct
            st.tp_proj = torch.empty(tp_pad, self.H, device=dev, dtype=dt)
            st.tp_shard32 = torch.empty(ct * self.H, device=dev, dtype=torch.float32)
            st.tp_shard16 = torch.empty(ct * self.H, device=dev, dtype=dt)
        st.qkv = torch.empty(T, self._n_qkv, device=dev, dtype=dt) if st.splits["qkv"] == 1 else None
        ws_n = max(self._ws_floats(T, st.splits), T * self.H, tp_pad * self.H)
        if decode and self.w4 is not None and T <= 32:   # W4A16 decode: every projection through the partial path with the W4 split factors
            sp = self._w4_splits(T)
            ws_n = max(ws_n, sp["qkv"] * T * self._n_qkv, sp["o"] * T * self.H, sp["gu"] * T * 2 * self.I, sp["d"] * T * self.H)
        if decode and self.fp8 is not None and T <= 32:  # FP8 decode: every projection through the partial path with the FP8 split factors
            sp = self._fp8_splits(T)
            ws_n = max(ws_n, sp["qkv"] * T * self._n_qkv, sp["o"] * T * self.H, sp["gu"] * T * 2 * self.I, sp["d"] * T * self.H)
        if decode and self.use_native_step:          # cts_decoder_step always takes the split-K partial path (also at factor 1)
            sp = st.splits
            ws_n = max(ws_n, sp["qkv"] * T * self._n_qkv, sp["o"] * T * self.H, sp["gu"] * T * 2 * self.I, sp["d"] * T * self.H)
        st.ws = torch.empty(ws_n, device=dev, dtype=torch.float32)                           # split-K partials [S, T, N]
        st.positions = torch.zeros(T, device=dev, dtype=torch.int32)
        st.slot_map = torch.zeros(T, device=dev, dtype=torch.int32)
        if decode:
            st.k_lin = st.v_lin = None
        else:
            st.k_lin = torch.empty(T, self.nkv * self.d, device=dev, dtype=dt)
            st.v_lin = torch.empty(T, self.nkv * self.d, device=dev, dtype=dt)
        return st

    # ------------------------------------------------------------------------------------------ prefill
    def _prepare_inputs(self, input_ids, attention_mask, timeseries, layout_kind="hf"):
        """Host side of A2/A3/A7: patch counts (one sync), merged layout, page allocation, H2D of the int maps."""
        cfg, dev = self.config, self.device
        ids_cpu = torch.as_tensor(input_ids).cpu().numpy()
        if ids_cpu.ndim == 1:
            ids_cpu = ids_cpu[None]
        am_cpu = None if attention_mask is None else torch.as_tensor(attention_mask).cpu().numpy()
        counts, cnt_h = None, np.zeros(0, dtype=np.int64)
        if timeseries is not None and timeseries.shape[0] > 0:
            if self.ts_encoder is None:
                raise ValueError("time series given but the checkpoint has no ts_encoder weights")
            if not isinstance(timeseries, torch.Tensor):
                raise ValueError(f"Incorrect type of ts input features. Got type: {type(timeseries)}")   # chatts_vllm.py:533-535
            counts = self.ts_encoder.patch_counts(timeseries)            # H2D (if needed) + count kernels, async
            host = torch.stack([counts[1], counts[2]]).cpu()             # the one host sync: (valid_len, patch_cnt)
            self._host_counts = (host[0], host[1])
            cnt_h = host[1].numpy().astype(np.int64)
        if layout_kind == "hf":
            lay = layout.hf_layout(ids_cpu, am_cpu, cnt_h, cfg.ts_token_start_index, self._merge_mode())
        else:
            lay = layout.vllm_layout(ids_cpu, int(cnt_h.sum()), cfg.ts_token_start_index)
        return ids_cpu, am_cpu, counts, lay

    def _merge_mode(self):
        import os as _os
        return _os.environ.get("CTS_TS_MERGE_MODE") or getattr(self.config, "ts_merge_mode", "insert")

    def _prefill(self, lay, counts, timeseries, page_tables, all_logits=False, cached=None, prompt_lp=None):
        """Runs the prompt through the TS encoder + decoder, fills the paged KV cache, returns logits
        ([B,V] last position, or [T,V] for every merged position when all_logits).  ``cached`` (prefix caching, from _alloc_prompt):
        per sequence, the number of leading positions whose KV the pages of ``page_tables`` already hold; only the rest is computed.
        ``prompt_lp`` = k: also the prompt logprobs -- returns (logits, (targets, rows, cols, LogprobBuffers of the targets))."""
        if cached is not None and int(np.max(cached, initial=0)) > 0:
            if all_logits or prompt_lp is not None:
                raise ValueError("all_logits / prompt logprobs need every position computed: no prefix-cache hits")
            return self._prefill_suffix(lay, counts, timeseries, page_tables, np.asarray(cached, dtype=np.int64))
        c, dev, dt = self.ctx, self.device, self.dtype
        T, B = lay.total, lay.cu_seqlens.shape[0] - 1
        lens = lay.lens
        if int(lens.max()) > self.n_pos:
            raise ValueError(f"prompt of {int(lens.max())} positions exceeds max_seq_len {self.n_pos}")
        st = self._alloc_step(T, decode=False)
        # slots of every prompt position in the paged cache
        b_of = np.repeat(np.arange(B), lens)
        pos = lay.positions.astype(np.int64)
        slot = page_tables[b_of, pos // self.page_size].astype(np.int64) * self.page_size + pos % self.page_size
        host = np.concatenate([lay.ids, lay.positions, slot.astype(np.int32), lay.cu_seqlens]).astype(np.int32)
        hbuf = torch.from_numpy(host).pin_memory()
        dbuf = hbuf.to(dev, non_blocking=True)
        ids_d, st.positions, st.slot_map, cu_d = dbuf[:T], dbuf[T:2 * T], dbuf[2 * T:3 * T], dbuf[3 * T:]
        c.embed_gather(self.embed, ids_d, st.h, t=T)
        if counts is not None and lay.row_map.shape[0] > 0:
            rmap = torch.from_numpy(lay.row_map).to(dev, non_blocking=True)
            self.ts_encoder.encode(timeseries, out=st.h, row_map=rmap, counts=counts, host_counts=self._host_counts)
        max_len = int(lens.max())
        scale = 1.0 / math.sqrt(self.d)

        def attend(l):
            c.attn_prefill(st.q, st.k_lin, st.v_lin, cu_d, B, max_len, self.nh, self.nkv, self.d, scale, st.ao)

        self._layers(st, T, attend)
        plp = None if prompt_lp is None else self._prompt_logprobs(lay, st.xn, prompt_lp)
        if all_logits:
            hn = st.xn
        else:
            last = torch.from_numpy((lay.cu_seqlens[1:] - 1).astype(np.int64)).to(dev)
            hn = st.xn.index_select(0, last).contiguous()        # row gather of B rows (plumbing)
        logits = torch.empty(hn.shape[0], self.V, device=dev, dtype=dt)
        c.gemm(hn, self.lm_head, logits, epilogue=EPI_NONE)
        if plp is not None:
            return logits, plp
        return self._gather_vocab(logits)

    PROMPT_LP_CHUNK = 1024

    def _prompt_logprobs(self, lay, xn, k):
        """Prompt logprobs from the final-norm rows xn [T, H] of a prefill: only the positions that predict a prompt token go through
        the lm_head (patch rows that predict a patch row are skipped), in chunks of at most PROMPT_LP_CHUNK rows into one reused logits
        buffer, then cts_logprobs with the next ids as the chosen ids.  -> (targets, rows, cols, LogprobBuffers [N, 1])."""
        dev = self.device
        pred, tgt, rows, cols = lpmod.prompt_targets(lay)
        N = int(pred.shape[0])
        chunk = min(self.PROMPT_LP_CHUNK, max(N, 1))
        buf = lpmod.LogprobBuffers(self.ctx, max(N, 1), 1, k, self.V, dev, launch_rows=chunk)
        if N:
            idx = torch.from_numpy(np.stack([pred.astype(np.int32), tgt])).to(dev, non_blocking=True)
            pred_d, tgt_d = idx[0].long(), idx[1].view(N, 1)
            logits = torch.empty(chunk, self.V, device=dev, dtype=self.dtype)
            for r0 in range(0, N, chunk):
                n = min(chunk, N - r0)
                hn = xn.index_select(0, pred_d[r0:r0 + n])                   # row gather of the predicting positions (plumbing)
                self.ctx.gemm(hn, self.lm_head, logits, epilogue=EPI_NONE, t=n)
                buf.launch(logits, n, tgt_d[r0:r0 + n], row0=r0)
        return tgt, rows, cols, buf

    def _prefill_suffix(self, lay, counts, timeseries, page_tables, cached):
        """_prefill of the positions past each sequence's cached prefix: the embeddings, the series that have a patch row among them and
        the decoder layers run on those positions only, and attention reads the cached keys from the pages (cts_attn_prefill_paged)."""
        c, dev, dt = self.ctx, self.device, self.dtype
        B, lens, cu = lay.cu_seqlens.shape[0] - 1, lay.lens.astype(np.int64), lay.cu_seqlens.astype(np.int64)
        if int(lens.max()) > self.n_pos:
            raise ValueError(f"prompt of {int(lens.max())} positions exceeds max_seq_len {self.n_pos}")
        qlens = lens - cached
        sel = np.concatenate([np.arange(cu[b] + cached[b], cu[b + 1]) for b in range(B)])      # merged positions computed now
        T = int(sel.shape[0])
        row_of = np.full(lay.total, T, dtype=np.int64)        # merged position -> row of this call; T: the discard row
        row_of[sel] = np.arange(T)
        st = self._alloc_step(T, decode=False)
        st.h = torch.empty(T + 1, self.H, device=dev, dtype=dt)
        pos = lay.positions[sel].astype(np.int64)
        b_of = np.repeat(np.arange(B), qlens)
        slot = page_tables[b_of, pos // self.page_size].astype(np.int64) * self.page_size + pos % self.page_size
        cu_q = np.concatenate([[0], np.cumsum(qlens)])
        host = np.concatenate([lay.ids[sel], pos, slot, cu_q, lens, page_tables.reshape(-1)]).astype(np.int32)
        dbuf = torch.from_numpy(host).pin_memory().to(dev, non_blocking=True)
        ids_d, st.positions, st.slot_map = dbuf[:T], dbuf[T:2 * T], dbuf[2 * T:3 * T]
        cu_d, kvl_d = dbuf[3 * T:3 * T + B + 1], dbuf[3 * T + B + 1:3 * T + 2 * B + 1]
        pt_d = dbuf[3 * T + 2 * B + 1:].view(B, -1)
        c.embed_gather(self.embed, ids_d, st.h, t=T)
        if counts is not None and lay.row_map.shape[0] > 0:
            # a series is encoded when one of its patch rows is computed now (whole: the rows of a series that straddles the cached
            # boundary land in the discard row); a series entirely inside the cached prefix is not encoded at all
            cnt = self._host_counts[1].numpy().astype(np.int64)
            series = np.repeat(np.arange(cnt.shape[0]), cnt)
            rows = row_of[lay.row_map]
            keep = np.bincount(series[rows < T], minlength=cnt.shape[0]) > 0
            if keep.any():
                rmap = torch.from_numpy(rows[keep[series]].astype(np.int32)).to(dev, non_blocking=True)
                if keep.all():
                    sub, sub_counts, host_counts = timeseries, counts, self._host_counts
                else:
                    idx = np.nonzero(keep)[0]
                    sub = counts[0][torch.from_numpy(idx).to(counts[0].device)]
                    sub_counts = self.ts_encoder.patch_counts(sub)
                    host_counts = tuple(h[torch.from_numpy(idx)] for h in self._host_counts)
                self.ts_encoder.encode(sub, out=st.h, row_map=rmap, counts=sub_counts, host_counts=host_counts)
        max_q, scale = int(qlens.max()), 1.0 / math.sqrt(self.d)

        def attend(l):
            c.attn_prefill_paged(st.q, cu_d, kvl_d, self.kv[l, 0], self.kv[l, 1], pt_d, B, max_q, self.nh, self.nkv, self.d,
                                 self.page_size, scale, st.ao)

        self._layers(st, T, attend)
        last = torch.from_numpy(cu_q[1:] - 1).to(dev)
        hn = st.xn.index_select(0, last).contiguous()
        logits = torch.empty(B, self.V, device=dev, dtype=dt)
        c.gemm(hn, self.lm_head, logits, epilogue=EPI_NONE)
        return logits

    # ------------------------------------------------------------------------------------------ prefix caching
    def _prefix_clear(self):
        """Invalidation: every weight change bumps the epoch of the key chain and drops the index (pages still in use stay with their
        holders as private pages)."""
        self._prefix_epoch += 1
        if self.enable_prefix_caching:
            self.pool.clear()

    def prefix_cache_stats(self):
        """Prompt positions prefilled through the cache so far, how many of them were hits, the pages in the index, pages evicted."""
        pool = self.pool
        return dict(queried_positions=self._prefix_queried, hit_positions=self._prefix_hits,
                    cached_pages=len(pool.page_of) if self.enable_prefix_caching else 0,
                    evictions=pool.evictions if self.enable_prefix_caching else 0)

    def _alloc_prompt(self, lay, timeseries, extra, lookup=True, spare=0):
        """Pages for the prompts of ``lay`` plus ``extra`` decode positions each: (page_tables, held, keys, cached).  With prefix
        caching on, the leading full pages an earlier prefill indexed are shared (cached = positions per sequence they hold) and keys
        are what _prefix_register indexes once the prefill is enqueued; off, keys and cached are None.  lookup=False: no page is
        shared (every position is computed), the keys are still returned for indexing.  ``spare`` more pages, in no page table, are
        taken in the same all-or-nothing check and are the last ``spare`` entries of held."""
        if not self.enable_prefix_caching:
            return self._alloc_pages(lay.lens, extra, spare) + (None, None)
        cnt = self._host_counts[1].numpy() if lay.row_map.shape[0] > 0 else np.zeros(0, dtype=np.int64)
        seed = prefix_cache.chain_seed(self._merge_mode(), self.page_size, self._prefix_epoch)
        keys = prefix_cache.page_keys(lay, prefix_cache.series_digests(timeseries) if cnt.shape[0] else [], cnt, seed, self.page_size)
        needs = self._page_needs(lay.lens, extra)
        pool, ps = self.pool, self.page_size
        hits = [pool.lookup(keys[b][: (int(n) - 1) // ps]) if lookup else [] for b, n in enumerate(lay.lens)]
        hit_set = {p for h in hits for p in h}
        new = sum(n - len(h) for n, h in zip(needs, hits)) + spare
        # all-or-nothing: hits + free + evictable (minus the evictable pages this batch hits) against the need, before any reference
        avail = len(pool.free) + sum(1 for p in pool.evictable if p not in hit_set)
        if new > avail:
            raise RuntimeError(f"KV cache exhausted: need {new} new pages, {avail} free or evictable of {pool.num_pages}")
        for h in hits:
            pool.acquire(h)
        pt = np.zeros((len(needs), self.max_pages), dtype=np.int32)
        held = []
        for b, (n, h) in enumerate(zip(needs, hits)):
            pages = h + pool.alloc(n - len(h))
            pt[b, :n] = pages
            held += pages
        held += pool.alloc(spare)
        cached = np.array([len(h) * ps for h in hits], dtype=np.int64)
        self._prefix_queried += int(lay.lens.sum())
        self._prefix_hits += int(cached.sum())
        return pt, held, keys, cached

    def _prefix_register(self, keys, page_tables, lens, cached):
        """Indexes the full prompt pages a prefill has just been enqueued to write (later prefills on the stream are ordered after it,
        and prompt pages are never written again).  No-op when prefix caching is off."""
        if keys is None:
            return
        ps = self.page_size
        for b, ks in enumerate(keys):
            for k in range(int(cached[b]) // ps, min(len(ks), int(lens[b]) // ps)):
                self.pool.register(ks[k], int(page_tables[b, k]))

    def _gather_vocab(self, logits):
        if self.tp_size == 1:
            return logits
        parts = [torch.empty_like(logits) for _ in range(self.tp_size)]
        torch.distributed.all_gather(parts, logits, group=self.comm)
        return torch.cat(parts, dim=-1)

    def forward(self, input_ids, attention_mask=None, timeseries=None, logits_to_keep=1, layout_kind="hf", **_):
        """HF-style forward.  layout_kind="hf": input_ids hold the un-expanded <ts><ts/> pairs, patch rows are inserted
        (HF surface); "vllm": one flat prompt whose <ts> copies are overwritten in order (chatts_vllm.py:405-415,569-573).
        logits_to_keep=1 -> [B,1,V] (next-token logits); 0 -> list of per-sample [T_b, V] tensors for every position."""
        _, _, counts, lay = self._prepare_inputs(input_ids, attention_mask, timeseries, layout_kind)
        B = lay.cu_seqlens.shape[0] - 1
        pts, held = self._alloc_pages(lay.lens, 0)
        try:
            logits = self._prefill(lay, counts, timeseries, pts, all_logits=(logits_to_keep == 0))
        finally:
            self.pool.release(held)
        if logits_to_keep == 0:
            cu = lay.cu_seqlens
            return CausalLMOutput([logits[cu[b]:cu[b + 1]] for b in range(B)])
        return CausalLMOutput(logits[:, None, :])

    __call__ = forward

    def _page_needs(self, lens, extra):
        B = len(lens)
        if B > self.max_batch:
            raise ValueError(f"batch {B} exceeds max_batch {self.max_batch}")
        needs = []
        for b in range(B):
            n_tok = int(lens[b]) + extra
            if n_tok > self.n_pos:
                raise ValueError(f"sequence of {n_tok} tokens exceeds the {self.n_pos} positions of the rotary table "
                                 f"(min(max_position_embeddings, max_seq_len))")
            need = (n_tok + self.page_size - 1) // self.page_size
            if need > self.max_pages:
                raise ValueError(f"sequence of {n_tok} tokens exceeds max_seq_len {self.max_seq_len}")
            needs.append(need)
        return needs

    def _alloc_pages(self, lens, extra, spare=0):
        needs = self._page_needs(lens, extra)
        pt = np.zeros((len(needs), self.max_pages), dtype=np.int32)
        # all-or-nothing: every need is checked before the first page leaves the pool, so a failure can never strand pages
        # (ContinuousEngine._admit retries a RuntimeError; a leak there would shrink the pool for good)
        if sum(needs) + spare > self.pool.available():
            raise RuntimeError(f"KV cache exhausted: need {sum(needs) + spare} pages, {self.pool.available()} free of {self.pool.num_pages}")
        held = []
        try:
            for b, need in enumerate(needs):
                pg = self.pool.alloc(need)
                held += pg
                pt[b, :need] = pg
            held += self.pool.alloc(spare)
        except BaseException:
            self.pool.release(held)
            raise
        return pt, held

    # ------------------------------------------------------------------------------------------ decode
    def _decode_state(self, B, max_new):
        key = B
        st = self._steps.get(key)
        if st is not None and st.out_tokens.shape[1] >= max_new:
            return st
        dev = self.device
        st = self._alloc_step(B, decode=True)
        st.B = B
        st.cur_ids = torch.zeros(B, device=dev, dtype=torch.int32)
        st.seq_lens = torch.zeros(B, device=dev, dtype=torch.int32)
        st.page_table = torch.zeros(B, self.max_pages, device=dev, dtype=torch.int32)
        st.out_tokens = torch.zeros(B, max(max_new, 256), device=dev, dtype=torch.int32)
        st.step_ptr = torch.zeros(2, device=dev, dtype=torch.int32)      # {step, arrival counter}
        st.logits = torch.empty(B, self.V, device=dev, dtype=self.dtype)
        # flash-decode split: fill the SMs with (split x kv head x batch) CTAs, at least 2 pages per split
        # (the kernel holds a 3-stage ring of 32 KB K+V tiles: TWO CTAs per SM; sizing for three gave 384 CTAs = two waves at TP2)
        per = max(1, (2 * 148) // max(1, B * self.nkv))
        max_tiles = max(1, (self.max_seq_len + 63) // 64)
        st.attn_splits = int(max(1, min(per, max_tiles, 32)))
        import os
        if os.environ.get("CTS_ATTN_SPLITS"):                      # tuning override
            st.attn_splits = int(os.environ["CTS_ATTN_SPLITS"])
        st.attn_ws = torch.zeros(self.ctx.attn_decode_workspace_floats(B, self.nh, self.d, st.attn_splits), device=dev,
                                 dtype=torch.float32)      # zero-filled once: holds the self-resetting split counters
        st.ssq = torch.zeros(B * 8, device=dev, dtype=torch.float32)
        tiles_h = (self.H + 127) // 128                             # per-tile sums of squares of h (fused decode level 2)
        st.ssq_a = torch.zeros(B, tiles_h, device=dev, dtype=torch.float32)
        st.ssq_b = torch.zeros(B, tiles_h, device=dev, dtype=torch.float32)
        st.chain_sync = torch.zeros(2, device=dev, dtype=torch.int32)       # grid-barrier counters of the chain kernel
        st.graph = st.graph_nosample = None
        self._steps[key] = st
        return st

    def _native_ok(self, B):
        return self.use_native_step and self.tp_size == 1 and B <= 128 and not self._chain_ok(B) and self.w4 is None and self.fp8 is None

    def _chain_ok(self, B):
        return (self.w4 is None and self.fp8 is None and self.use_chain and self.tp_size == 1 and B <= 32 and self.H % 64 == 0 and self.H // 64 <= 192 and self.I % 64 == 0)

    def _decode_layers_chain(self, st, attend):
        """Decode layers with the persistent chain kernel: per layer ONE attention launch + ONE chain launch
        (o_proj -> +resid/norm -> gate_up -> SwiGLU -> down -> +resid/norm -> next QKV -> RoPE/KV write)."""
        c, B, sp = self.ctx, st.B, st.splits
        common = dict(t=B, hidden=self.H, inter=self.I, nh=self.nh, nkv=self.nkv, head_dim=self.d,
                      splits=(sp["o"], sp["gu"], sp["d"], sp["qkv"]), h=st.h, xn=st.xn, act=st.act, ws=st.ws, ssq=st.ssq,
                      sync=st.chain_sync, eps=self.eps, dtype=self.dtype, positions=st.positions, cos=self.cos, sin=self.sin,
                      slot_map=st.slot_map, q_out=st.q, page_size=self.page_size)
        # head: RMSNorm(ln1[0]) -> QKV(0) -> RoPE / KV write(0)
        c.decode_chain(phases=(5, 8), norm5_has_partial=0, ln_next=self.ln1[0], wqkv=self.wqkv[0], bqkv=self.bqkv[0],
                       q_norm_w=self.qn[0], k_norm_w=self.kn[0], k_cache=self.kv[0, 0], v_cache=self.kv[0, 1], **common)
        for l in range(self.L):
            attend(l)
            last = l == self.L - 1
            nxt = {} if last else dict(wqkv=self.wqkv[l + 1], bqkv=self.bqkv[l + 1], q_norm_w=self.qn[l + 1], k_norm_w=self.kn[l + 1],
                                       k_cache=self.kv[l + 1, 0], v_cache=self.kv[l + 1, 1])
            c.decode_chain(phases=(0, 6 if last else 8), wo=self.wo[l], ao=st.ao, ln_post=self.ln2[l], wgu=self.wgu[l], wd=self.wd[l],
                           ln_next=self.final_norm if last else self.ln1[l + 1], **nxt, **common)

    def _decode_body(self, st, sample):
        c, B = self.ctx, st.B
        scale = 1.0 / math.sqrt(self.d)
        if self._native_ok(B):
            if not hasattr(self, "_layer_list"):
                self._layer_list = [dict(wqkv=self.wqkv[l], bqkv=self.bqkv[l], q_norm=self.qn[l], k_norm=self.kn[l], wo=self.wo[l],
                                         wgu=self.wgu[l], wd=self.wd[l], ln1=self.ln1[l], ln2=self.ln2[l], k_cache=self.kv[l, 0],
                                         v_cache=self.kv[l, 1]) for l in range(self.L)]
            sp = st.splits
            c.decoder_step(layers=self._layer_list, embed=self.embed, final_norm=self.final_norm, lm_head=self.lm_head, cos=self.cos,
                           sin=self.sin, hidden=self.H, inter=self.I, nh=self.nh, nkv=self.nkv, head_dim=self.d, eps=self.eps,
                           page_size=self.page_size, batch=B, splits=(sp["qkv"], sp["o"], sp["gu"], sp["d"]), attn_splits=st.attn_splits,
                           cur_ids=st.cur_ids, positions=st.positions, seq_lens=st.seq_lens, slot_map=st.slot_map, page_table=st.page_table,
                           out_tokens=st.out_tokens, step_ptr=st.step_ptr, h=st.h, xn=st.xn, q=st.q, ao=st.ao, act=st.act,
                           logits=st.logits, ws=st.ws, attn_ws=st.attn_ws, sample=sample)
            st.full_logits = st.logits
            return
        c.embed_gather(self.embed, st.cur_ids, st.h, t=B)

        def attend(l):
            c.attn_decode(st.q, self.kv[l, 0], self.kv[l, 1], st.page_table, st.seq_lens, B, self.nh, self.nkv, self.d,
                          self.page_size, scale, st.attn_splits, st.attn_ws, st.ao)

        if self._chain_ok(B):
            self._decode_layers_chain(st, attend)
        else:
            self._layers(st, B, attend)
        nb = self.next_prefetch_bytes if (B <= 32 and self.fp8 is None) else 0
        c.gemm(st.xn, self.lm_head, st.logits, epilogue=EPI_NONE, t=B,
               **(dict(next_w=self.wqkv[0], next_split=st.splits["qkv"], next_bytes=nb) if nb > 0 else {}))
        if sample and self.peer is not None:
            # vocab-parallel greedy over peer memory: no collective call, graph-capturable
            c.peer_greedy_advance(st.logits, B, self.tp_rank, self.tp_size, self.peer.cand, self.peer.cand_flags, self.peer.cand_state,
                                  self.peer.max_batch, st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map,
                                  st.page_table, self.page_size)
            return
        st.full_logits = self._gather_vocab(st.logits)           # identity on one GPU; all-gather of vocab shards under TP
        if sample:
            c.greedy_advance(st.full_logits, B, st.out_tokens, st.step_ptr, st.cur_ids, st.positions, st.seq_lens, st.slot_map,
                             st.page_table, self.page_size)

    def _decode_step(self, st, sample=True):
        """One decode step for the whole batch; replays the captured CUDA graph when enabled."""
        if not self.use_cuda_graph or (self.tp_size > 1 and not (self.graph_with_tp and self.peer is not None and sample)):
            self._decode_body(st, sample)
            return
        attr = "graph" if sample else "graph_nosample"
        g = getattr(st, attr)
        if g is None:
            # warm-up on a side stream (sets kernel attributes, touches every buffer), then capture.  The warm-up
            # step really runs, so save/restore the device-side loop state around it.
            saved = [t.clone() for t in (st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.step_ptr, st.out_tokens)]
            s = torch.cuda.Stream(device=self.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._decode_body(st, sample)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            for t, v in zip((st.cur_ids, st.positions, st.seq_lens, st.slot_map, st.step_ptr, st.out_tokens), saved):
                t.copy_(v)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._decode_body(st, sample)
            setattr(st, attr, g)
            # capture does not execute: state is intact
        g.replay()

    # ------------------------------------------------------------------------------------------ generate
    @torch.no_grad()
    def generate(self, input_ids=None, attention_mask=None, timeseries=None, max_new_tokens=None, max_length=None,
                 do_sample=None, temperature=None, top_p=None, top_k=None, streamer=None, eos_token_id=None, pad_token_id=None,
                 synced_gpus=False, sync_every=16, ignore_eos=False, seed=None, repetition_penalty=None, logprobs=None,
                 prompt_logprobs=None, structured_outputs=None, tokenizer=None, num_beams=None, length_penalty=1.0, early_stopping=False,
                 num_return_sequences=1, num_beam_groups=None, diversity_penalty=None, presence_penalty=0.0, frequency_penalty=0.0,
                 logit_bias=None, allowed_token_ids=None, min_new_tokens=None, **_):
        """model.generate(**processor_out, max_new_tokens=...) -> LongTensor [B, S + new] whose first S columns are
        the ORIGINAL (un-expanded) input ids (README.md:102-103).

        logprobs = k (0..20): every generated token's log probability and rank, and the k most likely tokens with theirs;
        prompt_logprobs = k: the same for every prompt token after the first.  They go to ``self.last_logprobs``
        (chatts_b200.logprobs.GenerationLogprobs; None when neither was asked).  They describe the distribution the token was picked
        from: log_softmax in fp32 of the logits, after the repetition penalty when one is set and before temperature, top-k and top-p
        (vLLM's raw logprobs whenever repetition_penalty == 1).  A call with prompt_logprobs computes every prompt position (no
        prefix-cache hits; its pages are still indexed).  Single GPU only.

        structured_outputs = StructuredOutputsParams or {"choice": [...]} / {"regex": "..."}: every row's output is one of the choices,
        or a full match of the regex (chatts_b200.structured), with ``tokenizer`` giving the bytes of each token id (None: ids < 256 are
        bytes, as SimpleTokenizer encodes).  Each step, the logits of the tokens the automaton does not allow become -inf, and the logprobs
        describe that masked distribution; the stop ids are allowed exactly where the output is complete.  If max_new_tokens runs out first, the output is cut there.  Not with ignore_eos; single
        GPU only.

        num_beams > 1: beam search with transformers' semantics (chatts_b200.beam), ``length_penalty``, ``early_stopping`` (True, False or
        "never") and ``num_return_sequences`` (<= num_beams) as there.  Returns [B * num_return_sequences, S + n], each prompt's best
        hypotheses first, padded with pad_token_id; ``self.last_beam_scores`` holds their scores (transformers' sequences_scores, fp32),
        and is None after any other call.  Greedy only (do_sample, repetition_penalty != 1, logprobs, structured outputs, a streamer
        and tensor parallelism are refused with ValueError), and max(2, 1 + number of EOS ids) * num_beams <= 20.

        presence_penalty, frequency_penalty (each in [-2, 2]), logit_bias ({token id: bias}, clamped to [-100, 100]), allowed_token_ids
        and min_new_tokens (vLLM's min_tokens: the stop ids are refused until a row has generated that many tokens): vLLM's logits
        processors, applied every step together with repetition_penalty (chatts_b200.logit_proc states their order); the logprobs
        describe the processed logits.  Not with beam search or tensor parallelism; allowed_token_ids and min_new_tokens not with
        structured_outputs.  chatts_b200.token_pipeline states the order of the per-step stages."""
        o = resolve_generate(self, input_ids, max_new_tokens=max_new_tokens, max_length=max_length, do_sample=do_sample,
                             temperature=temperature, top_p=top_p, top_k=top_k, streamer=streamer, eos_token_id=eos_token_id,
                             pad_token_id=pad_token_id, ignore_eos=ignore_eos, seed=seed, repetition_penalty=repetition_penalty,
                             logprobs=logprobs, prompt_logprobs=prompt_logprobs, structured_outputs=structured_outputs, tokenizer=tokenizer,
                             num_beams=num_beams, length_penalty=length_penalty, early_stopping=early_stopping,
                             num_return_sequences=num_return_sequences, num_beam_groups=num_beam_groups,
                             diversity_penalty=diversity_penalty, presence_penalty=presence_penalty, frequency_penalty=frequency_penalty,
                             logit_bias=logit_bias, allowed_token_ids=allowed_token_ids, min_new_tokens=min_new_tokens)
        self.last_logprobs = self.last_beam_scores = None
        if o.beams is not None:
            return self._beam_generate(input_ids, attention_mask, timeseries, o.max_new_tokens, sorted(o.eos), o.pad, int(num_beams),
                                       o.beams, length_penalty, early_stopping, int(num_return_sequences), sync_every)
        ids_cpu, am_cpu, counts, lay = self._prepare_inputs(input_ids, attention_mask, timeseries)
        B, S = ids_cpu.shape
        max_new_tokens, eos_set, V, dev = o.max_new_tokens, o.eos, self.config.vocab_size, self.device
        if max_new_tokens <= 0:
            return torch.as_tensor(ids_cpu, dtype=torch.long)
        page_tables, held, keys, cached = self._alloc_prompt(lay, timeseries, max_new_tokens, lookup=o.prompt_logprobs is None)
        try:
            with span("cts.prefill"):
                logits = self._prefill(lay, counts, timeseries, page_tables, cached=cached, prompt_lp=o.prompt_logprobs)
            plp = None
            if o.prompt_logprobs is not None:
                logits, plp = logits
            self._prefix_register(keys, page_tables, lay.lens, cached)
            self.last_cached_positions = cached          # per row: prompt positions whose KV came from the prefix cache (None: caching off)
            st = self._decode_state(B, max_new_tokens)
            lens32 = torch.from_numpy(lay.lens.astype(np.int32))
            st.page_table.copy_(torch.from_numpy(page_tables), non_blocking=True)
            st.positions.copy_(lens32 - 1, non_blocking=True)       # advanced to len by the first token's advance
            st.seq_lens.copy_(lens32, non_blocking=True)             # -> len + 1: cache length once the new token is written
            st.step_ptr.zero_()
            pipe = TokenPipeline(
                self.ctx, st, B, self.page_size, sampling=o.sampling,
                automaton=None if o.automaton is None else (o.automaton, torch.zeros(B, dtype=torch.int32, device=dev)),
                processors=generate_processors(self.ctx, o.procs, ids_cpu, am_cpu, eos_set, V, self.n_pos, dev),
                logprobs=None if o.logprobs is None else (lpmod.LogprobBuffers(self.ctx, B, max_new_tokens, o.logprobs, V, dev), o.logprobs))
            pipe.step(logits)
            done = np.zeros(B, dtype=bool)
            out = np.full((B, max_new_tokens), o.pad, dtype=np.int64)
            emitted = 0
            produced = 1
            chunk = 1 if streamer is not None else max(1, int(sync_every))
            while True:
                # flush what has been produced since the last sync
                if produced - emitted >= chunk or produced >= max_new_tokens:
                    toks = st.out_tokens[:, emitted:produced].cpu().numpy()      # D2H (sync)
                    for j in range(toks.shape[1]):
                        col = toks[:, j]
                        out[~done, emitted + j] = col[~done]
                        if streamer is not None:
                            streamer.put(torch.as_tensor(col))
                        done |= np.isin(col, list(eos_set))
                    emitted = produced
                    if produced >= max_new_tokens or done.all():
                        break
                with span("cts.decode_step"):
                    self._decode_step(st, sample=pipe.fused)
                    pipe.step()
                produced += 1
            if streamer is not None:
                streamer.end()
        finally:
            self.pool.release(held)
        is_eos = np.isin(out[:, :emitted], list(eos_set))
        first = np.where(is_eos.any(axis=1), is_eos.argmax(axis=1) + 1, emitted)
        n_out = int(min(max(first.max(), 1), max_new_tokens))
        if o.logprobs is not None or o.prompt_logprobs is not None:
            res = lpmod.GenerationLogprobs()
            if pipe.lpb is not None:
                res.logprobs, res.ranks, res.top_ids, res.top_logprobs = pipe.lpb.host(n_out)
                if o.automaton is not None:               # a token the constraint refused has probability 0: an empty top-k slot
                    gone = np.isneginf(res.top_logprobs)
                    res.top_ids[gone], res.top_logprobs[gone] = -1, np.nan
            if plp is not None:
                tgt, rows, cols, pbuf = plp
                res.prompt = lpmod.prompt_entries(ids_cpu, am_cpu, rows, cols, tgt, *(a[:, 0] for a in pbuf.host(1)))
            self.last_logprobs = res
        return torch.cat([torch.as_tensor(ids_cpu, dtype=torch.long), torch.as_tensor(out[:, :n_out])], dim=1)

    def _beam_generate(self, input_ids, attention_mask, timeseries, max_new, eos_ids, pad, nb, keep, length_penalty, early_stopping, nrs,
                       sync_every):
        """Beam search (see generate): one prefill per prompt, then every step the decode step of the B * nb beam rows (graph replay
        without the advance), cts_logprobs for each row's top ``keep`` candidates, cts_beam_select and cts_beam_fork_kv, all on one
        stream; the host reads the per-prompt done flags every ``sync_every`` steps and walks the back-pointers once at the end."""
        c, dev, ps = self.ctx, self.device, self.page_size
        ids_cpu, am_cpu, counts, lay = self._prepare_inputs(input_ids, attention_mask, timeseries)
        B, S = ids_cpu.shape
        if max_new <= 0:
            return torch.as_tensor(ids_cpu, dtype=torch.long).repeat_interleave(nrs, 0)
        R, V = B * nb, self.config.vocab_size
        needs = self._page_needs(lay.lens, max_new)
        n_extra = beammod.extra_pages(lay.lens, needs, nb, ps)
        page_tables, held, keys, cached = self._alloc_prompt(lay, timeseries, max_new, spare=n_extra)
        try:
            table, own, spare = beammod.page_plan(page_tables, lay.lens, needs, nb, ps, held[len(held) - n_extra:])
            with span("cts.prefill"):
                logits = self._prefill(lay, counts, timeseries, page_tables, cached=cached)
            self._prefix_register(keys, page_tables, lay.lens, cached)
            self.last_cached_positions = cached
            st = self._decode_state(R, max_new)
            lens = np.repeat(lay.lens.astype(np.int32), nb)
            run = np.zeros((B, nb), dtype=np.float32)
            run[:, 1:] = -1e9
            eos_arr = np.asarray(eos_ids, dtype=np.int32)
            ints = np.concatenate([table.reshape(-1), own.reshape(-1), spare, lens - 1, lens, eos_arr]).astype(np.int32)
            d_int = torch.from_numpy(ints).pin_memory().to(dev, non_blocking=True)
            o = 0

            def take(n):
                nonlocal o
                o += n
                return d_int[o - n:o]
            st.page_table.copy_(take(R * self.max_pages).view(R, self.max_pages))
            own_d, spare_d = take(R * self.max_pages), take(R)
            st.positions.copy_(take(R))                              # advanced to len by step 0's selection
            st.seq_lens.copy_(take(R))
            eos_d = take(len(eos_ids))
            floats = np.concatenate([run.reshape(-1), np.full(R, -1e9, dtype=np.float32), beammod.len_den(max_new, length_penalty)])
            d_f = torch.from_numpy(floats).pin_memory().to(dev, non_blocking=True)
            run_d, fin_scores, den_d = d_f[:R], d_f[R:2 * R], d_f[2 * R:]
            fin_info = torch.zeros(R, 4, dtype=torch.int32, device=dev)
            flags = torch.zeros(B, 2, dtype=torch.int32, device=dev)
            flags[:, 0] = 1                                          # early-stop heuristic unsatisfied, not done
            bstep = torch.zeros(2, dtype=torch.int32, device=dev)
            bp_tok = torch.zeros(max_new, R, dtype=torch.int32, device=dev)
            bp_par = torch.zeros(max_new, R, dtype=torch.int32, device=dev)
            table_old = torch.zeros_like(st.page_table)
            fork = torch.zeros(R, 3, dtype=torch.int32, device=dev)
            cand_ids = torch.zeros(R, 1, keep, dtype=torch.int32, device=dev)
            cand_lp = torch.zeros(R, 1, keep, dtype=torch.float32, device=dev)
            lp_ws = torch.empty(max(c.logprobs_workspace_floats(R, V, keep), 2), dtype=torch.float32, device=dev)
            lp_cnt = torch.zeros(R, dtype=torch.int32, device=dev)

            def select(lg):
                c.logprobs(lg, R, None, keep, None, None, cand_ids, cand_lp, lp_ws, lp_cnt, vocab=V)
                c.beam_select(B, nb, keep, V, cand_ids, cand_lp, eos_d, den_d, max_new, early_stopping, length_penalty, run_d,
                              fin_scores, fin_info, flags, bstep, bp_tok, bp_par, st.cur_ids, st.positions, st.seq_lens, st.slot_map,
                              st.page_table, table_old, own_d, spare_d, ps, fork)
                c.beam_fork_kv(self.kv, fork, R)

            select(logits[:, :V].repeat_interleave(nb, 0))          # step 0: every beam row sees its prompt's prefill logits
            produced, chunk = 1, max(1, int(sync_every))
            while produced < max_new:
                if produced % chunk == 0 and bool(flags[:, 1].all()):
                    break
                with span("cts.decode_step"):
                    self._decode_step(st, sample=False)
                    select(st.full_logits)
                produced += 1
            toks, pars = bp_tok[:produced].cpu().numpy(), bp_par[:produced].cpu().numpy()
            scores, info = fin_scores.cpu().numpy(), fin_info.cpu().numpy()
        finally:
            self.pool.release(held)
        hyps = [beammod.hypothesis(toks, pars, info[b * nb + i]) for b in range(B) for i in range(nrs)]
        n = max(max(len(h) for h in hyps), 1)
        out = np.full((B * nrs, S + n), pad, dtype=np.int64)
        out[:, :S] = np.repeat(ids_cpu, nrs, axis=0)
        for r, h in enumerate(hyps):
            out[r, S:S + len(h)] = h
        self.last_beam_scores = torch.from_numpy(np.stack([scores[b * nb:b * nb + nrs] for b in range(B)]).reshape(-1).copy())
        return torch.from_numpy(out)
