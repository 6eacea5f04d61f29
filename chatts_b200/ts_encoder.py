"""Value-Preserved Time-Series Encoder on H100 -- host mirror of ``TimeSeriesEmbedding``
(chatts/vllm/chatts_vllm.py:61-193): same constructor config, same ``forward(x) -> (feats, patch_cnt)``
contract, same error behaviour; the arithmetic runs in the sm_90a kernels behind the C-ABI
(cts_ts_patch_count, cts_ts_patchify, cts_gemm [+ cts_reduce_bias_act]).

One device->host copy of N int32 pairs per call (valid_len, patch_cnt) replaces the reference's 2-3 syncs
PER SERIES (:108-109,146); the host needs the counts to size the merged sequence.
"""
import torch

from . import _cabi
from ._cabi import EPI_GELU, EPI_NONE, EPI_PARTIAL_F32


class TimeSeriesEmbedding:
    def __init__(self, config, weights, device="cuda", dtype=torch.bfloat16, prefix="ts_encoder."):
        """config: the ``ts`` dict of the checkpoint config (chatts_vllm.py:64-71).  weights: name->tensor."""
        self.patch_size = int(config["patch_size"])
        self.num_layers = int(config["num_layers"])
        self.hidden_size = int(config["hidden_size"])
        self.num_features = int(config["num_features"])
        self.max_sequence_length = int(config["max_sequence_length"])     # required, like :68
        self.use_position_embedding = bool(config.get("use_position_embedding", False))
        self.use_position_idx = bool(config.get("use_position_idx", False))
        self.embedding_dim = int(config.get("embedding_dim", 16))
        self.device, self.dtype = torch.device(device), dtype
        if self.use_position_embedding:
            self.mode, self.input_size = 1, self.patch_size * (1 + self.embedding_dim)
            self.padding_idx = self.max_sequence_length                    # :76
            self.pos_table = weights[prefix + "position_embedding.weight"].to(self.device, dtype).contiguous()
        elif self.use_position_idx:
            self.mode, self.input_size, self.pos_table = 2, 2 * self.patch_size, None
        else:
            self.mode, self.input_size, self.pos_table = 0, self.patch_size, None
        self.w, self.b = [], []
        for li in range(self.num_layers):
            w = weights[f"{prefix}mlp.{2 * li}.weight"].to(self.device, dtype)
            if w.shape[1] % 8 != 0:
                raise _cabi.CtsError(f"TS-encoder layer {li}: input width {w.shape[1]} is not a multiple of 8 "
                                     "(TMA needs a 16-byte row pitch)")
            self.w.append(w.contiguous())
            self.b.append(weights[f"{prefix}mlp.{2 * li}.bias"].to(self.device, dtype).contiguous())
        self.ctx = _cabi.get_context(self.device)
        import os
        # prompts of up to 256 patch rows run as ONE launch (csrc/ts_encoder_fused.cu); CTS_TS_FUSED=0 keeps the multi-launch path
        self.use_fused = os.environ.get("CTS_TS_FUSED", "1") != "0" and hasattr(self.ctx, "ts_mlp_fused")

    # -- A3: patch counts -------------------------------------------------------------------------
    def patch_counts(self, x):
        """(valid_len, patch_cnt, row_offset, max_valid) device int32 tensors; no sync."""
        x = self._prep(x)
        return (x,) + self.ctx.ts_patch_count(x, self.num_features, self.patch_size)

    def _prep(self, x):
        if x.device != self.device or x.dtype != self.dtype:
            x = x.to(self.device, self.dtype)
        n = x.shape[0]
        return x.reshape(n, -1).contiguous()

    # -- A4..A7 -------------------------------------------------------------------------------------
    def encode(self, x, out=None, row_map=None, counts=None, host_counts=None):
        """Encode all series of ``x`` [N, 2L, 1].  Rows are written to ``out[row_map[r]]`` when given (the
        merged embedding sequence), else to a fresh [sum P, H] tensor.  Returns (feats_or_None, patch_cnt_cpu).
        ``host_counts`` = (valid_len, patch_cnt) CPU tensors from an earlier copy: skips the device->host sync."""
        if counts is None:
            counts = self.patch_counts(x)
        x, valid, cnt, off, mx = counts
        n = x.shape[0]
        if host_counts is None:
            host = torch.stack([valid, cnt]).cpu()             # the one sync of the call
            valid_h, cnt_h = host[0], host[1]
        else:
            valid_h, cnt_h = host_counts
        total = int(cnt_h.sum())
        if self.mode != 1 and bool(((valid_h % self.patch_size) != 0).any()):
            # reference behaviour: self.padding_idx is read at :128 but defined only under
            # use_position_embedding (:76) -> AttributeError for ragged lengths
            raise AttributeError("'TimeSeriesEmbedding' object has no attribute 'padding_idx'")
        if self.mode == 1 and n > 0 and int(valid_h.max()) > self.max_sequence_length:
            # reference behaviour: position ids 0..valid-1 index nn.Embedding(max_sequence_length + 1, emb) (chatts_vllm.py:76-80,
            # 119,163-165) -> IndexError for a series longer than the table; the kernel must never read past pos_table
            raise IndexError(f"index out of range in self: series of {int(valid_h.max())} points exceeds "
                             f"max_sequence_length {self.max_sequence_length} of the position embedding")
        if total == 0:
            feats = torch.empty(0, self.hidden_size, device=self.device)      # :191 (default dtype)
            return (feats if out is None else None), cnt_h.to(torch.int64)
        if self.use_fused and total <= 256:
            # metric-sized prompts (8 series x 256 points = 128 rows): patchify + MLP + row scatter in ONE launch (csrc/ts_encoder_fused.cu)
            dst = out if out is not None else torch.empty(total, self.hidden_size, device=self.device, dtype=self.dtype)
            if self.ctx.ts_mlp_fused(x, self.num_features, self.patch_size, self.mode, self.pos_table, self.embedding_dim,
                                     self.max_sequence_length, self.w, self.b, valid, off, mx, total, dst,
                                     row_map=row_map if out is not None else None):
                return (None if out is not None else dst), cnt_h.to(torch.int64)
        row_len = x.shape[1]
        max_patches = (row_len // self.num_features + self.patch_size - 1) // self.patch_size
        rows = torch.empty(total, self.input_size, device=self.device, dtype=self.dtype)
        self.ctx.ts_patchify(x, self.num_features, self.patch_size, self.mode, self.pos_table, self.embedding_dim,
                             self.max_sequence_length, valid, off, mx, max_patches, rows)
        h = rows
        feats = None
        for li in range(self.num_layers):
            last = li == self.num_layers - 1
            w, b = self.w[li], self.b[li]
            if last and out is not None:
                dst, rmap = out, row_map
            else:
                dst, rmap = torch.empty(total, self.hidden_size, device=self.device, dtype=self.dtype), None
            act = EPI_NONE if last else EPI_GELU
            split = self.ctx.suggest_split(w.shape[0], w.shape[1], total)
            if split > 1:
                part = torch.empty(split, total, w.shape[0], device=self.device, dtype=torch.float32)
                self.ctx.gemm(h, w, part, epilogue=EPI_PARTIAL_F32, split_k=split)
                self.ctx.reduce_bias_act(part, split, total, w.shape[0], b, act, dst, rmap)
            else:
                self.ctx.gemm(h, w, dst, bias=b, row_map=rmap, epilogue=act)
            h = dst
            if last and out is None:
                feats = dst
        return feats, cnt_h.to(torch.int64)

    def forward(self, x):
        """chatts_vllm.py:93-193: x [N, 2L, 1] -> (feats [sum P, H], patch_cnt [N] int64 on the device)."""
        feats, cnt = self.encode(x)
        return feats, cnt.to(self.device)

    __call__ = forward


def get_patch_cnt(x, ts_config):
    """chatts_vllm.py:198-207 on the device (no MLP): int64 patch counts."""
    n = x.shape[0]
    xx = x.reshape(n, -1).contiguous()
    if xx.dtype not in (torch.bfloat16, torch.float16):
        xx = xx.to(torch.bfloat16)
    ctx = _cabi.get_context(xx.device)
    _, cnt, _, _ = ctx.ts_patch_count(xx, int(ts_config["num_features"]), int(ts_config["patch_size"]))
    return cnt.to(torch.int64)
