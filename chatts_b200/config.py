"""Model configuration, read from the checkpoint's config.json (never hard-coded: SURVEY.md §2.2 dagger).

Mirrors what the reference reads: ``config.ts[...]`` and ``config.ts_token_start_index``
(chatts/vllm/chatts_vllm.py:64-71,376,384,441) on top of the stock Qwen2 fields."""
import json
import os
from dataclasses import dataclass, field, asdict


def _default_ts():
    return dict(patch_size=16, num_layers=5, hidden_size=5120, num_features=2, max_sequence_length=4096,
                use_position_embedding=True, use_position_idx=False, embedding_dim=16)


@dataclass
class ChatTSConfig:
    hidden_size: int = 5120
    intermediate_size: int = 13824
    num_hidden_layers: int = 48
    num_attention_heads: int = 40
    num_key_value_heads: int = 8
    head_dim: int = 128
    vocab_size: int = 152064
    rms_norm_eps: float = 1e-6
    rope_theta: float = 1e6
    max_position_embeddings: int = 32768
    tie_word_embeddings: bool = False
    attention_bias: bool = True                 # Qwen2: q/k/v bias; Qwen3 (ChatTS-8B): none
    qk_norm: bool = False                       # Qwen3 (ChatTS-8B): per-head RMSNorm of q and k before RoPE
    ts: dict = field(default_factory=_default_ts)
    ts_token_start_index: int = 151665          # <ts>; <ts/> = +1 (chatts_vllm.py:441)
    eos_token_id: int = 151645                  # stop ids 151643/151645 (chatts/utils/llm_utils.py:153)
    pad_token_id: int = 151643
    # HF-surface merge of the patch rows at <ts><ts/> (layout.py): "insert" keeps both special tokens, "overwrite" replaces the pair.
    # The checkpoint's remote code is not in the reference repo, so this cannot be pinned offline (INTEGRATION.md).
    ts_merge_mode: str = "insert"
    model_type: str = "chatts"                  # scripts/start_vllm_server.sh:5
    torch_dtype: str = "bfloat16"

    @property
    def ts_token_end_index(self):
        return self.ts_token_start_index + 1

    @classmethod
    def chatts_14b(cls):
        """Public Qwen2.5-14B shape + the TS encoder of the released ChatTS-14B (UNVERIFIED offline; a real
        checkpoint's config.json overrides every field through from_json)."""
        return cls()

    @classmethod
    def chatts_8b(cls):
        """ChatTS-8B = Qwen3-8B decoder (Qwen3TSForCausalLM, chatts_vllm.py:633-668) + the TS encoder at hidden 4096
        (public Qwen3-8B shape; UNVERIFIED offline, config.json overrides)."""
        ts = _default_ts()
        ts["hidden_size"] = 4096
        return cls(hidden_size=4096, intermediate_size=12288, num_hidden_layers=36, num_attention_heads=32,
                   num_key_value_heads=8, head_dim=128, vocab_size=151936, rms_norm_eps=1e-6, rope_theta=1e6,
                   max_position_embeddings=40960, attention_bias=False, qk_norm=True, ts=ts, ts_token_start_index=151669)

    @classmethod
    def tiny(cls, **kw):
        """Small shape for parity tests (head_dim 64, GQA 2:1, ragged K/N on purpose)."""
        d = dict(hidden_size=256, intermediate_size=704, num_hidden_layers=2, num_attention_heads=4,
                 num_key_value_heads=2, head_dim=64, vocab_size=1000, max_position_embeddings=2048,
                 ts=dict(patch_size=16, num_layers=3, hidden_size=256, num_features=2, max_sequence_length=512,
                         use_position_embedding=True, use_position_idx=False, embedding_dim=16),
                 ts_token_start_index=990, eos_token_id=998, pad_token_id=999)
        d.update(kw)
        return cls(**d)

    @classmethod
    def from_dict(cls, d):
        known = {k: d[k] for k in cls.__dataclass_fields__ if k in d}
        cfg = cls(**known)
        if "head_dim" not in d or d.get("head_dim") is None:
            cfg.head_dim = cfg.hidden_size // cfg.num_attention_heads
        if "rope_parameters" in d and isinstance(d["rope_parameters"], dict):
            cfg.rope_theta = d["rope_parameters"].get("rope_theta", cfg.rope_theta)
        arch = " ".join(d.get("architectures", []) or [])
        if "Qwen3" in arch or d.get("model_type") in ("qwen3", "chatts_qwen3"):
            cfg.qk_norm = d.get("qk_norm", True)
            cfg.attention_bias = bool(d.get("attention_bias", False))
        if isinstance(cfg.eos_token_id, (list, tuple)):
            cfg.eos_token_id = int(cfg.eos_token_id[0])
        return cfg

    @classmethod
    def from_json(cls, path):
        if os.path.isdir(path):
            path = os.path.join(path, "config.json")
        with open(path) as f:
            return cls.from_dict(json.load(f))

    def to_dict(self):
        return asdict(self)

    def ts_input_size(self):
        """chatts_vllm.py:73-81."""
        p = self.ts["patch_size"]
        if self.ts.get("use_position_embedding", False):
            return p + self.ts.get("embedding_dim", 16) * p
        if self.ts.get("use_position_idx", False):
            return 2 * p
        return p

    def ts_mode(self):
        if self.ts.get("use_position_embedding", False):
            return 1
        if self.ts.get("use_position_idx", False):
            return 2
        return 0
