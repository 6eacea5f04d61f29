"""chatts_b200 -- H100-native (sm_90a) hot path of ChatTS: the Value-Preserved Time-Series Encoder and the
Qwen2 decoder forward behind the reference's processor / ``<ts>`` protocol / generate() surface.

Importing the package is GPU-free (config, layout, processor are host logic); anything that computes goes through
libchatts_b200.so and raises if the library or an H100 is missing -- there is no fallback path."""
from .config import ChatTSConfig
from .processor import ChatTSProcessor, SimpleTokenizer, sp_encoding

__all__ = ["ChatTSConfig", "ChatTSProcessor", "SimpleTokenizer", "sp_encoding", "ChatTSForCausalLM", "TimeSeriesEmbedding"]


def __getattr__(name):
    if name == "ChatTSForCausalLM":
        from .model import ChatTSForCausalLM
        return ChatTSForCausalLM
    if name == "TimeSeriesEmbedding":
        from .ts_encoder import TimeSeriesEmbedding
        return TimeSeriesEmbedding
    raise AttributeError(name)
