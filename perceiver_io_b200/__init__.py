"""perceiver_io_b200 — B200 (sm_100a) latent-attention hot path for Perceiver / Perceiver IO /
Perceiver AR, behind the reference's own ``nn.Module`` interface.

Layout (tier scope: SURVEY.md §8 only):
  csrc/        CUDA kernels + the C-ABI (``include/pcv_attn.h``) -> ``lib/libpcv_attn.so``
  _lib.py      ctypes binding of the C-ABI (raises if the library is missing; no fallback)
  ops.py       tensor-level wrappers (attention, partial/merge, rotary, kv-append)
  modules.py   ``MultiHeadAttention`` ... ``PerceiverAR`` / ``CausalSequenceModel`` mirrors
  position.py / adapter.py / utils.py / config.py   the small pieces those modules need
  dist.py      M-sharded cross-attention across the GPUs of one box
  patch.py     swap the attention arithmetic inside an already-built reference model
  streaming.py host-resident K/V input pipelined against PCIe;  graphs.py  CUDA-graph capture of static-shape forwards
  generation.py  graph-replayed Perceiver AR decoding (GraphedDecoder: one generated token = one graph replay)
"""
from .utils import ModuleOutput, Residual, init_parameters, freeze  # noqa: F401
from .position import positions, RotaryPositionEmbedding, FrequencyPositionEncoding  # noqa: F401
from .modules import (  # noqa: F401
    KVCache,
    MultiHeadAttention,
    CrossAttention,
    SelfAttention,
    AbstractAttentionLayer,
    CrossAttentionLayer,
    SelfAttentionLayer,
    SelfAttentionBlock,
    MLP,
    PerceiverEncoder,
    PerceiverDecoder,
    PerceiverIO,
    PerceiverAR,
    CausalSequenceModel,
)
from .config import PerceiverARConfig, CausalSequenceModelConfig  # noqa: F401
from .patch import patch  # noqa: F401
from .generation import GraphedDecoder, decode_windows, speculative_budget, speculative_generate  # noqa: F401

__version__ = "0.1.0"
