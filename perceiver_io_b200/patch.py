"""In-place swap of the attention arithmetic inside an already constructed *reference* model.

``patch(model)`` rebinds ``forward`` of every reference ``MultiHeadAttention`` instance
(/root/reference/perceiver/model/core/modules.py:23) to this package's implementation.  Parameters,
sub-module names and everything above L1 (layers, encoder/decoder, Lightning / 🤗 wrappers) stay the
reference's own objects, so checkpoints, optimizers and FSDP wrap policies are untouched.
"""
from __future__ import annotations

import types

from torch import nn

from .modules import CrossAttention, MultiHeadAttention, SelfAttention

_REQUIRED = ("q_proj", "k_proj", "v_proj", "o_proj", "dp_scale", "num_heads", "causal_attention", "dropout")


def _is_reference_mha(module: nn.Module) -> bool:
    return type(module).__name__ == "MultiHeadAttention" and all(hasattr(module, a) for a in _REQUIRED)


def _is_reference_cross_attention(module: nn.Module) -> bool:
    return (type(module).__name__ == "CrossAttention" and not isinstance(module, CrossAttention)
            and all(hasattr(module, a) for a in ("q_norm", "kv_norm", "attention")))


def _is_reference_self_attention(module: nn.Module) -> bool:
    return (type(module).__name__ == "SelfAttention" and not isinstance(module, SelfAttention)
            and all(hasattr(module, a) for a in ("norm", "attention")))


def patch(model: nn.Module, impl: str = "auto") -> int:
    """Route every MultiHeadAttention under ``model`` through the sm_90a kernels.

    Reference ``CrossAttention`` / ``SelfAttention`` modules (modules.py:173-278) are rebound as well so that their
    LayerNorm -> projection chains run through the LayerNorm-folded tcgen05 GEMM (``modules.project_kv`` /
    ``modules.project_qkv``).
    Returns the number of attention modules rebound; idempotent."""
    count = 0
    for module in model.modules():
        if isinstance(module, MultiHeadAttention):
            module.kernel_impl = impl
            continue
        if _is_reference_mha(module):
            module.kernel_impl = impl
            module.forward = types.MethodType(MultiHeadAttention.forward, module)
            count += 1
        elif _is_reference_cross_attention(module):
            module.forward = types.MethodType(CrossAttention.forward, module)
        elif _is_reference_self_attention(module):
            module.forward = types.MethodType(SelfAttention.forward, module)
    return count
