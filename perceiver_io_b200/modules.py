"""Host-side mirror of the reference's attention building blocks and architectures
(/root/reference/perceiver/model/core/modules.py) with the attention arithmetic replaced by the
sm_100a kernels behind ``include/pcv_attn.h``.

Drop-in contract (SURVEY.md §8(b), level 1): class names, constructor and ``forward`` signatures,
``ModuleOutput`` return type, attribute names read by callers (``q_proj`` ... ``o_proj``,
``dp_scale``, ``num_qk_channels`` ...) and ``state_dict`` keys are those of the reference, so its
Lightning / 🤗 wrappers and checkpoints work on these modules unchanged.  What differs is *how*
``MultiHeadAttention.forward`` computes (reference lines cited inline):

  reference (modules.py:113-170)                      here
  --------------------------------------------------  ------------------------------------------------
  q/k/v/o nn.Linear                                   same (cuBLAS; not on the M-proportional path §8(f)1)
  torch.cat onto the cache                 :117-121   ops.kv_append (one launch for K and V)
  rearrange to (b h n c)                   :123       strides only, never materialised
  q * dp_scale                             :124       folded into the softmax exponent
  rotary on q / k (cos/sin temporaries)    :126-130   ops.rotary (pcv_rotary_apply)
  einsum, 2x masked_fill_, softmax, einsum :146-164   ops.attention (pcv_attn_fwd, online softmax,
                                                      scores never leave the SM)
  max_heads_parallel chunk loop            :144-150   accepted, no effect (nothing to bound)

Inputs must be CUDA tensors; there is no CPU implementation in this package.
"""
from __future__ import annotations

from typing import List, NamedTuple, Optional, Tuple

import torch
from torch import nn

from . import ops
from .adapter import (InputAdapter, OutputAdapter, QueryProvider, RotarySupport, TiedTokenOutputAdapter,
                      TokenInputAdapterWithRotarySupport, TrainableQueryProvider)
from .config import CausalSequenceModelConfig
from .position import RotaryPositionEmbedding, positions
from .utils import ModuleOutput, Residual, init_parameters

KVCache = Tuple[torch.Tensor, torch.Tensor]


def _rotate_qk(num_heads: int, q: torch.Tensor, k: torch.Tensor, rot_q, rot_k, cache_k=None, k_descale=None, **shadow):
    """``(q, k, from_shadow)``: q and k (B, n, H*d) as the attention takes them after the rotary embedding.

    With ``cache_k`` (the cache's keys after this call's append) both come from the rotated-key shadow
    (``ops.rotated_cache_keys``: keys are rotated once, when they enter the cache) when it can serve: both rotary objects
    right-aligned and the key one carrying its frequency table ``inv_freq``, as this package's models pass it.
    Otherwise each is rotated by its own rotary object, this package's ``RotaryPositionEmbedding`` or any object with the
    reference's attributes (``frq_pos_enc`` (B,1,n,f), ``right_align``); e4m3 keys with their per-head ``k_descale``,
    e4m3 to e4m3 (``ops.rotary_fp8``)."""
    if (cache_k is not None and rot_q is not None and getattr(rot_k, "inv_freq", None) is not None
            and bool(rot_q.right_align) and bool(rot_k.right_align)):
        hit = ops.rotated_cache_keys(cache_k, q, num_heads, rot_k.inv_freq, k_descale=k_descale, **shadow)
        if hit is not None:
            return hit[0], hit[1], True
    if rot_q is not None:
        q = ops.rotary(q, num_heads, rot_q.frq_pos_enc, bool(rot_q.right_align))
    if rot_k is not None and k.dtype == ops.F8:
        k = ops.rotary_fp8(k, num_heads, rot_k.frq_pos_enc, bool(rot_k.right_align), k_descale)
    elif rot_k is not None:
        k = ops.rotary(k, num_heads, rot_k.frq_pos_enc, bool(rot_k.right_align))
    return q, k, False


class MultiHeadAttention(nn.Module):
    """Multi-head attention with asymmetric query/key lengths, separate qk/v widths, key padding
    mask, right-aligned causal mask, rotary embeddings and a functional KV cache
    (reference modules.py:23-170)."""

    def __init__(
        self,
        num_heads: int,
        num_q_input_channels: int,
        num_kv_input_channels: int,
        num_qk_channels: Optional[int] = None,
        num_v_channels: Optional[int] = None,
        num_output_channels: Optional[int] = None,
        max_heads_parallel: Optional[int] = None,
        causal_attention: bool = False,
        dropout: float = 0.0,
        qkv_bias: bool = True,
        out_bias: bool = True,
    ):
        super().__init__()
        num_qk_channels = num_q_input_channels if num_qk_channels is None else num_qk_channels
        num_v_channels = num_qk_channels if num_v_channels is None else num_v_channels
        num_output_channels = num_q_input_channels if num_output_channels is None else num_output_channels

        if num_qk_channels % num_heads != 0:
            raise ValueError("num_qk_channels must be divisible by num_heads")
        if num_v_channels % num_heads != 0:
            raise ValueError("num_v_channels must be divisible by num_heads")

        self.dp_scale = (num_qk_channels // num_heads) ** -0.5
        self.num_heads = num_heads
        self.num_qk_channels = num_qk_channels
        self.num_v_channels = num_v_channels
        self.causal_attention = causal_attention
        # kept for interface parity; the fused kernel has no (B,h,N,M) tensor to chunk
        self.max_heads_parallel = num_heads if max_heads_parallel is None else max_heads_parallel

        self.q_proj = nn.Linear(num_q_input_channels, num_qk_channels, bias=qkv_bias)
        self.k_proj = nn.Linear(num_kv_input_channels, num_qk_channels, bias=qkv_bias)
        self.v_proj = nn.Linear(num_kv_input_channels, num_v_channels, bias=qkv_bias)
        self.o_proj = nn.Linear(num_v_channels, num_output_channels, bias=out_bias)
        self.dropout = nn.Dropout(dropout)
        self.kernel_impl = "auto"  # "auto" | "tcgen05" | "simt" (testing aid)

    def forward(
        self,
        x_q: torch.Tensor,
        x_kv: torch.Tensor,
        pad_mask: Optional[torch.Tensor] = None,
        rot_pos_emb_q: Optional[RotaryPositionEmbedding] = None,
        rot_pos_emb_k: Optional[RotaryPositionEmbedding] = None,
        kv_cache: Optional[KVCache] = None,
    ):
        """x_q (B|1, N, D), x_kv (B, L, C), pad_mask (B, L_total) bool with True = padding.
        Returns ``ModuleOutput(last_hidden_state=(B, N, F), kv_cache=(k, v) | None)``; cached k/v are
        (B, L_total, channels), un-rotated and pre-head-split exactly like the reference's."""
        q = self.q_proj(x_q)
        k = self.k_proj(x_kv)
        v = self.v_proj(x_kv)
        return attend(self, q, k, v, pad_mask, rot_pos_emb_q, rot_pos_emb_k, kv_cache)


def attend(mha, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, pad_mask=None, rot_pos_emb_q=None,
           rot_pos_emb_k=None, kv_cache: Optional[KVCache] = None, min_rows_key: str = "min_rows", kv8=None):
    """Everything of ``MultiHeadAttention.forward`` after the q/k/v projections (reference modules.py:117-170):
    cache append, rotary, fused attention, ``o_proj``.  ``mha`` is this package's module or a patched reference
    one (only its attributes are used).  ``kv8``: the scales of an FP8 KV cache (``_kv8_route``)."""
    if kv8 is not None:
        return _attend_kv8(mha, q, k, v, pad_mask, rot_pos_emb_q, rot_pos_emb_k, kv_cache, min_rows_key, kv8)
    # attention-probability dropout (reference :161): fused into the training kernels (ops.attention dropout_p)
    drop_p = float(mha.dropout.p) if mha.training else 0.0
    if kv_cache is not None:
        k, v = ops.kv_append(kv_cache[0], kv_cache[1], k, v)
        kv_cache = (k, v)

    # the shadow has no autograd: rows that need a gradient are rotated by the rotary objects
    shadow = kv_cache is not None and not (torch.is_grad_enabled() and (q.requires_grad or k.requires_grad))
    q, k_att, _ = _rotate_qk(mha.num_heads, q, k, rot_pos_emb_q, rot_pos_emb_k, k if shadow else None)
    o = ops.attention(q, k_att, v, mha.num_heads, mha.dp_scale, pad_mask=pad_mask,
                      causal=mha.causal_attention, impl=getattr(mha, "kernel_impl", "auto"), dropout_p=drop_p)
    o = fused_linear(mha, "_pcv_o_fold", None, mha.o_proj, o, min_rows_key)
    return ModuleOutput(last_hidden_state=o, kv_cache=kv_cache)


#: Query rows up to which a cached step on an FP8 KV cache reads the e4m3 rows directly (ops.attention_decode_fp8).
KV8_MAX_ROWS = 64


def _attend_kv8(mha, q, k, v, pad_mask, rot_pos_emb_q, rot_pos_emb_k, kv_cache, min_rows_key, kv8):
    """``attend`` with an FP8 (e4m3) KV cache: the new rows are quantised into the cache (ops.kv_append_fp8).  An empty
    incoming cache (the prompt) attends over this call's own bf16 / fp16 rows.  A cached step takes its rotated keys
    from the e4m3 shadow (ops.rotated_cache_keys) when the rotary object carries the frequency table (``inv_freq``, as
    this package's models pass it); without one (the reference's RotaryPositionEmbedding) the whole cache is rotated at
    the window-relative angles, e4m3 to e4m3 (ops.rotary_fp8), as the reference rotates it every step.  Up to
    ``KV8_MAX_ROWS`` (64) query rows read the e4m3 rows directly (ops.attention_decode_fp8: the streaming decode kernel
    up to 4 rows, the tensor-core kernel that converts e4m3 tiles in shared memory from 5 to 64).  More query rows
    dequantise the cache and take the bf16 path: there the O(N M) attention amortises the O(M) conversion, and the
    tuned forward kernel is the better one."""
    H = mha.num_heads
    L_old = kv_cache[0].shape[1]
    k8, v8 = ops.kv_append_fp8(kv_cache[0], kv_cache[1], k, v, kv8.k_inv, kv8.v_inv)
    # the prompt attends over its own bf16 / fp16 rows, a cached step over the e4m3 rows
    q_att, k_att, shadowed = _rotate_qk(H, q, k if L_old == 0 else k8, rot_pos_emb_q, rot_pos_emb_k, k8, kv8.k_descale,
                                        k_new=k)
    impl = getattr(mha, "kernel_impl", "auto")
    if L_old == 0:
        if shadowed:   # the prompt's own rows, rotated like q at the shadow's absolute positions
            k_att = ops.rotary_at(k, H, rot_pos_emb_k.inv_freq, ops.rotated_cache_shadow(k8)[1])
        o = ops.attention(q_att, k_att, v, H, mha.dp_scale, pad_mask=pad_mask, causal=mha.causal_attention, impl=impl)
    elif q.shape[1] <= KV8_MAX_ROWS:
        o = ops.attention_decode_fp8(q_att, k_att, v8, kv8.k_descale, kv8.v_descale, H, mha.dp_scale,
                                     pad_mask=pad_mask, causal=mha.causal_attention)
    else:
        o = ops.attention(q_att, ops.fp8_dequantize(k_att, kv8.k_descale, H, q.dtype),
                          ops.fp8_dequantize(v8, kv8.v_descale, H, q.dtype), H, mha.dp_scale, pad_mask=pad_mask,
                          causal=mha.causal_attention, impl=impl)
    o = fused_linear(mha, "_pcv_o_fold", None, mha.o_proj, o, min_rows_key)
    return ModuleOutput(last_hidden_state=o, kv_cache=(k8, v8))


#: Policy of the fused K/V producer (LayerNorm + k_proj + v_proj as one tcgen05 GEMM, ``ops.kv_project``).
#: ``min_rows``: below this many key rows the two library GEMMs are used (launch-bound either way).
#: ``min_rows_latent``: threshold of the SELF-attention projections (QKV and o_proj).  In eager mode a small latent array
#: (B*N of a few thousand rows) is bound by host-side dispatch, where ATen's nn.Linear path is leaner than three ctypes
#: calls; under a CUDA graph (``graphs.graph_latent_block`` lowers the threshold while recording) the fused path wins
#: because it launches 4 kernels per layer instead of 7 (tools/latent_stack_bench.py).
#: ``training``: the route of a LayerNorm -> projection chain that autograd needs (``_needs_grad``: grad mode on and x or
#: any weight or bias of the LayerNorm or the Linear layers requires grad).  On: ``ops.ln_linear`` (the fused producer
#: forward, which saves x and the row statistics instead of the LayerNorm output, and the ``pcv_ln_linear_bwd``
#: backward) for ``project_kv``, ``fused_linear`` with a norm and ``project_qkv``.  Off by default: such chains then run
#: LayerNorm + the library GEMMs.  A chain autograd does not need takes the inference kernel either way.
kv_producer_config = {"enabled": True, "min_rows": 512, "min_rows_latent": 4096, "training": False}


def _weight_cache(owner: nn.Module, slot: str, tensors, extra_key, build):
    """``build()`` cached on ``owner`` as ``owner.__dict__[slot] = (key, value)`` and rebuilt whenever ``extra_key``
    changes or one of ``tensors`` (entries may be None) was modified in place, replaced or moved (data_ptr /
    ``_version``)."""
    key = (extra_key,) + tuple((None if t is None else (t.data_ptr(), t._version)) for t in tensors)
    hit = owner.__dict__.get(slot)
    if hit is not None and hit[0] == key:
        return hit[1]
    value = build()
    owner.__dict__[slot] = (key, value)
    return value


def _params(norm: Optional[nn.Module], linears):
    """The weights and biases of ``norm`` (may be None) and ``linears``, in that order (entries may be None)."""
    return ([] if norm is None else [norm.weight, norm.bias]) + [t for lin in linears for t in (lin.weight, lin.bias)]


def _fold_cache(owner: nn.Module, slot: str, norm: Optional[nn.Module], linears, dtype: torch.dtype):
    """Folded weights ``(w_cat, col_st)`` of ``norm`` followed by ``linears`` (ops.fold_ln_linear), cached on ``owner``
    per weight version (``_weight_cache``)."""
    return _weight_cache(owner, slot, _params(norm, linears), dtype, lambda: ops.fold_ln_linear(
        None if norm is None else norm.weight, None if norm is None else norm.bias,
        [lin.weight for lin in linears], [lin.bias for lin in linears], dtype))


def _needs_grad(x: torch.Tensor, norm: Optional[nn.Module], linears) -> bool:
    """Whether autograd needs ``linears(norm(x))``: grad mode on and x, or any weight or bias of ``norm`` and
    ``linears``, requires grad.  Every kernel route that is not differentiable declines such a call."""
    return torch.is_grad_enabled() and (x.requires_grad or any(t is not None and t.requires_grad
                                                               for t in _params(norm, linears)))


def _covered(x: torch.Tensor, norm: Optional[nn.Module], linears) -> bool:
    """The conditions every LayerNorm-folded producer route shares: bf16 / fp16 CUDA rows outside autocast, a 1-D
    ``nn.LayerNorm`` over the channels of x (or no norm) and Linear weights in x's dtype reading those channels."""
    C = x.shape[-1]
    return (x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and not torch.is_autocast_enabled()
            and (norm is None or (isinstance(norm, nn.LayerNorm) and tuple(norm.normalized_shape) == (C,)))
            and all(lin.weight.dtype == x.dtype and lin.in_features == C for lin in linears))


def _has_affine(norm) -> bool:
    return isinstance(norm, nn.LayerNorm) and norm.weight is not None


def _ln_linear(owner: nn.Module, slot: str, norm: nn.LayerNorm, linears, x: torch.Tensor, n_k: int, n_v: int):
    """ops.ln_linear of ``linears(norm(x))`` with the folded weights cached on ``owner`` (rebuilt per weight version)."""
    w_cat, col_st = _fold_cache(owner, slot, norm if norm.weight is not None else None, linears, x.dtype)
    return ops.ln_linear(x, norm.weight, norm.bias, [lin.weight for lin in linears], [lin.bias for lin in linears],
                         n_k, n_v, norm.eps, w_cat, col_st)


def _ln_project(owner: nn.Module, slot: str, norm: Optional[nn.Module], linears, x: torch.Tensor,
                min_rows_key: str = "min_rows"):
    """``linears(norm(x))`` (``norm`` may be None), one output per Linear, from ONE LayerNorm-folded tcgen05 GEMM over
    the concatenated weights (the first Linear as the producer's first output, the others as column ranges of its
    second), folded weights cached on ``owner.__dict__[slot]``.  A chain autograd does not need (``_needs_grad``) runs
    the inference kernel (``ops.kv_project``); one it needs runs the training route (``_ln_linear``) when
    ``kv_producer_config["training"]`` is on and there is a norm.  None when neither covers the call: the caller then
    runs the library path."""
    n_k, n_v = linears[0].out_features, sum(lin.out_features for lin in linears[1:])
    if not (kv_producer_config["enabled"] and x.numel() // max(x.shape[-1], 1) >= kv_producer_config[min_rows_key]
            and _covered(x, norm, linears) and ops.kv_project_supported(x, n_k, n_v)):
        return None
    if not _needs_grad(x, norm, linears):
        w_cat, col_st = _fold_cache(owner, slot, norm if _has_affine(norm) else None, linears, x.dtype)
        first, rest = ops.kv_project(x, w_cat, col_st, n_k, n_v, eps=None if norm is None else norm.eps)
    elif kv_producer_config["training"] and norm is not None:
        first, rest = _ln_linear(owner, slot, norm, linears, x, n_k, n_v)
    else:
        return None
    if len(linears) == 1:
        return (first,)
    if len(linears) == 2:
        return first, rest
    n = linears[1].out_features
    return first, rest[..., :n], rest[..., n:]


def fused_linear(owner: nn.Module, slot: str, norm: Optional[nn.Module], linear: nn.Linear, x: torch.Tensor,
                 min_rows_key: str = "min_rows"):
    """``linear(norm(x))`` (``norm`` may be None) through the tcgen05 projection kernel when it applies — the q_norm ->
    q_proj chain of CrossAttention (reference modules.py:220, :113) and o_proj (:168) — else the library path."""
    y = _ln_project(owner, slot, norm, [linear], x, min_rows_key)
    return linear(x if norm is None else norm(x)) if y is None else y[0]


def project_kv(cross_attn, x_kv: torch.Tensor):
    """``k_proj(kv_norm(x_kv)), v_proj(kv_norm(x_kv))`` of a CrossAttention (reference modules.py:226, :114-115).

    bf16/fp16 CUDA rows go through the fused producer (one pass over x_kv on the tensor cores, LayerNorm folded into
    the GEMM epilogue, ``pcv_ln_stats`` + ``pcv_kv_project``; under autograd only on the training route); everything
    else — fp32, autocast, widths TMA cannot address, tiny inputs — uses LayerNorm + the two ``nn.Linear``."""
    attn, norm = cross_attn.attention, cross_attn.kv_norm
    kv = _ln_project(cross_attn, "_pcv_kv_fold", norm, [attn.k_proj, attn.v_proj], x_kv)
    if kv is None:
        x = norm(x_kv)
        kv = attn.k_proj(x), attn.v_proj(x)
    return kv


def project_qkv(self_attn, x: torch.Tensor):
    """``q_proj(norm(x)), k_proj(norm(x)), v_proj(norm(x))`` of a SelfAttention (reference modules.py:276, :113-115) as
    ONE LayerNorm-folded tcgen05 GEMM over [Wq; Wk; Wv] (``ops.kv_project`` with q as its first output and [k | v] as
    the second: k and v are column ranges of one buffer, the attention kernel takes them by stride).  Returns None when
    the fused path does not apply (``_ln_project``): the caller then runs the library path."""
    attn = self_attn.attention
    return _ln_project(self_attn, "_pcv_qkv_fold", self_attn.norm, [attn.q_proj, attn.k_proj, attn.v_proj], x,
                       "min_rows_latent")


#: FP8 (e4m3) inference route of ``CrossAttention.forward`` with ``x_kv`` (this package's class and reference modules
#: rebound by ``patch()``): q, K and V^T come out of the LayerNorm-folded producer as e4m3 (``ops.kv_project_fp8``,
#: scales derived once per weight set by ``ops.fp8_descales``) and the attention runs on the e4m3 tensor cores
#: (``ops.attention_fp8``).  Off by default because it changes the numbers; calls it does not cover (training mode,
#: a q / K / V chain autograd needs (``_needs_grad``), fp32, rotary, a KV cache, head dims that are not multiples of 16,
#: dqk > 256 or dv > 512) take the bf16 path.
#: ``kv_cache``: FP8 (e4m3) KV caches for cached generation, independent of ``enabled``: an empty incoming cache of a
#: covered CrossAttention / SelfAttention call becomes an e4m3 cache (``_kv8_route``), whose cached steps of up to 64
#: new tokens read the e4m3 rows directly (the e4m3 decode kernel up to 4, the tensor-core kernel of
#: ``pcv_attn_cached_fp8`` from 5 to 64; ``_attend_kv8``); longer steps dequantise the cache.  Off by default because
#: it changes the numbers.
fp8_config = {"enabled": False, "kv_cache": False}


class _Kv8Scales(NamedTuple):
    k_descale: torch.Tensor  # (H,) per-head K descale (pair-norm bound under rotary)
    v_descale: torch.Tensor  # (H, dv) per-channel V descale
    k_inv: torch.Tensor      # (H*dqk,) 1 / k_descale of every K channel
    v_inv: torch.Tensor      # (H*dv,)


def _kv8_scales(owner: nn.Module, norms, rotate_dim: int) -> _Kv8Scales:
    """Scales of the e4m3 KV cache of ``owner.attention``, whose k / v projections read rows normalised by ``norms``
    (one LayerNorm, or Perceiver AR's kv_norm and q_norm: its keys come from both, reference modules.py:222-224, so each
    bound is the elementwise max of the two).  Cached on ``owner`` per weight version (``_weight_cache``)."""
    attn = owner.attention
    H = attn.num_heads
    tensors = [t for n in norms for t in (n.weight, n.bias)] + _params(None, (attn.k_proj, attn.v_proj))

    def build():
        kc = torch.stack([ops.fp8_descales(n.weight, n.bias, attn.k_proj.weight, attn.k_proj.bias, H, per_channel=True)
                          for n in norms]).amax(dim=0)
        vd = torch.stack([ops.fp8_descales(n.weight, n.bias, attn.v_proj.weight, attn.v_proj.bias, H, per_channel=True)
                          for n in norms]).amax(dim=0).contiguous()
        kd = ops.fp8_pair_descale(kc, rotate_dim)
        return _Kv8Scales(kd, vd, (1.0 / kd).repeat_interleave(kc.shape[1]).contiguous(),
                          (1.0 / vd).reshape(-1).contiguous())

    return _weight_cache(owner, "_pcv_kv8_scales", tensors, rotate_dim, build)


def _kv8_route(owner: nn.Module, norms, x: torch.Tensor, rot_pos_emb_k, kv_cache) -> Optional[_Kv8Scales]:
    """The scales of the FP8 KV cache of this call of ``owner`` (a CrossAttention / SelfAttention, or a reference module
    rebound by ``patch()``), or None for the bf16 cache.  An e4m3 incoming cache always stays e4m3; an empty one becomes
    e4m3 when ``fp8_config["kv_cache"]`` is on and the call is covered: inference (no chain autograd needs, no attention
    dropout of a module in training mode) on the rows ``_covered`` takes, head dims multiples of 16 and at most 256,
    LayerNorms with an affine weight in front of k / v."""
    if kv_cache is None:
        return None
    sticky = kv_cache[0].dtype == ops.F8
    if not sticky and not (fp8_config["kv_cache"] and kv_cache[0].shape[1] == 0):
        return None
    attn = owner.attention
    H = attn.num_heads
    lins = (attn.k_proj, attn.v_proj)
    dqk, dv = attn.k_proj.out_features // H, attn.v_proj.out_features // H
    # attention dropout of a module left in training mode runs on the bf16 path only
    covered = (dqk % 16 == 0 and dv % 16 == 0 and dqk <= 256 and dv <= 256
               and not (attn.training and float(attn.dropout.p) > 0.0)
               and all(_covered(x, n, lins) and _has_affine(n) and not _needs_grad(x, n, lins) for n in norms))
    if not covered:
        if sticky:
            raise RuntimeError("an FP8 (e4m3) KV cache is inference-only: it needs bf16 / fp16 CUDA rows without "
                               "autograd, autocast or attention dropout, and a LayerNorm with an affine weight in front "
                               "of k_proj / v_proj")
        return None
    rotate_dim = 0 if rot_pos_emb_k is None else int(rot_pos_emb_k.frq_pos_enc.shape[-1])
    return _kv8_scales(owner, norms, rotate_dim)


def _fp8_scales(cross_attn, dtype: torch.dtype):
    """(q_descale (H,), k_descale (H,), v_descale (H, dv), inv_q (n_q,), inv_kv (n_k + n_v,)) of a CrossAttention,
    cached on it per weight version (``_weight_cache``)."""
    attn, H = cross_attn.attention, cross_attn.attention.num_heads
    qn, kvn = cross_attn.q_norm, cross_attn.kv_norm
    tensors = [qn.weight, qn.bias] + _params(kvn, (attn.q_proj, attn.k_proj, attn.v_proj))

    def build():
        qd = ops.fp8_descales(qn.weight, qn.bias, attn.q_proj.weight, attn.q_proj.bias, H)
        kd = ops.fp8_descales(kvn.weight, kvn.bias, attn.k_proj.weight, attn.k_proj.bias, H)
        vd = ops.fp8_descales(kvn.weight, kvn.bias, attn.v_proj.weight, attn.v_proj.bias, H, per_channel=True)
        inv_q = (1.0 / qd).repeat_interleave(attn.q_proj.out_features // H).contiguous()
        inv_kv = torch.cat([(1.0 / kd).repeat_interleave(attn.k_proj.out_features // H),
                            (1.0 / vd).reshape(-1)]).contiguous()
        return qd, kd, vd, inv_q, inv_kv

    return _weight_cache(cross_attn, "_pcv_fp8_scales", tensors, dtype, build)


def _fp8_cross_attention(cross_attn, x_q, x_kv, pad_mask, rot_pos_emb_q, rot_pos_emb_k, kv_cache):
    """The FP8 route of CrossAttention.forward, or None when it does not cover the call."""
    if not fp8_config["enabled"] or rot_pos_emb_q is not None or rot_pos_emb_k is not None or kv_cache is not None:
        return None
    attn = cross_attn.attention
    if cross_attn.training or attn.training or x_q.dim() != 3 or x_kv.dim() != 3 or x_q.dtype != x_kv.dtype:
        return None
    H = attn.num_heads
    n_q, n_k, n_v = attn.q_proj.out_features, attn.k_proj.out_features, attn.v_proj.out_features
    if n_q != n_k or n_q % H or n_v % H:
        return None
    dqk, dv = n_q // H, n_v // H
    if dqk % 16 or dv % 16 or dqk > 256 or dv > 512:
        return None
    chains = ((cross_attn.q_norm, x_q, [attn.q_proj]), (cross_attn.kv_norm, x_kv, [attn.k_proj, attn.v_proj]))
    if not all(_covered(x, n, lins) and _has_affine(n) and not _needs_grad(x, n, lins) for n, x, lins in chains):
        return None
    if not (ops.kv_project_fp8_supported(x_q, n_q, 0, H) and ops.kv_project_fp8_supported(x_kv, n_k, n_v, H)):
        return None
    qd, kd, vd, inv_q, inv_kv = _fp8_scales(cross_attn, x_kv.dtype)
    wq, stq = _fold_cache(cross_attn, "_pcv_q_fold", cross_attn.q_norm, [attn.q_proj], x_q.dtype)
    wkv, stkv = _fold_cache(cross_attn, "_pcv_kv_fold", cross_attn.kv_norm, [attn.k_proj, attn.v_proj], x_kv.dtype)
    q8, _ = ops.kv_project_fp8(x_q, wq, stq, inv_q, n_q, 0, H, eps=cross_attn.q_norm.eps)
    k8, vt8 = ops.kv_project_fp8(x_kv, wkv, stkv, inv_kv, n_k, n_v, H, eps=cross_attn.kv_norm.eps)
    o = ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, attn.dp_scale, pad_mask=pad_mask, causal=attn.causal_attention,
                          out_dtype=x_kv.dtype)
    o = fused_linear(attn, "_pcv_o_fold", None, attn.o_proj, o)
    return ModuleOutput(last_hidden_state=o, kv_cache=None)


class CrossAttention(nn.Module):
    """Pre-LayerNorm cross-attention (reference modules.py:173-230)."""

    def __init__(
        self,
        num_heads: int,
        num_q_input_channels: int,
        num_kv_input_channels: int,
        num_qk_channels: Optional[int] = None,
        num_v_channels: Optional[int] = None,
        max_heads_parallel: Optional[int] = None,
        causal_attention: bool = False,
        dropout: float = 0.0,
        qkv_bias: bool = True,
        out_bias: bool = True,
    ):
        super().__init__()
        self.q_norm = nn.LayerNorm(num_q_input_channels)
        self.kv_norm = nn.LayerNorm(num_kv_input_channels)
        self.attention = MultiHeadAttention(
            num_heads=num_heads,
            num_q_input_channels=num_q_input_channels,
            num_kv_input_channels=num_kv_input_channels,
            num_qk_channels=num_qk_channels,
            num_v_channels=num_v_channels,
            max_heads_parallel=max_heads_parallel,
            causal_attention=causal_attention,
            dropout=dropout,
            qkv_bias=qkv_bias,
            out_bias=out_bias,
        )

    def forward(
        self,
        x_q: torch.Tensor,
        x_kv: Optional[torch.Tensor] = None,
        x_kv_prefix: Optional[torch.Tensor] = None,
        pad_mask: Optional[torch.Tensor] = None,
        rot_pos_emb_q: Optional[RotaryPositionEmbedding] = None,
        rot_pos_emb_k: Optional[RotaryPositionEmbedding] = None,
        kv_cache: Optional[KVCache] = None,
    ):
        """With ``x_kv_prefix`` (Perceiver AR) the key/value input is prefix ⧺ query, where the query
        half is normalised by ``q_norm`` and only the prefix by ``kv_norm`` (reference :222-224)."""
        if x_kv is None:
            x_q = self.q_norm(x_q)
            x_kv = torch.cat([self.kv_norm(x_kv_prefix), x_q], dim=1)
            kv8 = _kv8_route(self, (self.kv_norm, self.q_norm), x_kv, rot_pos_emb_k, kv_cache)
            if kv8 is not None:
                a = self.attention
                return attend(a, a.q_proj(x_q), a.k_proj(x_kv), a.v_proj(x_kv), pad_mask, rot_pos_emb_q, rot_pos_emb_k,
                              kv_cache, kv8=kv8)
            return self.attention(x_q, x_kv, pad_mask=pad_mask, rot_pos_emb_q=rot_pos_emb_q,
                                  rot_pos_emb_k=rot_pos_emb_k, kv_cache=kv_cache)
        out = _fp8_cross_attention(self, x_q, x_kv, pad_mask, rot_pos_emb_q, rot_pos_emb_k, kv_cache)
        if out is not None:
            return out
        q = fused_linear(self, "_pcv_q_fold", self.q_norm, self.attention.q_proj, x_q)
        k, v = project_kv(self, x_kv)
        return attend(self.attention, q, k, v, pad_mask, rot_pos_emb_q, rot_pos_emb_k, kv_cache,
                      kv8=_kv8_route(self, (self.kv_norm,), x_kv, rot_pos_emb_k, kv_cache))


class SelfAttention(nn.Module):
    """Pre-LayerNorm self-attention (reference modules.py:233-278)."""

    def __init__(
        self,
        num_heads: int,
        num_channels: int,
        num_qk_channels: Optional[int] = None,
        num_v_channels: Optional[int] = None,
        max_heads_parallel: Optional[int] = None,
        causal_attention: bool = False,
        dropout: float = 0.0,
        qkv_bias: bool = True,
        out_bias: bool = True,
    ):
        super().__init__()
        self.norm = nn.LayerNorm(num_channels)
        self.attention = MultiHeadAttention(
            num_heads=num_heads,
            num_q_input_channels=num_channels,
            num_kv_input_channels=num_channels,
            num_qk_channels=num_qk_channels,
            num_v_channels=num_v_channels,
            max_heads_parallel=max_heads_parallel,
            causal_attention=causal_attention,
            dropout=dropout,
            qkv_bias=qkv_bias,
            out_bias=out_bias,
        )

    def forward(
        self,
        x: torch.Tensor,
        pad_mask: Optional[torch.Tensor] = None,
        rot_pos_emb: Optional[RotaryPositionEmbedding] = None,
        kv_cache: Optional[KVCache] = None,
    ):
        kv8 = _kv8_route(self, (self.norm,), x, rot_pos_emb, kv_cache)
        qkv = project_qkv(self, x)
        if qkv is None and kv8 is not None:
            a, xn = self.attention, self.norm(x)
            qkv = a.q_proj(xn), a.k_proj(xn), a.v_proj(xn)
        if qkv is not None:
            return attend(self.attention, qkv[0], qkv[1], qkv[2], pad_mask, rot_pos_emb, rot_pos_emb, kv_cache,
                          min_rows_key="min_rows_latent", kv8=kv8)
        x = self.norm(x)
        # a module call, so that hooks and wrappers (FSDP) see it
        # its o_proj gates on min_rows, not min_rows_latent: moving that would change the launch counts of eager latents
        return self.attention(x, x, pad_mask=pad_mask, rot_pos_emb_q=rot_pos_emb, rot_pos_emb_k=rot_pos_emb,
                              kv_cache=kv_cache)


class AbstractAttentionLayer(nn.Sequential):
    """[attention (optionally residual)] -> [residual MLP]; threads the KV cache through
    (reference modules.py:281-290)."""

    def empty_kv_cache(self, x) -> KVCache:
        shape = (x.shape[0], 0)
        return (torch.empty(*shape, self.num_qk_channels, dtype=x.dtype, device=x.device),
                torch.empty(*shape, self.num_v_channels, dtype=x.dtype, device=x.device))

    def forward(self, *args, kv_cache: Optional[KVCache] = None, **kwargs):
        attended = self[0](*args, kv_cache=kv_cache, **kwargs)
        transformed = self[1](attended.last_hidden_state)
        return ModuleOutput(last_hidden_state=transformed.last_hidden_state, kv_cache=attended.kv_cache)


class CrossAttentionLayer(AbstractAttentionLayer):
    def __init__(
        self,
        num_heads: int,
        num_q_input_channels: int,
        num_kv_input_channels: int,
        num_qk_channels: Optional[int] = None,
        num_v_channels: Optional[int] = None,
        max_heads_parallel: Optional[int] = None,
        causal_attention: bool = False,
        widening_factor: int = 1,
        dropout: float = 0.0,
        residual_dropout: float = 0.0,
        attention_residual: bool = True,
        qkv_bias: bool = True,
        out_bias: bool = True,
        mlp_bias: bool = True,
    ):
        attn = CrossAttention(
            num_heads=num_heads,
            num_q_input_channels=num_q_input_channels,
            num_kv_input_channels=num_kv_input_channels,
            num_qk_channels=num_qk_channels,
            num_v_channels=num_v_channels,
            max_heads_parallel=max_heads_parallel,
            causal_attention=causal_attention,
            dropout=dropout,
            qkv_bias=qkv_bias,
            out_bias=out_bias,
        )
        self.num_qk_channels = attn.attention.num_qk_channels
        self.num_v_channels = attn.attention.num_v_channels
        super().__init__(
            Residual(attn, residual_dropout) if attention_residual else attn,
            Residual(MLP(num_q_input_channels, widening_factor, bias=mlp_bias), residual_dropout),
        )


class SelfAttentionLayer(AbstractAttentionLayer):
    def __init__(
        self,
        num_heads: int,
        num_channels: int,
        num_qk_channels: Optional[int] = None,
        num_v_channels: Optional[int] = None,
        max_heads_parallel: Optional[int] = None,
        causal_attention: bool = False,
        widening_factor: int = 1,
        dropout: float = 0.0,
        residual_dropout: float = 0.0,
        qkv_bias: bool = True,
        out_bias: bool = True,
        mlp_bias: bool = True,
    ):
        attn = SelfAttention(
            num_heads=num_heads,
            num_channels=num_channels,
            num_qk_channels=num_qk_channels,
            num_v_channels=num_v_channels,
            max_heads_parallel=max_heads_parallel,
            causal_attention=causal_attention,
            dropout=dropout,
            qkv_bias=qkv_bias,
            out_bias=out_bias,
        )
        self.num_qk_channels = attn.attention.num_qk_channels
        self.num_v_channels = attn.attention.num_v_channels
        super().__init__(
            Residual(attn, residual_dropout),
            Residual(MLP(num_channels, widening_factor, bias=mlp_bias), residual_dropout),
        )


class SelfAttentionBlock(nn.Sequential):
    """Stack of self-attention layers; rotary only in the first ``num_rotary_layers`` (all if -1);
    one KV-cache pair per layer, ``[]`` meaning "initialise" (reference modules.py:370-441)."""

    def __init__(
        self,
        num_layers: int,
        num_heads: int,
        num_channels: int,
        num_qk_channels: Optional[int] = None,
        num_v_channels: Optional[int] = None,
        num_rotary_layers: int = 1,
        max_heads_parallel: Optional[int] = None,
        causal_attention: bool = False,
        widening_factor: int = 1,
        dropout: float = 0.0,
        residual_dropout: float = 0.0,
        activation_checkpointing: bool = False,
        activation_offloading: bool = False,
        qkv_bias: bool = True,
        out_bias: bool = True,
        mlp_bias: bool = True,
    ):
        # activation_checkpointing / activation_offloading: accepted for signature parity.  The fused
        # kernel never stores the (B,h,N,M) probabilities, which is what checkpointing was saving.
        super().__init__(*[
            SelfAttentionLayer(
                num_heads=num_heads,
                num_channels=num_channels,
                num_qk_channels=num_qk_channels,
                num_v_channels=num_v_channels,
                max_heads_parallel=max_heads_parallel,
                causal_attention=causal_attention,
                widening_factor=widening_factor,
                dropout=dropout,
                residual_dropout=residual_dropout,
                qkv_bias=qkv_bias,
                out_bias=out_bias,
                mlp_bias=mlp_bias,
            )
            for _ in range(num_layers)
        ])
        self.num_rotary_layers = num_rotary_layers

    def forward(
        self,
        x: torch.Tensor,
        pad_mask: Optional[torch.Tensor] = None,
        rot_pos_emb: Optional[RotaryPositionEmbedding] = None,
        kv_cache: Optional[List[KVCache]] = None,
    ):
        new_cache: Optional[List[KVCache]] = None
        if kv_cache is not None:
            if len(kv_cache) == 0:
                kv_cache = [layer.empty_kv_cache(x) for layer in self]
            new_cache = []

        for idx, layer in enumerate(self):
            use_rot = self.num_rotary_layers == -1 or idx < self.num_rotary_layers
            out = layer(x, pad_mask=pad_mask, rot_pos_emb=rot_pos_emb if use_rot else None,
                        kv_cache=None if kv_cache is None else kv_cache[idx])
            x = out.last_hidden_state
            if new_cache is not None:
                new_cache.append(out.kv_cache)

        return ModuleOutput(last_hidden_state=x, kv_cache=new_cache)


class MLP(nn.Sequential):
    """LayerNorm -> Linear -> GELU -> Linear (reference modules.py:444-454); stays on cuBLAS."""

    def __init__(self, num_channels: int, widening_factor: int, bias: bool = True):
        super().__init__(
            nn.LayerNorm(num_channels),
            nn.Linear(num_channels, widening_factor * num_channels, bias=bias),
            nn.GELU(),
            nn.Linear(widening_factor * num_channels, num_channels, bias=bias),
        )

    def forward(self, x):
        return ModuleOutput(last_hidden_state=super().forward(x))


class PerceiverEncoder(nn.Module):
    """Latents (1, N, D) cross-attend to adapted inputs (B, M, C), then run through self-attention
    blocks; optional repeated cross-attention and weight sharing (reference modules.py:457-607)."""

    def __init__(
        self,
        input_adapter: InputAdapter,
        num_latents: int,
        num_latent_channels: int,
        num_cross_attention_heads: int = 4,
        num_cross_attention_qk_channels: Optional[int] = None,
        num_cross_attention_v_channels: Optional[int] = None,
        num_cross_attention_layers: int = 1,
        first_cross_attention_layer_shared: bool = False,
        cross_attention_widening_factor: int = 1,
        num_self_attention_heads: int = 4,
        num_self_attention_qk_channels: Optional[int] = None,
        num_self_attention_v_channels: Optional[int] = None,
        num_self_attention_layers_per_block: int = 6,
        num_self_attention_blocks: int = 1,
        first_self_attention_block_shared: bool = True,
        self_attention_widening_factor: int = 1,
        dropout: float = 0.0,
        residual_dropout: float = 0.0,
        init_scale: float = 0.02,
        activation_checkpointing: bool = False,
        activation_offloading: bool = False,
    ):
        super().__init__()
        self.latent_provider = TrainableQueryProvider(num_latents, num_latent_channels, init_scale=init_scale)
        self.input_adapter = input_adapter

        if num_cross_attention_layers <= 0:
            raise ValueError("num_cross_attention_layers must be > 0")
        if num_self_attention_blocks <= 0:
            raise ValueError("num_self_attention_blocks must be > 0")
        if num_cross_attention_layers > num_self_attention_blocks:
            raise ValueError("num_cross_attention_layers must be <= num_self_attention_blocks")

        self.num_cross_attention_layers = num_cross_attention_layers
        self.num_self_attention_blocks = num_self_attention_blocks
        self.first_cross_attention_layer_shared = first_cross_attention_layer_shared
        self.first_self_attention_block_shared = first_self_attention_block_shared

        def make_cross_attn():
            return CrossAttentionLayer(
                num_heads=num_cross_attention_heads,
                num_q_input_channels=num_latent_channels,
                num_kv_input_channels=input_adapter.num_input_channels,
                num_qk_channels=num_cross_attention_qk_channels,
                num_v_channels=num_cross_attention_v_channels,
                widening_factor=cross_attention_widening_factor,
                dropout=dropout,
                residual_dropout=residual_dropout,
            )

        def make_self_attn():
            return SelfAttentionBlock(
                num_layers=num_self_attention_layers_per_block,
                num_heads=num_self_attention_heads,
                num_channels=num_latent_channels,
                num_qk_channels=num_self_attention_qk_channels,
                num_v_channels=num_self_attention_v_channels,
                widening_factor=self_attention_widening_factor,
                dropout=dropout,
                residual_dropout=residual_dropout,
                activation_checkpointing=activation_checkpointing,
                activation_offloading=activation_offloading,
            )

        self.cross_attn_1 = make_cross_attn()
        self.self_attn_1 = make_self_attn()
        if self.extra_cross_attention_layer:
            self.cross_attn_n = make_cross_attn()
        if self.extra_self_attention_block:
            self.self_attn_n = make_self_attn()

        self._init_parameters(init_scale)

    def _init_parameters(self, init_scale: float):
        with torch.no_grad():
            init_parameters(self, init_scale)

    @property
    def extra_cross_attention_layer(self):
        return self.num_cross_attention_layers > 1 and not self.first_cross_attention_layer_shared

    @property
    def extra_self_attention_block(self):
        return self.num_self_attention_blocks > 1 and not self.first_self_attention_block_shared

    def forward(self, x, pad_mask=None, return_adapted_input=False):
        x_adapted = self.input_adapter(x)
        x_latent = self.latent_provider()  # (1, N, D): broadcast by the kernel, never expanded

        x_latent = self.cross_attn_1(x_latent, x_adapted, pad_mask=pad_mask).last_hidden_state
        x_latent = self.self_attn_1(x_latent).last_hidden_state

        later_cross = self.cross_attn_n if self.extra_cross_attention_layer else self.cross_attn_1
        later_self = self.self_attn_n if self.extra_self_attention_block else self.self_attn_1
        for block in range(1, self.num_self_attention_blocks):
            if block < self.num_cross_attention_layers:
                x_latent = later_cross(x_latent, x_adapted, pad_mask=pad_mask).last_hidden_state
            x_latent = later_self(x_latent).last_hidden_state

        return (x_latent, x_adapted) if return_adapted_input else x_latent


class PerceiverDecoder(nn.Module):
    """Output queries cross-attend to the latents (reverse asymmetry: many queries, few keys);
    reference modules.py:610-675."""

    def __init__(
        self,
        output_adapter: OutputAdapter,
        output_query_provider: QueryProvider,
        num_latent_channels: int,
        num_cross_attention_heads: int = 4,
        num_cross_attention_qk_channels: Optional[int] = None,
        num_cross_attention_v_channels: Optional[int] = None,
        cross_attention_widening_factor: int = 1,
        cross_attention_residual: bool = True,
        dropout: float = 0.0,
        init_scale: float = 0.02,
        activation_checkpointing: bool = False,
        activation_offloading: bool = False,
    ):
        super().__init__()
        self.output_query_provider = output_query_provider
        self.output_adapter = output_adapter
        self.cross_attn = CrossAttentionLayer(
            num_heads=num_cross_attention_heads,
            num_q_input_channels=output_query_provider.num_query_channels,
            num_kv_input_channels=num_latent_channels,
            num_qk_channels=num_cross_attention_qk_channels,
            num_v_channels=num_cross_attention_v_channels,
            widening_factor=cross_attention_widening_factor,
            attention_residual=cross_attention_residual,
            dropout=dropout,
        )
        self._init_parameters(init_scale)

    def _init_parameters(self, init_scale: float):
        with torch.no_grad():
            init_parameters(self, init_scale)

    def forward(self, x_latent, x_adapted=None, **kwargs):
        output_query = self.output_query_provider(x_adapted)
        decoded = self.cross_attn(output_query, x_latent).last_hidden_state
        return self.output_adapter(decoded, **kwargs)


class PerceiverIO(nn.Sequential):
    def __init__(self, encoder: PerceiverEncoder, decoder: PerceiverDecoder):
        super().__init__(encoder, decoder)

    @property
    def encoder(self):
        return self[0]

    @property
    def decoder(self):
        return self[1]


class PerceiverAR(nn.Module):
    """Perceiver AR: the last ``n - prefix_len`` positions are latents that cross-attend causally to
    prefix ⧺ latents, followed by causal latent self-attention; left padding, prefix dropout,
    right-aligned rotary embeddings and KV caching as in reference modules.py:691-871."""

    def __init__(
        self,
        input_adapter: RotarySupport,
        num_heads: int = 8,
        max_heads_parallel: Optional[int] = None,
        num_self_attention_layers: int = 6,
        num_self_attention_rotary_layers: int = 1,
        self_attention_widening_factor: int = 4,
        cross_attention_widening_factor: int = 4,
        cross_attention_dropout: float = 0.5,
        post_attention_dropout: float = 0.0,
        residual_dropout: float = 0.0,
        activation_checkpointing: bool = False,
        activation_offloading: bool = False,
    ):
        super().__init__()
        channels = input_adapter.num_input_channels
        self.input_adapter = input_adapter
        self.cross_attention_dropout = cross_attention_dropout
        self.cross_attention = CrossAttentionLayer(
            num_heads=num_heads,
            num_q_input_channels=channels,
            num_kv_input_channels=channels,
            max_heads_parallel=max_heads_parallel,
            causal_attention=True,
            widening_factor=cross_attention_widening_factor,
            dropout=post_attention_dropout,
            residual_dropout=residual_dropout,
            qkv_bias=False,
            out_bias=True,
            mlp_bias=False,
        )
        self.self_attention = SelfAttentionBlock(
            num_layers=num_self_attention_layers,
            num_heads=num_heads,
            num_channels=channels,
            causal_attention=True,
            widening_factor=self_attention_widening_factor,
            dropout=post_attention_dropout,
            residual_dropout=residual_dropout,
            num_rotary_layers=num_self_attention_rotary_layers,
            activation_checkpointing=activation_checkpointing,
            activation_offloading=activation_offloading,
            qkv_bias=False,
            out_bias=False,
            mlp_bias=False,
        )

    def forward(
        self,
        x: torch.Tensor,
        prefix_len: int,
        pad_mask: Optional[torch.Tensor] = None,
        kv_cache: Optional[List[KVCache]] = None,
    ):
        # ---- integer path (must match the reference bit for bit; modules.py:776-807) -------------
        shift = None if pad_mask is None else pad_mask.sum(dim=1, keepdim=True)  # x is left-padded
        cache_active = kv_cache is not None and len(kv_cache) > 0
        b = x.shape[0]
        n = x.shape[1] + (kv_cache[0][0].shape[1] if cache_active else 0)
        if not 0 <= prefix_len < n:
            raise ValueError(f"prefix_len ({prefix_len}) out of valid range [0..{n})")

        x, frq_pos_enc = self.input_adapter(x, abs_pos=positions(b, n, shift=shift, device=x.device))

        if cache_active:
            x_latent, x_prefix = x, x[:, :0]
        else:
            x_latent, x_prefix = x[:, prefix_len:], x[:, :prefix_len]

        frq_latent, frq_prefix = frq_pos_enc[:, prefix_len:], frq_pos_enc[:, :prefix_len]
        if pad_mask is not None:
            pad_latent, pad_prefix = pad_mask[:, prefix_len:], pad_mask[:, :prefix_len]

        # ---- training-time prefix dropout: keep a random subset of prefix positions (:809-830) ----
        if self.training and prefix_len > 0 and self.cross_attention_dropout > 0.0:
            if kv_cache is not None:
                raise ValueError("cross-attention dropout not supported with caching")
            rand = torch.rand(b, prefix_len, device=x.device)
            keep = prefix_len - int(prefix_len * self.cross_attention_dropout)
            keep_idx = rand.topk(keep, dim=-1).indices
            keep_mask = torch.zeros_like(rand, dtype=torch.bool).scatter_(dim=1, index=keep_idx, value=1)
            x_prefix = x_prefix[keep_mask].reshape(b, keep, x_prefix.shape[-1])
            frq_prefix = frq_prefix[keep_mask].reshape(b, keep, frq_prefix.shape[-1])
            if pad_mask is not None:
                pad_prefix = pad_prefix[keep_mask].reshape(b, keep)

        frq_keys = torch.cat([frq_prefix, frq_latent], dim=1)
        if pad_mask is not None:
            pad_mask = torch.cat([pad_prefix, pad_latent], dim=1)

        # ---- cache routing (:838-848) -------------------------------------------------------------
        if kv_cache is None:
            ca_cache, sa_cache, new_cache = None, None, None
        elif len(kv_cache) == 0:
            ca_cache, sa_cache, new_cache = self.cross_attention.empty_kv_cache(x_latent), [], []
        else:
            ca_cache, sa_cache, new_cache = kv_cache[0], list(kv_cache[1:]), []

        # frequency table of the adapter: lets cached decoding rotate new keys only (ops.rotated_cache_keys)
        inv_freq = getattr(getattr(self.input_adapter, "frq_pos_encoding", None), "inv_freq", None)
        ca_out = self.cross_attention(
            x_latent,
            x_kv_prefix=x_prefix,
            pad_mask=pad_mask,
            rot_pos_emb_q=RotaryPositionEmbedding(frq_latent, right_align=True, inv_freq=inv_freq),
            rot_pos_emb_k=RotaryPositionEmbedding(frq_keys, right_align=True, inv_freq=inv_freq),
            kv_cache=ca_cache,
        )
        if new_cache is not None:
            new_cache.append(ca_out.kv_cache)

        sa_out = self.self_attention(
            ca_out.last_hidden_state,
            rot_pos_emb=RotaryPositionEmbedding(frq_latent, right_align=True, inv_freq=inv_freq),
            kv_cache=sa_cache,
        )
        if new_cache is not None:
            new_cache.extend(sa_out.kv_cache)

        return ModuleOutput(last_hidden_state=sa_out.last_hidden_state, kv_cache=new_cache)


class CausalSequenceModel(PerceiverAR):
    """Perceiver AR + token adapters + tied-embedding logits (reference modules.py:874-930)."""

    def __init__(self, config: CausalSequenceModelConfig):
        rotated = config.num_channels // config.num_heads
        if config.abs_pos_emb:
            rotated //= 2  # rotary on the first half of each head's channels only
        input_adapter = TokenInputAdapterWithRotarySupport(
            rotated_channels_per_head=rotated,
            vocab_size=config.vocab_size,
            max_seq_len=config.max_seq_len,
            num_input_channels=config.num_channels,
            abs_pos_emb=config.abs_pos_emb,
        )
        super().__init__(input_adapter=input_adapter, **config.base_kwargs())
        self.config = config
        if config.output_norm:
            self.out_norm = nn.LayerNorm(config.num_channels)
        self.output_adapter = TiedTokenOutputAdapter(vocab_size=config.vocab_size, emb_bias=config.output_bias)
        self._init_parameters(config.init_scale)

    def _init_parameters(self, init_scale: float):
        with torch.no_grad():
            init_parameters(self, init_scale)

    @property
    def max_seq_len(self):
        return self.input_adapter.max_seq_len

    @property
    def max_latents(self):
        return self.config.max_latents

    @property
    def max_prefix_len(self):
        return self.max_seq_len - self.max_latents

    def forward(
        self,
        x: torch.Tensor,
        prefix_len: int,
        pad_mask: Optional[torch.Tensor] = None,
        kv_cache: Optional[List[KVCache]] = None,
    ):
        if prefix_len > self.max_prefix_len:
            raise ValueError(f"prefix_len ({prefix_len}) exceeds max_prefix_len ({self.max_prefix_len})")
        output = super().forward(x, prefix_len=prefix_len, pad_mask=pad_mask, kv_cache=kv_cache)
        if self.config.output_norm:
            output.last_hidden_state = self.out_norm(output.last_hidden_state)
        output.logits = self.output_adapter(output.last_hidden_state, txt_embedding=self.input_adapter.txt_embedding)
        return output
