"""CPU oracle for the latent-attention hot path — TEST INFRASTRUCTURE ONLY.

This is a from-scratch restatement, in plain torch CPU ops on explicit weight dictionaries, of the
algorithm in /root/reference/perceiver/model/core/{modules,position,utils}.py.  It exists to CHECK
the CUDA path: only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import it.  The product package (``perceiver_io_b200``) never does.

Pinning (SURVEY.md §8(c)): the reference holds no stored numeric vectors for this path, so the
oracle is pinned against outputs of the reference itself — ``oracle/gen_golden.py`` imports the
real reference modules in the authoring container and writes ``tests/golden/*.pt``;
``tests/test_oracle_golden.py`` replays them through this file (fp32, atol 1e-5 / bit-exact for
integer paths) on every CPU test run.

Every function names the reference lines it follows.  Weights are addressed by the reference's own
``state_dict`` keys (e.g. ``"attention.q_proj.weight"``), so a reference checkpoint feeds the
oracle directly.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

Tensor = torch.Tensor
Weights = Dict[str, Tensor]
Rotary = Optional[Tuple[Tensor, bool]]  # (angles (B|1, n, f), right_align)


# ------------------------------------------------------------------------------------------------
# leaf math
# ------------------------------------------------------------------------------------------------
def linear(x: Tensor, w: Weights, name: str) -> Tensor:
    """nn.Linear with optional bias."""
    y = x @ w[name + ".weight"].to(x.dtype).T
    b = w.get(name + ".bias")
    return y if b is None else y + b.to(x.dtype)


def layer_norm(x: Tensor, w: Weights, name: str, eps: float = 1e-5) -> Tensor:
    """nn.LayerNorm over the last dim (affine, eps 1e-5 — torch default used at modules.py:191-192,253)."""
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w[name + ".weight"].to(x.dtype) + w[name + ".bias"].to(x.dtype)


def gelu(x: Tensor) -> Tensor:
    """Exact (erf) GELU — nn.GELU() default at modules.py:449."""
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def positions(b: int, n: int, shift: Optional[Tensor] = None) -> Tensor:
    """position.py:9-17 — clamp(arange(n) - shift, min=0); integer, bit-exact."""
    pos = torch.arange(n).reshape(1, n).repeat(b, 1)
    if shift is not None:
        pos = pos - shift.reshape(b, 1)
    return pos.clamp(min=0)


def frequency_angles(abs_pos: Tensor, dim: int, dtype=torch.float32) -> Tensor:
    """position.py:53-71 — angles[b,n,2i] = angles[b,n,2i+1] = pos * 10000^(-2i/dim)."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dim, 2).float() / dim))
    enc = abs_pos.to(torch.float32)[..., None] * inv_freq
    return torch.stack((enc, enc), dim=-1).flatten(-2).to(dtype)


def rotate(t: Tensor, angles: Tensor, right_align: bool) -> Tensor:
    """position.py:30-50 — t is (B, H, n, d); angles (B|1, n_a, f) broadcast over heads.

    Rows: last n angle rows if right_align else first n (:32-37).  Channels [0,f) rotated pairwise with
    rotate_half [x1,x2,x3,x4..] -> [-x2,x1,-x4,x3..] (:44-50); channels >= f pass through (:39-42)."""
    n = t.shape[-2]
    a = angles[:, None, -n:, :] if right_align else angles[:, None, :n, :]
    a = a.to(t.dtype)
    f = a.shape[-1]
    rot, keep = t[..., :f], t[..., f:]
    even, odd = rot[..., 0::2], rot[..., 1::2]
    half = torch.stack((-odd, even), dim=-1).flatten(-2)
    return torch.cat((rot * a.cos() + half * a.sin(), keep), dim=-1)


def split_heads(x: Tensor, h: int) -> Tensor:
    """modules.py:123 — (b, n, h*c) -> (b, h, n, c)."""
    b, n, hc = x.shape
    return x.reshape(b, n, h, hc // h).permute(0, 2, 1, 3)


def merge_heads(x: Tensor) -> Tensor:
    """modules.py:167 — (b, h, n, c) -> (b, n, h*c)."""
    b, h, n, c = x.shape
    return x.permute(0, 2, 1, 3).reshape(b, n, h * c)


def masked_scores(q: Tensor, k: Tensor, pad_mask: Optional[Tensor], causal: bool,
                  m_total: Optional[int] = None, m_offset: int = 0) -> Tensor:
    """modules.py:151-158 — S = q k^T with padding / right-aligned causal entries REPLACED by
    -finfo(dtype).max.  q is already scaled.  (m_total, m_offset) describe an M-shard: key j has global
    index m_offset + j; the causal rule masks global col > row + (m_total - N) (:135-140)."""
    s = q @ k.transpose(-1, -2)
    neg = -torch.finfo(s.dtype).max
    n, m = s.shape[-2], s.shape[-1]
    if pad_mask is not None:
        s = s.masked_fill(pad_mask[:, None, None, :].bool(), neg)
    if causal:
        mt = m if m_total is None else m_total
        rows = torch.arange(n, device=s.device)[:, None]
        cols = torch.arange(m, device=s.device)[None, :] + m_offset
        s = s.masked_fill(cols > rows + (mt - n), neg)
    return s


def core_attention(q: Tensor, k: Tensor, v: Tensor, scale: float, pad_mask: Optional[Tensor] = None,
                   causal: bool = False) -> Tensor:
    """modules.py:124,146-164 on head-split tensors: softmax(masked(scale*q k^T)) v.  (B,H,N,dv)."""
    s = masked_scores(q * scale, k, pad_mask, causal)
    return s.softmax(dim=-1) @ v


# ------------------------------------------------------------------------------------------------
# partial softmax state of an M-shard and its exact merge (SURVEY.md §8(e)); log2 domain like the
# kernels: t = s*log2(e), m = rowmax(t), l = sum 2^(t-m), o = sum 2^(t-m) v
# ------------------------------------------------------------------------------------------------
LOG2E = 1.4426950408889634


def partial_state(q: Tensor, k: Tensor, v: Tensor, scale: float, pad_mask: Optional[Tensor], causal: bool,
                  m_total: int, m_offset: int) -> Tuple[Tensor, Tensor, Tensor]:
    s = masked_scores(q * scale, k, pad_mask, causal, m_total, m_offset)
    neg = -torch.finfo(s.dtype).max
    t = torch.where(s == neg, s, s * LOG2E)  # the finite fill is a sentinel, it is not rescaled
    m = t.amax(dim=-1)
    p = torch.exp2(t - m[..., None])
    return p @ v, m, p.sum(-1)


def merge_states(parts: Sequence[Tuple[Tensor, Tensor, Tensor]]) -> Tensor:
    o = torch.stack([p[0] for p in parts])
    m = torch.stack([p[1] for p in parts])
    l = torch.stack([p[2] for p in parts])
    mx = m.amax(dim=0)
    w = torch.exp2(m - mx)
    return (o * w[..., None]).sum(0) / (l * w).sum(0)[..., None]


# ------------------------------------------------------------------------------------------------
# modules
# ------------------------------------------------------------------------------------------------
def sub(w: Weights, prefix: str) -> Weights:
    """Weights under ``prefix`` with the prefix stripped."""
    return {k[len(prefix):]: v for k, v in w.items() if k.startswith(prefix)}


def mha(w: Weights, x_q: Tensor, x_kv: Tensor, num_heads: int, pad_mask: Optional[Tensor] = None,
        rot_q: Rotary = None, rot_k: Rotary = None, kv_cache: Optional[Tuple[Tensor, Tensor]] = None,
        causal: bool = False):
    """MultiHeadAttention.forward, modules.py:113-170, in order: project (:113-115) -> cache concat on
    the sequence dim, cache stays un-rotated (:117-121) -> head split (:123) -> scale q (:124) ->
    rotary (:126-130) -> masks/softmax/PV (:132-164) -> merge heads, o_proj (:166-168)."""
    q = linear(x_q, w, "q_proj")
    k = linear(x_kv, w, "k_proj")
    v = linear(x_kv, w, "v_proj")
    if kv_cache is not None:
        k = torch.cat([kv_cache[0].to(k.dtype), k], dim=1)
        v = torch.cat([kv_cache[1].to(v.dtype), v], dim=1)
        kv_cache = (k, v)
    qh, kh, vh = (split_heads(t, num_heads) for t in (q, k, v))
    scale = qh.shape[-1] ** -0.5
    qh = qh * scale
    if rot_q is not None:
        qh = rotate(qh, *rot_q)
    if rot_k is not None:
        kh = rotate(kh, *rot_k)
    s = masked_scores(qh, kh, pad_mask, causal)
    o = merge_heads(s.softmax(dim=-1) @ vh)
    return linear(o, w, "o_proj"), kv_cache


def cross_attention(w: Weights, x_q: Tensor, x_kv: Optional[Tensor], num_heads: int,
                    x_kv_prefix: Optional[Tensor] = None, **kw):
    """CrossAttention.forward, modules.py:220-230 (prefix mode: kv = kv_norm(prefix) ⧺ q_norm(x_q))."""
    x_q = layer_norm(x_q, w, "q_norm")
    if x_kv is None:
        x_kv = torch.cat([layer_norm(x_kv_prefix, w, "kv_norm"), x_q], dim=1)
    else:
        x_kv = layer_norm(x_kv, w, "kv_norm")
    return mha(sub(w, "attention."), x_q, x_kv, num_heads, **kw)


def self_attention(w: Weights, x: Tensor, num_heads: int, pad_mask=None, rot: Rotary = None, kv_cache=None,
                   causal: bool = False):
    """SelfAttention.forward, modules.py:269-278."""
    x = layer_norm(x, w, "norm")
    return mha(sub(w, "attention."), x, x, num_heads, pad_mask=pad_mask, rot_q=rot, rot_k=rot,
               kv_cache=kv_cache, causal=causal)


def mlp(w: Weights, x: Tensor) -> Tensor:
    """MLP, modules.py:444-454: LayerNorm -> Linear -> GELU -> Linear (Sequential indices 0,1,3)."""
    return linear(gelu(linear(layer_norm(x, w, "0"), w, "1")), w, "3")


def _layer_prefixes(w: Weights) -> Tuple[str, bool]:
    residual = any(k.startswith("0.module.") for k in w)
    return ("0.module." if residual else "0."), residual


def cross_attention_layer(w: Weights, x_q: Tensor, x_kv: Optional[Tensor], num_heads: int, **kw):
    """CrossAttentionLayer via AbstractAttentionLayer.forward (modules.py:287-290) and Residual
    (utils.py:29-32): h = attn(x_q, ...) [+ x_q] ; y = mlp(h) + h.  ``attention_residual=False`` is
    recognised from the weight names (no ``module.`` level under ``0.``)."""
    pre, residual = _layer_prefixes(w)
    h, cache = cross_attention(sub(w, pre), x_q, x_kv, num_heads, **kw)
    if residual:
        h = h + x_q
    return mlp(sub(w, "1.module."), h) + h, cache


def self_attention_layer(w: Weights, x: Tensor, num_heads: int, **kw):
    h, cache = self_attention(sub(w, "0.module."), x, num_heads, **kw)
    h = h + x
    return mlp(sub(w, "1.module."), h) + h, cache


def self_attention_block(w: Weights, x: Tensor, num_heads: int, num_layers: int, num_rotary_layers: int = 1,
                         pad_mask=None, rot: Rotary = None, kv_cache: Optional[List] = None, causal: bool = False):
    """SelfAttentionBlock.forward, modules.py:414-441."""
    new_cache = None
    if kv_cache is not None:
        if len(kv_cache) == 0:
            kv_cache = [None] * num_layers  # "initialise": an empty cache concatenates to nothing
        new_cache = []
    for i in range(num_layers):
        use_rot = num_rotary_layers == -1 or i < num_rotary_layers
        cache_i = None
        if kv_cache is not None:
            cache_i = kv_cache[i]
            if cache_i is None:
                lw = sub(w, f"{i}.0.module.attention.")
                cache_i = (x.new_zeros(x.shape[0], 0, lw["k_proj.weight"].shape[0]),
                           x.new_zeros(x.shape[0], 0, lw["v_proj.weight"].shape[0]))
        x, c = self_attention_layer(sub(w, f"{i}."), x, num_heads, pad_mask=pad_mask, rot=rot if use_rot else None,
                                    kv_cache=cache_i, causal=causal)
        if new_cache is not None:
            new_cache.append(c)
    return x, new_cache


def prefix_keep_mask(rand: Tensor, prefix_len: int, p: float) -> Tuple[Tensor, Tensor, int]:
    """Training-time prefix (cross-attention) dropout, integer path of modules.py:816-821: keep the
    ``prefix_len - int(prefix_len * p)`` positions with the largest random numbers.  Returns
    (keep_mask (b, prefix_len) bool, keep_idx (b, keep) int64, keep)."""
    keep = prefix_len - int(prefix_len * p)                                                         # :817
    keep_idx = rand.topk(keep, dim=-1).indices                                                      # :818
    keep_mask = torch.zeros_like(rand, dtype=torch.bool).scatter_(dim=1, index=keep_idx, value=1)   # :820-821
    return keep_mask, keep_idx, keep


def perceiver_ar(w: Weights, x_tokens: Tensor, prefix_len: int, num_heads: int, num_layers: int,
                 num_rotary_layers: int, rotated_channels: int, abs_pos_emb: bool,
                 pad_mask: Optional[Tensor] = None, kv_cache: Optional[List] = None,
                 output_norm: bool = False, output_bias: bool = True,
                 dropout_rand: Optional[Tensor] = None, dropout_p: float = 0.0):
    """CausalSequenceModel.forward = PerceiverAR.forward + logits (modules.py:768-871, 914-930).  Eval mode
    unless ``dropout_rand`` (the (b, prefix_len) matrix the reference draws with torch.rand, :816) is given, in
    which case the training-time prefix dropout of :809-830 is applied.  Returns (hidden, logits, kv_cache)."""
    shift = None if pad_mask is None else pad_mask.sum(dim=1, keepdim=True)
    cache_active = kv_cache is not None and len(kv_cache) > 0
    b = x_tokens.shape[0]
    n = x_tokens.shape[1] + (kv_cache[0][0].shape[1] if cache_active else 0)
    if not 0 <= prefix_len < n:
        raise ValueError(f"prefix_len ({prefix_len}) out of valid range [0..{n})")
    abs_pos = positions(b, n, shift)
    emb = w["input_adapter.txt_embedding.weight"]
    x = emb[x_tokens]
    if abs_pos_emb:
        pos_for_x = abs_pos[:, -x_tokens.shape[1]:] if x_tokens.shape[1] < n else abs_pos
        x = x + w["input_adapter.pos_embedding.weight"][pos_for_x]
    frq = frequency_angles(abs_pos, rotated_channels, x.dtype)

    if cache_active:
        x_latent, x_prefix = x, x[:, :0]
    else:
        x_latent, x_prefix = x[:, prefix_len:], x[:, :prefix_len]
    frq_latent = frq[:, prefix_len:]
    frq_keys = frq
    if dropout_rand is not None and prefix_len > 0 and dropout_p > 0.0:
        if kv_cache is not None:
            raise ValueError("cross-attention dropout not supported with caching")                  # :810-812
        keep_mask, _, keep = prefix_keep_mask(dropout_rand, prefix_len, dropout_p)
        x_prefix = x_prefix[keep_mask].reshape(b, keep, x_prefix.shape[-1])                         # :823
        frq_prefix = frq[:, :prefix_len][keep_mask].reshape(b, keep, frq.shape[-1])                 # :824
        frq_keys = torch.cat([frq_prefix, frq_latent], dim=1)                                       # :832
        if pad_mask is not None:
            pad_prefix = pad_mask[:, :prefix_len][keep_mask].reshape(b, keep)                       # :826-827
            pad_mask = torch.cat([pad_prefix, pad_mask[:, prefix_len:]], dim=1)                     # :835-836

    ca_cache = None
    sa_cache = None
    if kv_cache is not None:
        if cache_active:
            ca_cache, sa_cache = kv_cache[0], list(kv_cache[1:])
        else:
            c = w["cross_attention.0.module.attention.k_proj.weight"].shape[0]
            cv = w["cross_attention.0.module.attention.v_proj.weight"].shape[0]
            ca_cache, sa_cache = (x.new_zeros(b, 0, c), x.new_zeros(b, 0, cv)), []

    h, ca_new = cross_attention_layer(sub(w, "cross_attention."), x_latent, None, num_heads, x_kv_prefix=x_prefix,
                                      pad_mask=pad_mask, rot_q=(frq_latent, True), rot_k=(frq_keys, True),
                                      kv_cache=ca_cache, causal=True)
    h, sa_new = self_attention_block(sub(w, "self_attention."), h, num_heads, num_layers, num_rotary_layers,
                                     rot=(frq_latent, True), kv_cache=sa_cache, causal=True)
    new_cache = None if kv_cache is None else [ca_new] + sa_new
    if output_norm:
        h = layer_norm(h, w, "out_norm")
    logits = h @ emb.to(h.dtype).T
    if output_bias:
        logits = logits + w["output_adapter.bias"].to(h.dtype)
    return h, logits, new_cache


def encoder(w: Weights, x_adapted: Tensor, num_ca_heads: int, num_sa_heads: int, num_sa_layers: int,
            num_blocks: int = 1, num_ca_layers: int = 1, first_ca_shared: bool = False,
            first_sa_shared: bool = True, pad_mask: Optional[Tensor] = None) -> Tensor:
    """PerceiverEncoder.forward on already adapted input, modules.py:587-607."""
    lat = w["latent_provider._query"][None]
    lat, _ = cross_attention_layer(sub(w, "cross_attn_1."), lat, x_adapted, num_ca_heads, pad_mask=pad_mask)
    lat, _ = self_attention_block(sub(w, "self_attn_1."), lat, num_sa_heads, num_sa_layers, num_rotary_layers=0)
    ca_n = "cross_attn_n." if (num_ca_layers > 1 and not first_ca_shared) else "cross_attn_1."
    sa_n = "self_attn_n." if (num_blocks > 1 and not first_sa_shared) else "self_attn_1."
    for i in range(1, num_blocks):
        if i < num_ca_layers:
            lat, _ = cross_attention_layer(sub(w, ca_n), lat, x_adapted, num_ca_heads, pad_mask=pad_mask)
        lat, _ = self_attention_block(sub(w, sa_n), lat, num_sa_heads, num_sa_layers, num_rotary_layers=0)
    return lat


def decoder(w: Weights, x_latent: Tensor, query: Tensor, num_heads: int) -> Tensor:
    """PerceiverDecoder.forward without the task adapters, modules.py:672-675."""
    out, _ = cross_attention_layer(sub(w, "cross_attn."), query, x_latent, num_heads)
    return out
