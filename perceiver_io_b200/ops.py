"""Torch-facing wrappers of the C-ABI ops (``include/pcv_attn.h``).

PyTorch is plumbing here: it owns device memory and the stream.  Every function below passes raw
``data_ptr()`` values, element strides and ``torch.cuda.current_stream().cuda_stream`` to
``libpcv_attn.so``; nothing synchronises.  Inputs must live on a CUDA device — there is no CPU
path and no PyTorch re-implementation to fall back to (``PcvError`` / ``RuntimeError`` instead).

dtype policy (SURVEY.md §8(b) "dtype / device"): the kernels compute on bf16 (or fp16) operands
with fp32 accumulation.  fp32 inputs are explicitly rounded to bf16 at this boundary and the
result is returned in the caller's dtype; parity tolerances are defined against the reference
evaluated on the same bf16-rounded operands.
"""
from __future__ import annotations

import ctypes as C
import math
import operator
import struct
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import (AttnParams, CombineParams, KvAppendParams, KvProjParams, LnStatsParams, RescaleParams, RotaryParams,
                   PcvError, check)

__all__ = [
    "attention", "attention_partial", "attention_sharded_fused", "combine_partials", "merge_partials", "rescale_partial_", "rotary", "kv_append",
    "device_info", "tcgen05_supported", "rotated_cache_keys", "ln_stats", "fold_ln_linear", "kv_project", "kv_project_supported",
    "attention_fp8", "attention_fp8_supported", "fp8_descales", "fp8_quantize", "fp8_transpose_v", "kv_project_fp8",
    "kv_project_fp8_supported", "ln_linear", "ln_linear_backward", "kv_append_fp8", "attention_decode_fp8",
    "attention_decode_fp8_supported", "fp8_pair_descale", "fp8_dequantize", "rotated_cache_shadow", "rotary_at", "rotary_fp8",
    "attention_decode_window", "kv_append_at", "rotary_apply_at", "rotary_angle_table", "attention_window",
    "sample_tokens", "sample_uniforms", "spec_verify", "spec_uniforms", "BeamState", "beam_step", "KvGatherTable",
    "kv_gather_rows",
]


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _require_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "perceiver_io_b200 ops run on CUDA (sm_90a) tensors only; got a tensor on "
                f"{t.device}. There is no CPU fallback for the attention path."
            )


def _pcv_dtype(dt: torch.dtype) -> int:
    if dt == torch.bfloat16:
        return _lib.PCV_BF16
    if dt == torch.float16:
        return _lib.PCV_F16
    raise RuntimeError(f"unsupported compute dtype {dt}")


def _compute_dtype(dt: torch.dtype) -> torch.dtype:
    return dt if dt in (torch.bfloat16, torch.float16) else torch.bfloat16


def _rows_contiguous(t: torch.Tensor) -> torch.Tensor:
    """Unit channel stride (every other stride is passed through to the kernel)."""
    return t if t.stride(-1) == 1 else t.contiguous()


def device_info() -> dict:
    info = _lib.DeviceInfo()
    check(_lib.lib().pcv_get_device_info(C.byref(info)), "pcv_get_device_info")
    return {f[0]: getattr(info, f[0]) for f in info._fields_}


def _fill_attn_params(q, k, v, num_heads, scale, pad_mask, causal, m_total, m_offset, impl,
                      dtype: Optional[int] = None) -> Tuple[AttnParams, tuple]:
    # ``dtype``: the pcv_dtype of the operands when it is not that of q's torch dtype (PCV_E4M3).
    # Each operand is either (B, L, H*d) — heads split by stride arithmetic — or an explicit 4-D
    # (B, L, H, d) view with arbitrary batch/row/head strides (e.g. a head-major (B,H,L,d) buffer permuted).
    def geom(t, name):
        if t.dim() == 3:
            if t.shape[2] % num_heads:
                raise ValueError("channel counts must be divisible by num_heads")
            d = t.shape[2] // num_heads
            return t.shape[0], t.shape[1], d, t.stride(0), t.stride(1), d
        if t.dim() == 4:
            if t.shape[2] != num_heads:
                raise ValueError(f"{name}: 4-D operands must be (B, L, H={num_heads}, d), got {tuple(t.shape)}")
            if t.stride(3) != 1:
                raise ValueError(f"{name}: the channel dimension must have unit stride")
            return t.shape[0], t.shape[1], t.shape[3], t.stride(0), t.stride(1), t.stride(2)
        raise ValueError("q, k, v must be (B, L, C) or (B, L, H, d) tensors")

    Bq, N, dqk, q_sb, q_sn, q_sh = geom(q, "q")
    B, M, dk, k_sb, k_sm, k_sh = geom(k, "k")
    Bv, Mv, dv, v_sb, v_sm, v_sh = geom(v, "v")
    if Bv != B or Mv != M:
        raise ValueError(f"k {tuple(k.shape)} and v {tuple(v.shape)} disagree on (B, M)")
    if Bq not in (1, B):
        raise ValueError(f"query batch {Bq} must be 1 or equal to key batch {B}")
    if dqk != dk:
        raise ValueError(f"q head channels {dqk} != k head channels {dk}")
    H = num_heads
    p = AttnParams()
    p.q, p.k, p.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    p.q_stride_b = 0 if (Bq == 1 and B > 1) else q_sb
    p.q_stride_n, p.q_stride_h = q_sn, q_sh
    p.k_stride_b, p.k_stride_m, p.k_stride_h = k_sb, k_sm, k_sh
    p.v_stride_b, p.v_stride_m, p.v_stride_h = v_sb, v_sm, v_sh
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.scale = float(scale)
    p.dtype = _pcv_dtype(q.dtype) if dtype is None else dtype
    p.causal = 1 if causal else 0
    p.m_total = M if m_total is None else int(m_total)
    p.m_offset = int(m_offset)
    keep = [q, k, v]
    if pad_mask is not None:
        if pad_mask.shape != (B, M):
            raise ValueError(f"pad_mask shape {tuple(pad_mask.shape)} != {(B, M)}")
        pm = pad_mask
        if pm.dtype == torch.bool:
            pm = pm.view(torch.uint8) if pm.stride(-1) == 1 else pm.contiguous().view(torch.uint8)
        elif pm.dtype != torch.uint8:
            pm = (pm != 0).view(torch.uint8)
        if pm.stride(-1) != 1:
            pm = pm.contiguous()
        p.pad_mask = pm.data_ptr()
        p.pad_stride_b = pm.stride(0)
        keep.append(pm)
    p.impl = _lib.IMPL_BY_NAME[impl]
    return p, tuple(keep)


def _workspace(p, device, entry: str, *args) -> Optional[torch.Tensor]:
    """Size (by ``<entry>_workspace_bytes(*args)``), allocate and attach the workspace of the launch ``p`` describes.
    Returns the tensor, to be kept until the launch is enqueued, or None when the launch needs no bytes.  torch aligns
    every block to 512 bytes, beyond the 256 the backward and dropout forward entry points require."""
    query = entry + "_workspace_bytes"
    need = C.c_size_t(0)
    check(getattr(_lib.lib(), query)(*args, C.byref(need)), query)
    if not need.value:
        return None
    ws = torch.empty(need.value, dtype=torch.uint8, device=device)
    p.workspace, p.workspace_bytes = ws.data_ptr(), need.value
    return ws


def _run_attn(p: AttnParams, device) -> None:
    ws = _workspace(p, device, "pcv_attn", C.byref(p))
    check(_lib.lib().pcv_attn_fwd(C.byref(p), _stream()), "pcv_attn_fwd")
    del ws


def _new_output(p, dtype: torch.dtype, device) -> torch.Tensor:
    """A new (B, N, H*dv) output for the launch ``p`` describes, attached to it."""
    out = torch.empty(p.B, p.N, p.H * p.dv, dtype=dtype, device=device)
    p.out = out.data_ptr()
    p.o_stride_b, p.o_stride_n, p.o_stride_h = out.stride(0), out.stride(1), p.dv
    return out


def _partial_state(p, device, out=None):
    """The float32 partial state (part_o (B,H,N,dv), part_m (B,H,N), part_l (B,H,N)) the launch ``p`` describes writes,
    attached to it: the caller's ``out`` tensors, checked, or new ones."""
    if out is not None:
        part_o, part_m, part_l = out
        if (tuple(part_o.shape) != (p.B, p.H, p.N, p.dv) or tuple(part_m.shape) != (p.B, p.H, p.N)
                or tuple(part_l.shape) != (p.B, p.H, p.N)):
            raise ValueError("attention_partial: `out` tensors have the wrong shape")
        for t in out:
            if t.dtype != torch.float32 or not t.is_contiguous() or not t.is_cuda:
                raise ValueError("attention_partial: `out` tensors must be contiguous float32 CUDA tensors")
    else:
        part_o = torch.empty(p.B, p.H, p.N, p.dv, dtype=torch.float32, device=device)
        part_m = torch.empty(p.B, p.H, p.N, dtype=torch.float32, device=device)
        part_l = torch.empty(p.B, p.H, p.N, dtype=torch.float32, device=device)
    p.write_partial = 1
    p.part_o, p.part_m, p.part_l = part_o.data_ptr(), part_m.data_ptr(), part_l.data_ptr()
    return part_o, part_m, part_l


def _check_stats(p, stat_m, stat_l) -> None:
    """The forward's row statistics, as the launch ``p`` describes them: contiguous float32 (B, H, N)."""
    for name, t in (("stat_m", stat_m), ("stat_l", stat_l)):
        if tuple(t.shape) != (p.B, p.H, p.N) or t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous float32 (B, H, N) tensor")


def _prep(q, k, v, *more, num_heads: Optional[int] = None, pad: bool = False):
    """Attention operands on the kernels' terms -> ``(q, k, v, *more, dims)``.

    Every operand must be on CUDA; it is cast to the compute dtype of q (fp32 -> bf16) and given unit channel stride.
    ``more`` are (B, N, H*dv) tensors that go with v (the backward's out and grad_out).  With ``pad``, head dims that are
    not multiples of 8 are zero-padded per head (``_pad_heads_to8``) and every operand is returned as (B, L, H*d8), so
    that the tensor-core kernels (TMA) can take them: zero channels change neither the scores, nor the first dv channels
    of P V, nor delta = rowsum(dO * O), nor the dropout mask.  ``dims`` is then the true (dqk, dv), to slice results back
    with ``_unpad_heads``; it is None when nothing was padded."""
    ts = (q, k, v) + more
    _require_cuda(*ts)
    cdt = _compute_dtype(q.dtype)
    ts = tuple(_rows_contiguous(t if t.dtype == cdt else t.to(cdt)) for t in ts)
    dims = None
    if pad:
        dqk, dv = _head_dim(q, num_heads), _head_dim(v, num_heads)
        if dqk % 8 or dv % 8:
            dims = (dqk, dv)
            ts = tuple(_pad_heads_to8(t, num_heads).flatten(2) for t in ts)
    return ts + (dims,)


def _unpad_heads(t: torch.Tensor, num_heads: int, d: int) -> torch.Tensor:
    """The first ``d`` channels of every head of a result computed from ``_prep(pad=True)`` operands: a (B, L, H*d8)
    output or gradient, or a (B, H, N, d8) partial numerator."""
    if t.dim() == 4:
        return t[..., :d]
    return t.unflatten(2, (num_heads, -1))[..., :d].flatten(2)


def _pad_heads_to8(t: torch.Tensor, num_heads: int) -> torch.Tensor:
    """(B, L, H*d) or (B, L, H, d) with d % 8 != 0 -> zero-padded (B, L, H, d8) copy, d8 = next multiple of 8.

    TMA needs 16-byte strides; zero channels change neither q.k nor the first d channels of P.V (the MNIST
    encoder has d = 131, the optical-flow encoder d = 322)."""
    if t.dim() == 3:
        t = t.reshape(t.shape[0], t.shape[1], num_heads, t.shape[2] // num_heads)
    d = t.shape[3]
    return torch.nn.functional.pad(t, (0, (-d) % 8))


def _head_dim(t: torch.Tensor, num_heads: int) -> int:
    return t.shape[2] // num_heads if t.dim() == 3 else t.shape[3]


def _attention_forward(q, k, v, num_heads, scale, pad_mask, causal, impl):
    out_dtype = q.dtype
    q, k, v, dims = _prep(q, k, v, num_heads=num_heads, pad=impl != "simt")
    _require_cuda(pad_mask)
    with torch.cuda.device(k.device):
        p, keep = _fill_attn_params(q, k, v, num_heads, scale, pad_mask, causal, None, 0, impl)
        out = _new_output(p, q.dtype, k.device)
        _run_attn(p, k.device)
    del keep
    if dims is not None:
        out = _unpad_heads(out, num_heads, dims[1])
    return out if out.dtype == out_dtype else out.to(out_dtype)


#: Budget of the backward shim: the largest fp32 score block (B, H, N, chunk) it materialises at a time.
# "impl": "auto" = the tcgen05 backward kernels (pcv_attn_bwd) whenever they cover the call, else the torch shim;
# "kernel" = kernels or raise; "shim" = always the shim.  "max_score_bytes" bounds the shim's score chunk.
backward_config = {"max_score_bytes": 1 << 30, "impl": "auto"}


def _fill_bwd_params(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal, dropout_p,
                     dropout_seed):
    """Backward parameters of prepared operands, with the strides of dense (B, L, H*d) gradients but no gradient
    pointers yet."""
    ap, keep = _fill_attn_params(q, k, v, num_heads, scale, pad_mask, causal, None, 0, "auto")
    B, H, N, M, dqk, dv = ap.B, ap.H, ap.N, ap.M, ap.dqk, ap.dv
    for name, t in (("out", out), ("grad_out", grad_out)):
        if tuple(t.shape) != (B, N, H * dv) or t.stride(2) != 1:
            raise ValueError(f"{name} must be a (B, N, H*dv) tensor with unit channel stride, got {tuple(t.shape)}")
    _check_stats(ap, stat_m, stat_l)
    p = _lib.AttnBwdParams()
    p.q, p.k, p.v, p.out, p.grad_out = ap.q, ap.k, ap.v, out.data_ptr(), grad_out.data_ptr()
    p.stat_m, p.stat_l = stat_m.data_ptr(), stat_l.data_ptr()
    for f in ("q_stride_b", "q_stride_n", "q_stride_h", "k_stride_b", "k_stride_m", "k_stride_h",
              "v_stride_b", "v_stride_m", "v_stride_h"):
        setattr(p, f, getattr(ap, f))
    p.o_stride_b, p.o_stride_n, p.o_stride_h = out.stride(0), out.stride(1), dv
    p.go_stride_b, p.go_stride_n, p.go_stride_h = grad_out.stride(0), grad_out.stride(1), dv
    p.gq_stride_b, p.gq_stride_n, p.gq_stride_h = N * H * dqk, H * dqk, dqk
    p.gk_stride_b, p.gk_stride_m, p.gk_stride_h = M * H * dqk, H * dqk, dqk
    p.gv_stride_b, p.gv_stride_m, p.gv_stride_h = M * H * dv, H * dv, dv
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.scale, p.dtype, p.causal = float(scale), ap.dtype, ap.causal
    p.pad_mask, p.pad_stride_b = ap.pad_mask, ap.pad_stride_b
    p.dropout_p, p.dropout_seed = float(dropout_p), int(dropout_seed)
    return p, keep + (out, grad_out, stat_m, stat_l)


def _backward_kernels(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal, dropout_p,
                      dropout_seed, shard, mode):
    """pcv_attn_bwd, or pcv_attn_bwd_shard for a key shard ``shard = (m_total, m_offset)``, on operands ``_prep``
    prepared -> (grad_q, grad_k, grad_v); a shard's grad_q is its fp32 contribution grad_q32.  ``mode`` as in
    ``_backward``.  The support check and the launch read the same params; the check allocates no gradient."""
    lib = _lib.lib()
    with torch.cuda.device(k.device):
        p, keep = _fill_bwd_params(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal,
                                   dropout_p, dropout_seed)
        entry, args = "pcv_attn_bwd", (C.byref(p),)
        if shard is not None:
            s = _lib.KeyShard()
            s.m_total, s.m_offset = int(shard[0]), int(shard[1])
            entry, args = "pcv_attn_bwd_shard", (C.byref(p), C.byref(s))
        if mode != "run":
            if shard is not None:  # the check reads only the alignment of grad_q32
                placeholder = torch.empty(16, device=k.device)
                s.grad_q32 = placeholder.data_ptr()
            ok = bool(getattr(lib, entry + "_supported")(*args))
            if mode == "check" or not ok:
                return ok if mode == "check" else None
        gq = torch.empty(q.shape[0], p.N, p.H * p.dqk, dtype=q.dtype if shard is None else torch.float32,
                         device=k.device)
        gk = torch.empty(p.B, p.M, p.H * p.dqk, dtype=q.dtype, device=k.device)
        gv = torch.empty(p.B, p.M, p.H * p.dv, dtype=q.dtype, device=k.device)
        p.grad_k, p.grad_v = gk.data_ptr(), gv.data_ptr()
        if shard is None:
            p.grad_q = gq.data_ptr()
        else:
            s.grad_q32 = gq.data_ptr()
        ws = _workspace(p, k.device, entry, *args)
        check(getattr(lib, entry)(*args, _stream()), entry)
    del keep, ws
    return gq, gk, gv


def _backward(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal, dropout_p, dropout_seed,
              shard=None, mode="try", pad=True):
    """The backward kernels (of the key shard ``shard = (m_total, m_offset)``) with the operands prepared once.  With
    ``pad``, head dims that are not multiples of 8 are zero-padded per head, as the forward padded them, and the
    gradients of the padding channels dropped.  mode "check": whether the kernels cover the call; "run": the gradients
    (an uncovered call raises); "try": the gradients, or None where the kernels do not cover the call."""
    q, k, v, out, grad_out, dims = _prep(q, k, v, out, grad_out, num_heads=num_heads, pad=pad)
    _require_cuda(stat_m, stat_l, pad_mask)
    grads = _backward_kernels(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal, dropout_p,
                              dropout_seed, shard, mode)
    if mode == "check" or grads is None or dims is None:
        return grads
    dqk, dv = dims
    return tuple(_unpad_heads(g, num_heads, d) for g, d in zip(grads, (dqk, dqk, dv)))


def attention_backward(q, k, v, out, grad_out, stat_m, stat_l, num_heads: int, scale: float, pad_mask=None,
                       causal: bool = False, check_only: bool = False, dropout_p: float = 0.0, dropout_seed: int = 0):
    """Gradients (grad_q, grad_k, grad_v) of ``attention`` on the tcgen05 backward kernels (pcv_attn_bwd): head dims
    that are multiples of 8, up to 192.  Above 128, grad_q is summed in a fixed order (bitwise reproducible).

    ``out`` is the forward output, ``stat_m`` / ``stat_l`` the (B, H, N) row statistics of ``attention_partial`` over all
    keys.  grad_q has q's batch size (a batch-1 ``q`` shared by the batch receives the sum).  ``check_only`` launches
    nothing and returns whether the kernels cover these operands.  ``dropout_p`` / ``dropout_seed``: the values the
    dropout forward (``attention_partial`` or ``attention_dropout_forward``) ran with — the kernels regenerate its
    mask."""
    return _backward(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal, dropout_p, dropout_seed,
                     mode="check" if check_only else "run", pad=False)


def attention_backward_shard(q, k, v, out, grad_out, stat_m, stat_l, num_heads: int, scale: float, m_total: int,
                             m_offset: int, pad_mask=None, causal: bool = False, dropout_p: float = 0.0,
                             dropout_seed: int = 0, check_only: bool = False):
    """Backward of one key shard (pcv_attn_bwd_shard) -> (grad_q32, grad_k, grad_v).

    ``k`` / ``v`` / ``pad_mask`` hold the keys [m_offset, m_offset + M) of ``m_total`` (m_offset even); ``stat_m`` /
    ``stat_l`` are the row statistics MERGED over all keys and ``out`` the merged output.  grad_k / grad_v are this
    shard's gradients; grad_q32 is its fp32 contribution to grad_q (q's batch size): the sum over all shards is grad_q.
    Head dims up to 192; those that are not multiples of 8 are zero-padded as in the autograd backward.  ``check_only``
    launches nothing and returns whether the kernels cover these operands."""
    return _backward(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal, dropout_p, dropout_seed,
                     shard=(m_total, m_offset), mode="check" if check_only else "run")


def _attention_grads(q, k, v, out, grad_out, pm, pl, num_heads: int, scale: float, pad_mask, causal: bool,
                     dropout_p: float, dropout_seed: int, shard=None):
    """The gradients of attention, or of the key shard ``shard = (m_total, m_offset)`` (grad_q then being its
    contribution), as ``backward_config["impl"]`` selects: the backward kernels, or the torch shim."""
    mode = backward_config["impl"]
    if mode not in ("auto", "kernel", "shim"):
        raise ValueError(f"backward_config['impl'] = {mode!r}")
    if mode != "shim":
        grads = None
        if pm is not None and q.is_cuda and q.dim() == 3 and k.dim() == 3 and v.dim() == 3:
            grads = _backward(q, k, v, out, grad_out, pm, pl, num_heads, scale, pad_mask, causal, dropout_p,
                              dropout_seed, shard)
        if grads is not None:
            return grads
        if mode == "kernel":
            entry = "pcv_attn_bwd" if shard is None else "pcv_attn_bwd_shard"
            raise RuntimeError(f"backward_config['impl'] = 'kernel' but {entry} does not cover this call: "
                               + _lib.lib().pcv_last_error().decode())
    m_total, m_offset = (None, 0) if shard is None else shard
    return _backward_shim(q, k, v, out, grad_out, pm, pl, num_heads, scale, pad_mask, causal, dropout_p, dropout_seed,
                          m_total, m_offset)


def new_dropout_seed() -> int:
    """A fresh 62-bit seed from torch's CPU generator: reproducible under ``torch.manual_seed``, no device sync."""
    return int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())


def attention_dropout_forward(q, k, v, stat_m, stat_l, num_heads: int, scale: float, dropout_p: float, dropout_seed: int,
                              pad_mask=None, causal: bool = False, check_only: bool = False):
    """out = dropout(softmax(...)) V for training (reference modules.py:161): the dropout forward of
    ``attention_partial`` (pcv_attn_fwd_partial_dropout) over all keys, then ``combine_partials``.  The kernel recomputes
    the row statistics, so ``stat_m`` / ``stat_l`` (the (B, H, N) part_m / part_l of ``attention_partial`` over all
    keys) are only checked, when given, to be the statistics the backward would take.  The keep decision of every
    (b, h, query, key) is a pure function of ``dropout_seed`` (``dropout_keep_mask`` exports it); the drop probability is
    ``dropout_p`` rounded to 1/256.  ``check_only``: launch nothing, return whether the kernel covers the operands."""
    out_dtype = q.dtype
    q, k, v, _ = _prep(q, k, v)
    _require_cuda(stat_m, stat_l, pad_mask)
    if check_only:
        return _partial_dropout_supported(q, k, v, num_heads, pad_mask, causal, dropout_p, "auto")
    if stat_m is not None or stat_l is not None:
        _check_stats(_fill_attn_params(q, k, v, num_heads, scale, pad_mask, causal, None, 0, "auto")[0], stat_m, stat_l)
    po, pm, pl = attention_partial(q, k, v, num_heads, scale, pad_mask=pad_mask, causal=causal, dropout_p=dropout_p,
                                   dropout_seed=dropout_seed)
    out = combine_partials(po[None], pm[None], pl[None], q.dtype)
    return out if out.dtype == out_dtype else out.to(out_dtype)


def dropout_keep_mask(B: int, H: int, N: int, M: int, dropout_p: float, dropout_seed: int, device="cuda",
                      key_begin: int = 0, key_end: Optional[int] = None) -> torch.Tensor:
    """(B, H, N, key_end - key_begin) bool keep mask the dropout kernels use for this seed over the keys
    [key_begin, key_end) (default: all M keys) — pcv_attn_dropout_mask_range."""
    key_end = M if key_end is None else int(key_end)
    keep = torch.empty(B, H, N, max(key_end - key_begin, 0), dtype=torch.uint8, device=device)
    with torch.cuda.device(keep.device):
        check(_lib.lib().pcv_attn_dropout_mask_range(keep.data_ptr(), B, H, N, int(key_begin), key_end, float(dropout_p),
                                                     int(dropout_seed), _stream()), "pcv_attn_dropout_mask_range")
    return keep.bool()


def _dropout_keep(B: int, H: int, N: int, key_begin: int, key_end: int, dropout_p: float, dropout_seed: int,
                  device) -> torch.Tensor:
    """The backward shim's view of the dropout mask: keys [key_begin, key_end) as a (B, H, N, key_end - key_begin) bool
    tensor on `device`.  The one place the shim fetches the mask (a CPU test substitutes the numpy oracle here)."""
    if torch.device(device).type != "cuda":
        raise RuntimeError(f"attention dropout: the mask is generated on the GPU, got tensors on {device}")
    return dropout_keep_mask(B, H, N, key_end, dropout_p, dropout_seed, device=device, key_begin=key_begin,
                             key_end=key_end)


def _dropout_scale(dropout_p: float) -> float:
    """The survivors' scale 256 / (256 - thresh) of the kernels, thresh = clamp(lround(256 p), 1, 255) of the float32 p."""
    p32 = struct.unpack("f", struct.pack("f", float(dropout_p)))[0]
    return 256.0 / (256.0 - min(255, max(1, int(math.floor(p32 * 256.0 + 0.5)))))


def _partial_dropout_supported(q, k, v, num_heads: int, pad_mask, causal: bool, dropout_p: float, impl: str) -> bool:
    """Whether the dropout forward (attention_partial with dropout_p > 0) takes these prepared operands."""
    with torch.cuda.device(k.device):
        p, keep = _fill_attn_params(q, k, v, num_heads, 1.0, pad_mask, causal, None, 0, impl)
        dummy = torch.empty(16, device=k.device)
        p.write_partial = 1
        p.part_o = p.part_m = p.part_l = dummy.data_ptr()
        return bool(_lib.lib().pcv_attn_fwd_partial_dropout_supported(C.byref(p), float(dropout_p)))


class _FusedAttention(torch.autograd.Function):
    """Forward = the fused CUDA kernel (partial-state mode, so the row max and denominator are kept).  With dropout:
    the dropout forward (``attention_partial`` with ``dropout_p``) on the single-CTA tensor-core kernel, whichever other
    kernel ``impl`` names, for every head dim that kernel takes.
    Backward = the tensor-core backward kernels (pcv_attn_bwd: dK/dV and dQ kernels, SURVEY.md §8(f) rank 2) for head
    dims up to 192; head dims that are not multiples of 8 are zero-padded as in the forward (``_backward``).  Other
    shapes (head dims above 192, the decode forward) take the labelled SHIM below: the
    flash-attention backward recurrence in plain torch ops, chunked over the key axis from the saved statistics,
    memory bounded by ``backward_config["max_score_bytes"]``, with dropout regenerating the mask of each key chunk
    (``_dropout_keep``); neither path ever holds the (B, H, N, M) score tensor (8.6 GB at the north-star shape).
    The inference forward never routes through this class."""

    @staticmethod
    def forward(ctx, q, k, v, num_heads, scale, pad_mask, causal, impl, dropout_p=0.0, dropout_seed=0):
        ctx.dropout = (float(dropout_p), int(dropout_seed))
        ctx.meta = (num_heads, scale, causal)
        if impl == "decode" and not dropout_p > 0.0:
            # the decode kernel keeps no partial state: plain forward, statistics recomputed by the shim
            out = _attention_forward(q, k, v, num_heads, scale, pad_mask, causal, impl)
            ctx.save_for_backward(q, k, v, pad_mask, out, None, None)
            return out
        # head dims that are not multiples of 8 are zero-padded, so that the statistics exist for the backward kernels
        qc, kc, vc, dims = _prep(q, k, v, num_heads=num_heads, pad=True)
        if dropout_p > 0.0:
            impl = impl if impl == "tcgen05" else "auto"  # only the single-CTA tensor-core kernel takes dropout
            if not _partial_dropout_supported(qc, kc, vc, num_heads, pad_mask, causal, dropout_p, impl):
                raise NotImplementedError("attention dropout is not available for this call: "
                                          + _lib.lib().pcv_last_error().decode())
        # the (dropped) numerator and the dropout-free statistics, merged by the combine kernel
        po, pm, pl = attention_partial(qc, kc, vc, num_heads, scale, pad_mask=pad_mask, causal=causal, impl=impl,
                                       dropout_p=dropout_p, dropout_seed=dropout_seed)
        out = combine_partials(po[None], pm[None], pl[None], qc.dtype)
        del po
        if dims is not None:
            out = _unpad_heads(out, num_heads, dims[1])
        out = out if out.dtype == q.dtype else out.to(q.dtype)
        ctx.save_for_backward(q, k, v, pad_mask, out, pm, pl)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        q, k, v, pad_mask, out, pm, pl = ctx.saved_tensors
        H, scale, causal = ctx.meta
        drop_p, drop_seed = getattr(ctx, "dropout", (0.0, 0))
        gq, gk, gv = _attention_grads(q, k, v, out, grad_out, pm, pl, H, scale, pad_mask, causal, drop_p, drop_seed)
        return gq.to(q.dtype), gk.to(k.dtype), gv.to(v.dtype), None, None, None, None, None, None, None


def _backward_shim(q, k, v, out, grad_out, pm, pl, H: int, scale: float, pad_mask, causal: bool, drop_p: float,
                   drop_seed: int, m_total: Optional[int] = None, m_offset: int = 0):
    """TRAINING-SUPPORT SHIM: the flash-attention backward recurrence in plain torch ops, chunked over the key axis
    (see ``_FusedAttention``).  -> fp32 (grad_q, grad_k, grad_v); grad_q has q's batch size (summed for a batch-1 q).

    ``k`` / ``v`` / ``pad_mask`` may be the keys [m_offset, m_offset + M) of ``m_total`` (default: all keys): the causal
    diagonal and the dropout mask then take global key indices, and ``pm`` / ``pl`` / ``out`` must be the statistics
    and output merged over all ``m_total`` keys; grad_q is this shard's contribution."""
    B, M = k.shape[0], k.shape[1]
    N = q.shape[1]
    m_total = M if m_total is None else int(m_total)
    cdt = _compute_dtype(q.dtype)
    # the kernel saw operands rounded to the compute dtype: differentiate the same function
    qh = q.to(cdt).float().expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)      # (B,H,N,dqk)
    kh = k.to(cdt).float().reshape(B, M, H, -1).transpose(1, 2)                         # (B,H,M,dqk)
    vh = v.to(cdt).float().reshape(B, M, H, -1).transpose(1, 2)                         # (B,H,M,dv)
    go = grad_out.float().reshape(B, N, H, -1).transpose(1, 2)                          # (B,H,N,dv)
    oh = out.float().reshape(B, N, H, -1).transpose(1, 2)
    t_scale = scale * 1.4426950408889634
    neg = -torch.finfo(torch.float32).max
    chunk = max(128, int(backward_config["max_score_bytes"] // (4 * B * H * N)) // 128 * 128)

    def scores(j0, j1):  # log2-domain scores with the reference's finite mask fill, and the fill mask
        t = torch.matmul(qh, kh[:, :, j0:j1].transpose(-1, -2)) * t_scale
        filled = None
        if pad_mask is not None:
            filled = pad_mask[:, j0:j1].bool()[:, None, None, :].expand(B, 1, N, j1 - j0)
        if causal:
            rows = torch.arange(N, device=t.device)[:, None] + (m_total - N - m_offset)
            cm = (torch.arange(j0, j1, device=t.device)[None, :] > rows)[None, None]
            filled = cm if filled is None else (filled | cm)
        if filled is not None:
            t = t.masked_fill(filled, neg)
        return t, filled

    if pm is None:  # statistics were not saved: one chunked pass to rebuild them
        m_run = torch.full((B, H, N), -float("inf"), device=q.device)
        l_run = torch.zeros(B, H, N, device=q.device)
        for j0 in range(0, M, chunk):
            t, _ = scores(j0, min(M, j0 + chunk))
            m_new = torch.maximum(m_run, t.amax(-1))
            l_run = l_run * torch.exp2(m_run - m_new) + torch.exp2(t - m_new[..., None]).sum(-1)
            m_run = m_new
        pm, pl = m_run, l_run
    delta = (go * oh).sum(-1)                                                            # (B,H,N)
    gq = torch.zeros_like(qh)
    gk = torch.empty_like(kh)
    gv = torch.empty_like(vh)
    inv_l = 1.0 / pl
    for j0 in range(0, M, chunk):
        j1 = min(M, j0 + chunk)
        t, filled = scores(j0, j1)
        p = torch.exp2(t - pm[..., None]) * inv_l[..., None]                             # (B,H,N,c) probabilities
        dp = torch.matmul(go, vh[:, :, j0:j1].transpose(-1, -2))
        if drop_p > 0.0:  # O = (P o K r) V:  dV = (P o K r)^T dO,  dP = (dO V^T) o K r
            kr = (_dropout_keep(B, H, N, m_offset + j0, m_offset + j1, drop_p, drop_seed, k.device).to(p.dtype)
                  * _dropout_scale(drop_p))
            gv[:, :, j0:j1] = torch.matmul((p * kr).transpose(-1, -2), go)
            dp = dp * kr
        else:
            gv[:, :, j0:j1] = torch.matmul(p.transpose(-1, -2), go)
        ds = p * (dp - delta[..., None])
        if filled is not None:
            ds = ds.masked_fill(filled, 0.0)  # a filled score is a constant (masked_fill_): no gradient through it
        gq += torch.matmul(ds, kh[:, :, j0:j1])
        gk[:, :, j0:j1] = torch.matmul(ds.transpose(-1, -2), qh)
    gq = (gq * scale).transpose(1, 2).reshape(B, N, -1)
    if q.shape[0] == 1 and B > 1:
        gq = gq.sum(0, keepdim=True)
    gk = (gk * scale).transpose(1, 2).reshape(B, M, -1)
    gv = gv.transpose(1, 2).reshape(B, M, -1)
    return gq, gk, gv


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, num_heads: int, scale: float,
              pad_mask: Optional[torch.Tensor] = None, causal: bool = False, impl: str = "auto",
              dropout_p: float = 0.0, dropout_seed: Optional[int] = None) -> torch.Tensor:
    """softmax(scale * Q K^T + masks) V with heads split by stride.

    q: (B or 1, N, H*dqk), k: (B, M, H*dqk), v: (B, M, H*dv) -> (B, N, H*dv).
    Semantics of the reference's ``MultiHeadAttention.forward`` lines 123-167
    (/root/reference/perceiver/model/core/modules.py): q is scaled by ``scale``, ``pad_mask`` (True =
    padding) and the right-aligned causal mask use the finite fill ``-finfo.max``.  ``dropout_p`` > 0 applies the
    reference's dropout on the attention probabilities (:161) with a counter-based mask derived from
    ``dropout_seed`` (default: a fresh seed from torch's CPU generator), for every head dim the forward takes (up to
    512).  Under autograd the backward runs on the tensor-core kernels for head dims up to 192 (odd ones zero-padded
    to multiples of 8), above that on the torch shim.
    """
    if dropout_p > 0.0:
        if not 0.0 < dropout_p < 1.0:
            raise ValueError(f"dropout_p must be in [0, 1), got {dropout_p}")
        seed =new_dropout_seed() if dropout_seed is None else int(dropout_seed)
        return _FusedAttention.apply(q, k, v, num_heads, scale, pad_mask, causal, impl, float(dropout_p), seed)
    if torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad):
        return _FusedAttention.apply(q, k, v, num_heads, scale, pad_mask, causal, impl)
    return _attention_forward(q, k, v, num_heads, scale, pad_mask, causal, impl)


def attention_partial(q, k, v, num_heads: int, scale: float, pad_mask=None, causal: bool = False,
                      m_total: Optional[int] = None, m_offset: int = 0, impl: str = "auto", out=None,
                      dropout_p: float = 0.0, dropout_seed: int = 0):
    """One M-shard's un-normalised softmax state: (part_o (B,H,N,dv) f32, part_m (B,H,N), part_l (B,H,N)).

    ``k``/``v``/``pad_mask`` hold this shard's keys [m_offset, m_offset+M) of ``m_total``.  ``out`` may
    supply the three (contiguous, float32) destination tensors.  ``dropout_p`` > 0: the dropout forward
    (pcv_attn_fwd_partial_dropout, or pcv_attn_fwd_partial_dropout_shard on a key shard, m_offset even) — part_o is
    the numerator with the mask of ``dropout_keep_mask`` over the shard's global key range applied and scaled by
    1/(1-p), part_m / part_l stay the dropout-free statistics."""
    q, k, v, _ = _prep(q, k, v)
    with torch.cuda.device(k.device):
        p, keep = _fill_attn_params(q, k, v, num_heads, scale, pad_mask, causal, m_total, m_offset, impl)
        state = _partial_state(p, k.device, out)
        if dropout_p > 0.0:
            if p.impl == _lib.PCV_IMPL_AUTO:  # the dropout forward runs on the tensor-core kernel: size its workspace
                p.impl = _lib.PCV_IMPL_TCGEN05
            ws = _workspace(p, k.device, "pcv_attn", C.byref(p))
            entry = "pcv_attn_fwd_partial_dropout"
            if p.m_total != p.M or p.m_offset != 0:
                entry += "_shard"
            check(getattr(_lib.lib(), entry)(C.byref(p), float(dropout_p), int(dropout_seed), _stream()), entry)
            del ws
        else:
            _run_attn(p, k.device)
    del keep
    return state


def _fill_fp8_params(q8, k8, vt8, q_descale, k_descale, v_descale, num_heads, scale, pad_mask, causal, m_total,
                     m_offset, out_dtype):
    """(AttnParams, Fp8Attn, tensors to keep alive) of an FP8 forward; shapes as in :func:`attention_fp8`."""
    _require_cuda(q8, k8, vt8, q_descale, k_descale, v_descale, pad_mask)
    f8 = torch.float8_e4m3fn
    for name, t in (("q8", q8), ("k8", k8), ("vt8", vt8)):
        if t.dtype != f8:
            raise ValueError(f"attention_fp8: {name} must be torch.float8_e4m3fn, got {t.dtype}")
    if vt8.dim() != 4 or vt8.stride(3) != 1:
        raise ValueError("attention_fp8: vt8 must be (B, H, dv, M_pad) with contiguous keys")
    B, H, dv, m_pad = vt8.shape
    if H != num_heads:
        raise ValueError(f"attention_fp8: vt8 has {H} heads, expected {num_heads}")
    q8, k8 = _rows_contiguous(q8), _rows_contiguous(k8)
    # the (B, M, H, d) geometry of q / k; v is described by the Fp8Attn strides (its AttnParams strides are unused)
    v_geom = vt8.as_strided((B, k8.shape[1], H, dv), (0, 0, 0, 1))
    p, keep = _fill_attn_params(q8, k8, v_geom, num_heads, scale, pad_mask, causal, m_total, m_offset, "tcgen05",
                                dtype=_lib.PCV_E4M3)
    if m_pad < p.M:
        raise ValueError(f"attention_fp8: vt8 holds {m_pad} keys, fewer than the {p.M} of k8")
    p.v = vt8.data_ptr()
    p.v_stride_b = p.v_stride_m = p.v_stride_h = 0
    qd, kd = q_descale.float().contiguous(), k_descale.float().contiguous()
    vd = v_descale.float().contiguous()
    if qd.shape != (H,) or kd.shape != (H,) or vd.shape != (H, dv):
        raise ValueError(f"attention_fp8: descales must be (H,), (H,) and (H, dv) = ({H},), ({H},), ({H}, {dv})")
    f = _lib.Fp8Attn()
    f.q_descale, f.k_descale, f.v_descale = qd.data_ptr(), kd.data_ptr(), vd.data_ptr()
    f.vt_stride_b, f.vt_stride_h, f.vt_stride_c = vt8.stride(0), vt8.stride(1), vt8.stride(2)
    f.out_dtype = _pcv_dtype(out_dtype)
    return p, f, keep + (q8, k8, vt8, qd, kd, vd)


def attention_fp8_supported(q8, k8, vt8, q_descale, k_descale, v_descale, num_heads: int, scale: float = 1.0,
                            pad_mask=None, causal: bool = False, m_total: Optional[int] = None, m_offset: int = 0,
                            out_dtype: torch.dtype = torch.bfloat16, partial: bool = False) -> bool:
    """Whether :func:`attention_fp8` covers these operands (no launch; the reason is in ``_lib.lib().pcv_last_error()``)."""
    with torch.cuda.device(k8.device):
        p, f, keep = _fill_fp8_params(q8, k8, vt8, q_descale, k_descale, v_descale, num_heads, scale, pad_mask, causal,
                                      m_total, m_offset, out_dtype)
        dummy = torch.empty(64, device=k8.device)
        if partial:
            p.write_partial = 1
            p.part_o = p.part_m = p.part_l = dummy.data_ptr()
        else:
            p.out = dummy.data_ptr()
            p.o_stride_b, p.o_stride_n, p.o_stride_h = p.N * p.H * p.dv, p.H * p.dv, p.dv
        return bool(_lib.lib().pcv_attn_fwd_fp8_supported(C.byref(p), C.byref(f)))


def attention_fp8(q8, k8, vt8, q_descale, k_descale, v_descale, num_heads: int, scale: float, pad_mask=None,
                  causal: bool = False, m_total: Optional[int] = None, m_offset: int = 0,
                  out_dtype: torch.dtype = torch.bfloat16, partial: bool = False):
    """FP8 (e4m3) inference attention on already quantised operands (pcv_attn_fwd_fp8).

    q8: (B or 1, N, H*dqk), k8: (B, M, H*dqk) (or 4-D (B, L, H, d) views), vt8: V transposed, (B, H, dv, M_pad) with
    contiguous keys in order and M_pad >= M (a multiple of 16 keeps the strides TMA-aligned), all
    ``torch.float8_e4m3fn``.  The operands stand for ``q8 * q_descale[h]``, ``k8 * k_descale[h]`` and
    ``vt8[:, h, c] * v_descale[h, c]`` (float32 descales of shapes (H,), (H,), (H, dv)).  Masks and key sharding
    (``m_total`` / ``m_offset``) as in :func:`attention_partial`.  Each probability is rounded to e4m3 as
    ``e4m3(P * 2^8)`` relative to the running row maximum of its 128-key tile; the denominators are fp32 sums of the
    unrounded probabilities.  Returns (B, N, H*dv) in ``out_dtype`` (bf16 / fp16), or with ``partial`` the fp32 state
    ``(part_o, part_m, part_l)`` that :func:`combine_partials` merges.  Head dims: multiples of 16, dqk <= 256, dv <= 512.
    No autograd: this is an inference path."""
    with torch.cuda.device(k8.device):
        p, f, keep = _fill_fp8_params(q8, k8, vt8, q_descale, k_descale, v_descale, num_heads, scale, pad_mask, causal,
                                      m_total, m_offset, out_dtype)
        result = _partial_state(p, k8.device) if partial else _new_output(p, out_dtype, k8.device)
        ws = _workspace(p, k8.device, "pcv_attn", C.byref(p))
        check(_lib.lib().pcv_attn_fwd_fp8(C.byref(p), C.byref(f), _stream()), "pcv_attn_fwd_fp8")
    del keep, ws
    return result


def attention_sharded_fused(q, k, v, num_heads: int, scale: float, fuse, pad_mask=None, causal: bool = False,
                            m_total: Optional[int] = None, m_offset: int = 0, check_only: bool = False):
    """One launch: partial state of this rank's key shard + cross-GPU merge in the kernel tail (pcv_attn_fwd_sharded).

    ``fuse`` is a filled ``_lib.ShardFuse`` (symmetric-memory pointers of every rank, this call's epoch).  With
    ``check_only`` nothing is launched: returns whether the fused path covers these operands."""
    q, k, v, _ = _prep(q, k, v)
    with torch.cuda.device(k.device):
        p, keep = _fill_attn_params(q, k, v, num_heads, scale, pad_mask, causal, m_total, m_offset, "auto")
        p.write_partial = 1
        if check_only:
            dummy = torch.empty(16, device=k.device)
            p.part_o = p.part_m = p.part_l = dummy.data_ptr()
            return bool(_lib.lib().pcv_attn_fwd_sharded_supported(C.byref(p)))
        dummy_ptr = fuse.part[fuse.rank]
        p.part_o = p.part_m = p.part_l = dummy_ptr
        ws = _workspace(p, k.device, "pcv_attn", C.byref(p))
        check(_lib.lib().pcv_attn_fwd_sharded(C.byref(p), C.byref(fuse), _stream()), "pcv_attn_fwd_sharded")
    del keep, ws


def combine_partials(part_o: torch.Tensor, part_m: torch.Tensor, part_l: torch.Tensor,
                     out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """Merge G partial states (G,B,H,N,dv)/(G,B,H,N)/(G,B,H,N) -> (B, N, H*dv)."""
    _require_cuda(part_o, part_m, part_l)
    G, B, H, N, dv = part_o.shape
    part_o, part_m, part_l = part_o.contiguous(), part_m.contiguous(), part_l.contiguous()
    cdt = _compute_dtype(out_dtype)
    with torch.cuda.device(part_o.device):
        out = torch.empty(B, N, H * dv, dtype=cdt, device=part_o.device)
        p = CombineParams()
        p.part_o, p.part_m, p.part_l, p.out = part_o.data_ptr(), part_m.data_ptr(), part_l.data_ptr(), out.data_ptr()
        p.o_stride_b, p.o_stride_n, p.o_stride_h = out.stride(0), out.stride(1), dv
        p.num_parts, p.B, p.H, p.N, p.dv = G, B, H, N, dv
        p.dtype = _pcv_dtype(cdt)
        check(_lib.lib().pcv_attn_combine(C.byref(p), _stream()), "pcv_attn_combine")
    return out if cdt == out_dtype else out.to(out_dtype)


def merge_partials(part_o: torch.Tensor, part_m: torch.Tensor, part_l: torch.Tensor, out=None):
    """Merge G partial states (G,B,H,N,dv)/(G,B,H,N)/(G,B,H,N) into ONE un-normalised partial state
    (B,H,N,dv)/(B,H,N)/(B,H,N) — the local level of a two-level merge.  ``out`` may supply the destination tensors
    (e.g. views of a symmetric-memory buffer)."""
    _require_cuda(part_o, part_m, part_l)
    G, B, H, N, dv = part_o.shape
    part_o, part_m, part_l = part_o.contiguous(), part_m.contiguous(), part_l.contiguous()
    if out is None:
        out = (torch.empty(B, H, N, dv, dtype=torch.float32, device=part_o.device),
               torch.empty(B, H, N, dtype=torch.float32, device=part_o.device),
               torch.empty(B, H, N, dtype=torch.float32, device=part_o.device))
    for t in out:
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("merge_partials: `out` tensors must be contiguous float32")
    p = _lib.MergeParams()
    p.part_o, p.part_m, p.part_l = part_o.data_ptr(), part_m.data_ptr(), part_l.data_ptr()
    p.out_o, p.out_m, p.out_l = out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr()
    p.rows, p.num_parts, p.dv = B * H * N, G, dv
    with torch.cuda.device(part_o.device):
        check(_lib.lib().pcv_attn_merge_partials(C.byref(p), _stream()), "pcv_attn_merge_partials")
    return out


def rescale_partial_(part_o: torch.Tensor, part_m: torch.Tensor, part_l: torch.Tensor, new_m: torch.Tensor) -> None:
    """In place: re-express a partial state relative to the row maxima ``new_m`` (>= part_m)."""
    _require_cuda(part_o, part_m, part_l, new_m)
    for t in (part_o, part_m, part_l, new_m):
        if not t.is_contiguous() or t.dtype != torch.float32:
            raise ValueError("rescale_partial_ expects contiguous float32 tensors")
    p = RescaleParams()
    p.part_o, p.part_m, p.part_l, p.new_m = part_o.data_ptr(), part_m.data_ptr(), part_l.data_ptr(), new_m.data_ptr()
    p.rows, p.dv = part_m.numel(), part_o.shape[-1]
    with torch.cuda.device(part_o.device):
        check(_lib.lib().pcv_partial_rescale(C.byref(p), _stream()), "pcv_partial_rescale")


def _rotary_params(x: torch.Tensor, y: torch.Tensor, num_heads: int, angles: torch.Tensor, right_align: bool,
                   dtype: int) -> RotaryParams:
    """RotaryParams of y <- rotate(x), x and y (B, n, H*d), angles as :func:`_rotary_angles` leaves them."""
    B, n, Cx = x.shape
    d = Cx // num_heads
    p = RotaryParams()
    p.x, p.y, p.angles = x.data_ptr(), y.data_ptr(), angles.data_ptr()
    p.x_stride_b, p.x_stride_n, p.x_stride_h = x.stride(0), x.stride(1), d
    p.y_stride_b, p.y_stride_n, p.y_stride_h = y.stride(0), y.stride(1), d
    p.a_stride_b = 0 if (angles.shape[0] == 1 and B > 1) else angles.stride(0)
    p.a_stride_n = angles.stride(1)
    p.B, p.n, p.H, p.d = B, n, num_heads, d
    p.rotate_dim = angles.shape[-1]
    p.angle_row0 = (angles.shape[1] - n) if right_align else 0
    p.dtype = dtype
    return p


def _launch_rotary(p: RotaryParams, f=None, rows=None) -> None:
    """Enqueue the rotary launch ``p``: e4m3 output when ``f`` (RotaryFp8) is given, angle and output rows read from
    device memory when ``rows`` (DevRows) is (pcv_rotary_apply, _fp8, _at, _at_fp8)."""
    entry = "pcv_rotary_apply" + ("_at" if rows is not None else "") + ("_fp8" if f is not None else "")
    check(getattr(_lib.lib(), entry)(*(C.byref(s) for s in (p, f, rows) if s is not None), _stream()), entry)


def _rotary_angles(angles: torch.Tensor) -> torch.Tensor:
    """``frq_pos_enc`` (B or 1, [1,] n_angles, f) as the rotary kernels take it: 3-D float32, unit stride."""
    if angles.dim() == 4:  # (B, 1, n, f) as stored by RotaryPositionEmbedding
        angles = angles[:, 0]
    angles = angles.float()
    return angles if angles.stride(-1) == 1 else angles.contiguous()


def _rotary_forward(x: torch.Tensor, num_heads: int, angles: torch.Tensor, right_align: bool,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _require_cuda(x, angles)
    out_dtype = x.dtype
    cdt = _compute_dtype(x.dtype)
    x = _rows_contiguous(x if x.dtype == cdt else x.to(cdt))
    B, n, Cx = x.shape
    if out is not None:
        if out.shape != x.shape or out.dtype != cdt or out.stride(2) != 1:
            raise ValueError("rotary: `out` must match x in shape and compute dtype with unit channel stride")
        y = out
    else:
        y = torch.empty(B, n, Cx, dtype=cdt, device=x.device)
    if n == 0:
        return y if out is not None else y.to(out_dtype)
    p = _rotary_params(x, y, num_heads, angles, right_align, _pcv_dtype(cdt))
    with torch.cuda.device(x.device):
        _launch_rotary(p)
    if out is not None:
        return y
    return y if cdt == out_dtype else y.to(out_dtype)


class _Rotary(torch.autograd.Function):
    """Forward = pcv_rotary_apply.  Backward = TRAINING-SUPPORT SHIM in torch ops (like ``_FusedAttention``): the
    transpose of the pairwise rotation,  dx[2p] = dy[2p] cos a[2p] + dy[2p+1] sin a[2p+1],
    dx[2p+1] = dy[2p+1] cos a[2p+1] - dy[2p] sin a[2p],  channels beyond ``rotate_dim`` pass through.  Without it the
    rotated q / k would be constants for autograd and q_proj / k_proj of every rotary layer would get no gradient."""

    @staticmethod
    def forward(ctx, x, angles, num_heads, right_align):
        ctx.save_for_backward(angles)
        ctx.meta = (num_heads, right_align)
        return _rotary_forward(x, num_heads, angles, right_align)

    @staticmethod
    def backward(ctx, gy):
        (angles,) = ctx.saved_tensors
        H, right_align = ctx.meta
        B, n, Cx = gy.shape
        d, f = Cx // H, angles.shape[-1]
        a = angles[:, angles.shape[1] - n:] if right_align else angles[:, :n]
        a = a[:, :, None, :].float()                       # (Ba, n, 1, f)
        g = gy.float().reshape(B, n, H, d)
        gr = g[..., :f]
        ge, go = gr[..., 0::2], gr[..., 1::2]
        ae, ao = a[..., 0::2], a[..., 1::2]
        dxe = ge * torch.cos(ae) + go * torch.sin(ao)
        dxo = go * torch.cos(ao) - ge * torch.sin(ae)
        dx = torch.cat([torch.stack([dxe, dxo], dim=-1).flatten(-2), g[..., f:]], dim=-1)
        return dx.reshape(B, n, Cx).to(gy.dtype), None, None, None


def rotary(x: torch.Tensor, num_heads: int, angles: torch.Tensor, right_align: bool) -> torch.Tensor:
    """Rotate the first ``angles.shape[-1]`` channels of every head of x (B, n, H*d).

    ``angles`` is the reference's ``frq_pos_enc`` (B or 1, n_angles, rotate_dim); row selection follows
    /root/reference/perceiver/model/core/position.py:32-37 (last n rows if right_align else first n)."""
    _require_cuda(x, angles)
    angles = _rotary_angles(angles)
    B, n, _ = x.shape
    Ba, n_angles, _ = angles.shape
    if Ba not in (1, B):
        raise ValueError(f"angle batch {Ba} must be 1 or {B}")
    if n_angles < n:
        raise ValueError(f"rotary: {n_angles} angle rows for a sequence of {n}")
    if torch.is_grad_enabled() and x.requires_grad:
        return _Rotary.apply(x, angles, num_heads, bool(right_align))
    return _rotary_forward(x, num_heads, angles, bool(right_align))


class _KvArena:
    """Bookkeeping of a growing KV cache's backing buffer ``(B, capacity, C)``: the first unused row.  The arena is
    an attribute OF the buffer and refers back to it only weakly, so a superseded buffer is released by reference
    counting as soon as the last cache view of it is dropped (no tensor <-> arena cycle waiting for the cyclic GC)."""

    __slots__ = ("buf_ref", "used", "rot")

    def __init__(self, buf: torch.Tensor):
        import weakref

        self.buf_ref = weakref.ref(buf)
        self.used = 0
        self.rot = None  # rotated shadow of a K arena: dict(buf, lo, hi, key), see rotated_cache_keys


_ARENA_ATTR = "_pcv_kv_arena"
#: Arena policy of :func:`kv_append` (``enabled=False`` restores plain concat into exact-size tensors).
kv_arena_config = {"enabled": True, "growth": 1.5, "min_rows": 64}


def _arena_of(t: torch.Tensor):
    """``(arena, first_row)`` if ``t`` is a row range of an arena this module allocated, else ``None``.

    Views keep ``._base`` pointing at the root buffer through any chain of slices, so a cache the caller
    truncated (``k[:, -m:]``, core/huggingface.py:146-156) is still recognised; ``index_select`` (beam
    reordering, :140-144) yields a fresh tensor and is not."""
    root = t._base if t._base is not None else t
    arena = getattr(root, _ARENA_ATTR, None)
    if arena is None or arena.buf_ref() is not root or t.dim() != 3 or t.dtype != root.dtype:
        return None
    B, cap, C = root.shape
    if t.shape[0] != B or t.shape[2] != C or t.shape[1] == 0:
        return None
    if t.stride(2) != 1 or t.stride(1) != C or (B > 1 and t.stride(0) != cap * C):
        return None
    off = t.storage_offset() - root.storage_offset()
    if off < 0 or off % C or off // C + t.shape[1] > cap:
        return None
    return arena, off // C


def _arena_target(cache: torch.Tensor, n: int):
    """Where the appended cache lives: ``(dst_view (B, L+n, C), in_place)``.

    In place only when the cache is the row range that ends at the arena's frontier and ``n`` more rows
    fit: rows a caller may still hold are never overwritten, so the functional semantics of the
    reference's ``torch.cat`` (modules.py:117-121; two different continuations of one cache stay
    independent) are preserved.  Otherwise a new arena with head-room is allocated and the kernel copies
    the old rows once — amortised O(new rows) per decode step instead of O(cache)."""
    B, L, C = cache.shape
    hit = _arena_of(cache) if kv_arena_config["enabled"] else None
    if hit is not None:
        arena, start = hit
        root = cache._base if cache._base is not None else cache
        if start + L == arena.used and arena.used + n <= root.shape[1]:
            arena.used += n
            return root[:, start:start + L + n], True
    if not kv_arena_config["enabled"]:
        return torch.empty(B, L + n, C, dtype=cache.dtype, device=cache.device), False
    cap = max(int((L + n) * kv_arena_config["growth"]) + 1, kv_arena_config["min_rows"], L + n)
    cap = (cap + 63) // 64 * 64
    buf = torch.empty(B, cap, C, dtype=cache.dtype, device=cache.device)
    arena = _KvArena(buf)
    arena.used = L + n
    setattr(buf, _ARENA_ATTR, arena)
    return buf[:, :L + n], False


def _launch_kv_append(k_cache, v_cache, k_new, v_new, k_dst, v_dst, k_in_place, v_in_place, scales=None,
                      rows=None) -> None:
    """One launch: dst[:, :L] = cache (skipped for a half appended in place), dst[:, L:] = new rows.  ``scales``: the
    (k_inv_scale, v_inv_scale) of e4m3 caches (the new rows are quantised on the way in).  ``rows`` (DevRows, no cache):
    the new rows go to dst rows ``rows.bounds[0]`` on, read from device memory (pcv_kv_append, _fp8, _at, _at_fp8)."""
    codes = {torch.bfloat16: _lib.PCV_BF16, torch.float16: _lib.PCV_F16, torch.float32: _lib.PCV_F32}
    p = KvAppendParams()
    if k_cache is not None:
        # an in-place half passes its own destination as the cache pointer: the library skips that copy
        kc = k_dst if k_in_place else k_cache
        vc = v_dst if v_in_place else v_cache
        p.L_old = k_cache.shape[1]
        p.k_cache, p.v_cache = (kc.data_ptr(), vc.data_ptr()) if p.L_old else (None, None)
        p.kc_stride_b, p.kc_stride_l = kc.stride(0), kc.stride(1)
        p.vc_stride_b, p.vc_stride_l = vc.stride(0), vc.stride(1)
    p.k_new, p.v_new, p.k_dst, p.v_dst = k_new.data_ptr(), v_new.data_ptr(), k_dst.data_ptr(), v_dst.data_ptr()
    p.kn_stride_b, p.kn_stride_l = k_new.stride(0), k_new.stride(1)
    p.vn_stride_b, p.vn_stride_l = v_new.stride(0), v_new.stride(1)
    p.kd_stride_b, p.kd_stride_l = k_dst.stride(0), k_dst.stride(1)
    p.vd_stride_b, p.vd_stride_l = v_dst.stride(0), v_dst.stride(1)
    p.B, p.n, p.Ck, p.Cv = k_new.shape[0], k_new.shape[1], k_new.shape[2], v_new.shape[2]
    p.dtype = codes[k_new.dtype]
    f = None if scales is None else _lib.KvFp8Scales(k_inv_scale=scales[0].data_ptr(), v_inv_scale=scales[1].data_ptr())
    entry = "pcv_kv_append" + ("_at" if rows is not None else "") + ("_fp8" if f is not None else "")
    with torch.cuda.device(k_new.device):
        check(getattr(_lib.lib(), entry)(*(C.byref(s) for s in (p, f, rows) if s is not None), _stream()), entry)


def kv_append(k_cache: torch.Tensor, v_cache: torch.Tensor, k_new: torch.Tensor, v_new: torch.Tensor):
    """Functional KV-cache concat along dim 1 in one launch (reference modules.py:117-121).

    Returns ``(B, L_old+n, C)`` tensors that the 🤗-side cache consumers may slice / ``index_select`` freely
    (SURVEY.md §8(b) ownership) and that never alias rows of the inputs a caller could observe changing.
    They are row ranges of arenas with head-room (see :func:`_arena_target`): a decode loop that feeds the
    returned cache back in appends its new row in place instead of re-copying the whole cache every step."""
    _require_cuda(k_cache, v_cache, k_new, v_new)
    # torch.cat type-promotes (reference modules.py:119-121): under autocast the first cached step meets an fp32
    # empty cache and bf16 projections.  An EMPTY cache simply adopts the dtype of the new rows (so a decode loop
    # keeps its cache in the compute dtype); otherwise both sides are promoted like torch.cat would.
    def _common(cache, new):
        if cache.dtype == new.dtype:
            return cache, new
        if cache.shape[1] == 0:
            return cache.to(new.dtype), new
        dt_ = torch.promote_types(cache.dtype, new.dtype)
        return cache.to(dt_), new.to(dt_)

    k_cache, k_new = _common(k_cache, k_new)
    v_cache, v_new = _common(v_cache, v_new)
    if k_new.dtype != v_new.dtype:
        dt_ = torch.promote_types(k_new.dtype, v_new.dtype)
        k_cache, k_new, v_cache, v_new = (t.to(dt_) for t in (k_cache, k_new, v_cache, v_new))
    dt = k_new.dtype
    if dt not in (torch.bfloat16, torch.float16, torch.float32):
        raise RuntimeError(f"kv_append supports bf16/fp16/fp32 caches, got {dt}")
    return _append(k_cache, v_cache, k_new, v_new)


def _append(k_cache, v_cache, k_new, v_new, scales=None):
    """The arena step of :func:`kv_append` / :func:`kv_append_fp8`: destinations by :func:`_arena_target`, one launch."""
    k_cache, v_cache, k_new, v_new = (_rows_contiguous(t) for t in (k_cache, v_cache, k_new, v_new))
    L_old, n = k_cache.shape[1], k_new.shape[1]
    k_dst, k_in_place = _arena_target(k_cache, n)
    v_dst, v_in_place = _arena_target(v_cache, n)
    if L_old + n == 0:
        return k_dst, v_dst
    args = (k_cache, v_cache, k_new, v_new, k_dst, v_dst, k_in_place, v_in_place)
    if scales is None:
        _launch_kv_append(*args)
    else:
        _launch_kv_append(*args, scales=scales)
    return k_dst, v_dst


F8 = torch.float8_e4m3fn


def kv_append_fp8(k_cache: torch.Tensor, v_cache: torch.Tensor, k_new: torch.Tensor, v_new: torch.Tensor,
                  k_inv_scale: torch.Tensor, v_inv_scale: torch.Tensor):
    """:func:`kv_append` onto an FP8 (e4m3) KV cache, in one launch (pcv_kv_append_fp8).

    ``k_cache`` / ``v_cache`` are ``torch.float8_e4m3fn`` (B, L, C) caches, or empty caches of any dtype (the first
    append decides the cache dtype); ``k_new`` / ``v_new`` are bf16 / fp16 rows, stored as the codes of
    ``clamp(x.float() * inv_scale, +-448)`` (per-channel ``inv_scale`` (C,) float32, round to nearest even).  The result
    is a row range of an e4m3 arena with the functional semantics of :func:`kv_append`."""
    _require_cuda(k_cache, v_cache, k_new, v_new, k_inv_scale, v_inv_scale)
    k_cache, v_cache = (c.to(F8) if c.shape[1] == 0 else c for c in (k_cache, v_cache))
    if k_cache.dtype != F8 or v_cache.dtype != F8:
        raise ValueError(f"kv_append_fp8: the caches must be float8_e4m3fn or empty, got {k_cache.dtype} / {v_cache.dtype}")
    if k_new.dtype not in (torch.bfloat16, torch.float16) or v_new.dtype != k_new.dtype:
        raise ValueError(f"kv_append_fp8: new rows must be bf16 / fp16 of one dtype, got {k_new.dtype} / {v_new.dtype}")
    scales = tuple(t.float().contiguous() for t in (k_inv_scale, v_inv_scale))
    if scales[0].shape != (k_new.shape[-1],) or scales[1].shape != (v_new.shape[-1],):
        raise ValueError("kv_append_fp8: inverse scales must be (Ck,) and (Cv,)")
    return _append(k_cache, v_cache, k_new, v_new, scales)


#: Rotated-key cache of the decode path (``enabled=False``: re-rotate the whole cache every step like the reference).
rotated_cache_config = {"enabled": True}


def _abs_angles(inv_freq: torch.Tensor, row0: int, n: int) -> torch.Tensor:
    """(1, n, 2*len(inv_freq)) angles of absolute positions row0 .. row0+n-1: position * inv_freq with every frequency
    repeated twice — exactly FrequencyPositionEncoding.forward (reference position.py:69-71)."""
    pos = torch.arange(row0, row0 + n, device=inv_freq.device, dtype=inv_freq.dtype)
    return (pos[None, :, None] * inv_freq[None, None, :]).repeat_interleave(2, dim=-1).float()


def _rotary_fp8(x: torch.Tensor, num_heads: int, angles: torch.Tensor, y: torch.Tensor, y_inv_scale: torch.Tensor,
                x_descale: Optional[torch.Tensor] = None, right_align: bool = False) -> None:
    """y (B, n, H*d) e4m3 <- e4m3(rotate(x) * y_inv_scale[h]) (pcv_rotary_apply_fp8).  x is bf16 / fp16, or e4m3 codes
    standing for ``x * x_descale[h]``; ``angles`` (B or 1, n_angles, f) float32, rows as in :func:`rotary`."""
    p = _rotary_params(x, y, num_heads, angles, right_align, _lib.PCV_E4M3 if x.dtype == F8 else _pcv_dtype(x.dtype))
    f = _lib.RotaryFp8()
    f.x_descale = None if x_descale is None else x_descale.data_ptr()
    f.y_inv_scale = y_inv_scale.data_ptr()
    with torch.cuda.device(x.device):
        _launch_rotary(p, f)


def rotary_fp8(x8: torch.Tensor, num_heads: int, angles: torch.Tensor, right_align: bool,
               descale: torch.Tensor) -> torch.Tensor:
    """e4m3 codes x8 (B, n, H*d) standing for ``x8 * descale[h]`` (descale (H,)), rotated like :func:`rotary` (the
    reference's ``frq_pos_enc`` angles, (B or 1, [1,] n_angles, rotate_dim)) and requantised with the same descale, in
    one pass (pcv_rotary_apply_fp8): a new (B, n, H*d) e4m3 tensor.  The descale must bound the rotated rows too
    (:func:`fp8_pair_descale`).  Each code is rounded a second time."""
    _require_cuda(x8, angles, descale)
    if x8.dtype != F8:
        raise ValueError(f"rotary_fp8: x8 must be torch.float8_e4m3fn, got {x8.dtype}")
    angles = _rotary_angles(angles)
    B, n, _ = x8.shape
    if angles.shape[0] not in (1, B) or angles.shape[1] < n:
        raise ValueError(f"rotary_fp8: angles {tuple(angles.shape)} do not cover x8 {tuple(x8.shape)}")
    x8 = _rows_contiguous(x8)
    kd = descale.float().contiguous()
    y = torch.empty(x8.shape, dtype=F8, device=x8.device)
    if n:
        _rotary_fp8(x8, num_heads, angles, y, 1.0 / kd, kd, bool(right_align))
    return y


def rotated_cache_keys(k: torch.Tensor, q: torch.Tensor, num_heads: int, inv_freq: torch.Tensor,
                       k_new: Optional[torch.Tensor] = None, k_descale: Optional[torch.Tensor] = None):
    """Rotary embedding of a cached decode step WITHOUT re-rotating the cache: returns ``(q_rot, k_rot)`` or None.

    ``k`` (B, L, C) must be a row range of a KV arena (what :func:`kv_append` returns) and the rows of ``q`` (B, N, C)
    must be the LAST N tokens of ``k`` (true for the Perceiver-AR cross-attention and the causal latent self-attention).
    Rotary scores depend on position DIFFERENCES only, so instead of the reference's window-relative positions
    (``positions(b, n, shift)``, which change for every cached key whenever the window slides or the batch rows are
    padded differently) every key is rotated ONCE, when it is first seen, at the absolute position "its row index in
    the arena", into a shadow buffer kept beside the arena; q is rotated at the row index of its own token.  For every
    non-masked (query, key) pair the angle difference equals the reference's (pos_q - pos_k = row_q - row_k; padded
    rows are masked out), so the scores agree up to rounding, and a decode step rotates N new rows instead of L.
    Arena rows are write-once (an append that is not at the frontier gets a fresh arena), so shadow rows never go stale.

    An e4m3 arena (:func:`kv_append_fp8`) gets an e4m3 shadow with the per-head ``k_descale`` (H,) of its codes, which
    must bound the rotated rows too (:func:`fp8_pair_descale`).  ``k_new`` are the bf16 / fp16 rows this call appended
    (the last ``k_new.shape[1]`` rows of ``k``): their shadow rows are rotated from those values and rounded once.  Older
    rows the shadow lacks (a fresh or re-ordered arena) are rebuilt from the codes: dequantised, rotated, requantised."""
    if not rotated_cache_config["enabled"]:
        return None
    hit = _arena_of(k)
    fp8 = k.dtype == F8
    if hit is None or inv_freq is None or q.shape[1] > k.shape[1] or k.dtype not in (torch.bfloat16, torch.float16, F8):
        return None
    if fp8 and k_descale is None:
        raise ValueError("rotated_cache_keys: an e4m3 cache needs k_descale")
    arena, start = hit
    root = k._base if k._base is not None else k
    L, N = k.shape[1], q.shape[1]
    # identity of the frequency table as the caller holds it (a bf16 model's buffer is converted below: the converted
    # copy is kept with the shadow, otherwise every step would see a "new" table and re-rotate the whole cache)
    key = (inv_freq.data_ptr(), inv_freq.dtype, int(inv_freq.numel()), num_heads, inv_freq._version)
    rot = arena.rot
    if rot is None or rot["key"] != key:
        rot = {"buf": torch.empty_like(root), "lo": 0, "hi": 0, "key": key,
               "inv_freq": inv_freq.detach().to(device=k.device, dtype=torch.float32)}
        arena.rot = rot
    inv_freq = rot["inv_freq"]
    end = start + L
    if not (rot["lo"] <= start <= rot["hi"]):   # nothing reusable: rotate the whole range once
        rot["lo"], rot["hi"] = start, start
    if rot["hi"] < end and fp8:
        kd = k_descale.float().contiguous()
        inv = 1.0 / kd
        a, b = rot["hi"], end
        fresh = end - (0 if k_new is None else k_new.shape[1])   # first row this call appended
        if a < fresh:   # rebuilt from the codes: rounded twice
            _rotary_fp8(root[:, a:fresh], num_heads, _abs_angles(inv_freq, a, fresh - a), rot["buf"][:, a:fresh], inv, kd)
        a = max(a, fresh)
        if a < b:       # rotated from this call's bf16 / fp16 rows: rounded once
            _rotary_fp8(_rows_contiguous(k_new[:, a - fresh:]), num_heads, _abs_angles(inv_freq, a, b - a),
                        rot["buf"][:, a:b], inv)
        rot["hi"] = end
    elif rot["hi"] < end:
        a, b = rot["hi"], end
        _rotary_forward(root[:, a:b], num_heads, _abs_angles(inv_freq, a, b - a), False, out=rot["buf"][:, a:b])
        rot["hi"] = end
    q_rot = _rotary_forward(q, num_heads, _abs_angles(inv_freq, end - N, N), False)
    return q_rot, rot["buf"][:, start:end]


def rotary_at(x: torch.Tensor, num_heads: int, inv_freq: torch.Tensor, row0: int) -> torch.Tensor:
    """x (B, n, H*d) rotated at the absolute positions row0 .. row0 + n - 1 (fp32 angles from ``inv_freq``), as
    :func:`rotated_cache_keys` rotates q and the shadow rows."""
    return _rotary_forward(x, num_heads, _abs_angles(inv_freq.detach().float(), row0, x.shape[1]), False)


def rotated_cache_shadow(k: torch.Tensor):
    """``(rows, first_position)`` of the rotated-key shadow that :func:`rotated_cache_keys` keeps for the cache ``k``:
    ``rows`` (B, L, C) are k's rows rotated at the absolute positions ``first_position`` .. ``first_position + L - 1``
    (bf16 / fp16, or the e4m3 codes of an FP8 cache).  None when k has no complete shadow (yet)."""
    hit = _arena_of(k)
    if hit is None or hit[0].rot is None:
        return None
    rot, start = hit[0].rot, hit[1]
    if not (rot["lo"] <= start and start + k.shape[1] <= rot["hi"]):
        return None
    return rot["buf"][:, start:start + k.shape[1]], start


# --------------------------------------------------------------------------------------------------
# device-resident rows: decode, append and rotary whose rows are read from device int32s when the kernel runs, so a
# recorded CUDA graph replays every step of a decode loop (generation.GraphedDecoder).  They do no arena bookkeeping.
# The bounds are 1-D (one set shared by every batch row) or (B, >= width) (row b reads bounds[b], at any row stride).
# --------------------------------------------------------------------------------------------------
def _dev_rows(bounds: torch.Tensor, capacity: int, batch: int, width: int, what: str):
    if bounds.dtype != torch.int32 or not bounds.is_cuda or bounds.dim() not in (1, 2) or bounds.stride(-1) != 1:
        raise ValueError(f"{what}: bounds must be a 1-D or 2-D CUDA int32 tensor with unit stride in its last dim")
    if bounds.shape[-1] < width or (bounds.dim() == 2 and bounds.shape[0] != batch):
        raise ValueError(f"{what}: bounds must be ({width},) shared by every batch row or ({batch}, {width}) per row, "
                         f"got {tuple(bounds.shape)}")
    r = _lib.DevRows()
    r.bounds, r.capacity = bounds.data_ptr(), int(capacity)
    r.bounds_stride_b = bounds.stride(0) if bounds.dim() == 2 else 0
    return r


def rotary_angle_table(inv_freq: torch.Tensor, capacity: int) -> torch.Tensor:
    """(capacity, 2*len(inv_freq)) float32 angles of the absolute positions 0 .. capacity - 1, with exactly the arithmetic
    of the angles :func:`rotated_cache_keys` and :func:`rotary_at` build, so rotations from it are bit-equal to theirs."""
    return _abs_angles(inv_freq.detach().float(), 0, capacity)[0].contiguous()


def attention_decode_window(q, k, v, bounds: torch.Tensor, num_heads: int, scale: float, pad_mask=None,
                            causal: bool = False, k_descale=None, v_descale=None) -> torch.Tensor:
    """Attention of at most 4 query rows on the key window ``[bounds[0], bounds[1])`` of KV arenas, the window read from
    device memory when the kernel runs (pcv_attn_decode_window / _fp8): nothing is read back to the host, so the call
    can be recorded in a CUDA graph and replayed for every window.

    q: (B or 1, N <= 4, H*dqk) bf16 / fp16; k, v: (B, capacity, H*d) arenas, bf16 / fp16 like q or ``float8_e4m3fn``
    codes (then ``k_descale`` (H,) and ``v_descale`` (H, dv) as in :func:`attention_decode_fp8`); ``pad_mask`` (B,
    capacity), indexed by the absolute arena row; ``bounds`` a CUDA int32 tensor whose first two entries are the window,
    or a (B, >= 2) one whose row b holds batch row b's window (unit stride in its last dim, any row stride).  The causal
    mask is right-aligned to the window's end; a window of length <= 0 gives zeros.  Returns (B, N, H*dv)."""
    _require_cuda(q, k, v, bounds, pad_mask)
    with torch.cuda.device(k.device):
        p, f, keep = _fill_decode(q, k, v, num_heads, scale, pad_mask, causal, k_descale, v_descale)
        out = _new_output(p, _compute_dtype(q.dtype), k.device)
        _run_decode(p, f, _dev_rows(bounds, p.M, p.B, 2, "attention_decode_window"), k.device)
    del keep
    return out


#: Query rows of one :func:`attention_window` call (one m64 tensor-core tile).
WINDOW_MAX_ROWS = 64


def attention_window(q, k, v, bounds: torch.Tensor, num_heads: int, scale: float, band: int = 0, pad_mask=None,
                     causal: bool = False, k_descale=None, v_descale=None) -> torch.Tensor:
    """Attention of 1 to 64 query rows on the key window ``[bounds[0], bounds[1])`` of KV arenas on the tensor cores,
    the window read from device memory when the kernel runs (pcv_attn_cached_window / _fp8): nothing is read back to
    the host, so the call can be recorded in a CUDA graph and replayed for every window.

    q: (B or 1, N <= 64, H*dqk) bf16 / fp16; k, v: (B, capacity, H*d) arenas of q's dtype (head dims multiples of 8) or
    ``float8_e4m3fn`` codes (head dims multiples of 16, with ``k_descale`` (H,) and ``v_descale`` (H, dv) as in
    :func:`attention_decode_fp8`); ``pad_mask`` (B, capacity), indexed by the absolute arena row.  ``bounds`` 1-D is one
    window for every batch row; (B, >= 2) gives batch row b its own window ``bounds[b, 0:2]`` (unit stride in its last
    dim, any row stride; also with a batch-1 q).  Query i sits at row ``r_i = end - N + i`` of its batch row's window.  With ``band`` W > 0 (``causal`` only) query i sees exactly the keys ``[r_i + 1 - W, r_i]``:
    a key outside its band contributes nothing, a padded key inside it takes the finite fill — N rows of one call
    are then N one-token steps whose windows are ``[max(0, r_i + 1 - W), r_i + 1)``.  With W = 0 the causal mask is
    right-aligned to the window's end and masks as :func:`attention`.  A window of length <= 0 gives zeros.  P is
    rounded to q's dtype before P V, as :func:`attention` does.  Returns (B, N, H*dv) in q's dtype."""
    _require_cuda(q, k, v, bounds, pad_mask, k_descale, v_descale)
    if q.dtype not in (torch.bfloat16, torch.float16):
        raise ValueError(f"attention_window: q must be bf16 / fp16, got {q.dtype}")
    fp8 = k.dtype == F8
    if fp8 != (v.dtype == F8) or (not fp8 and (k.dtype != q.dtype or v.dtype != q.dtype)):
        raise ValueError(f"attention_window: the K / V arenas ({k.dtype} / {v.dtype}) must both be q's dtype "
                         f"({q.dtype}) or float8_e4m3fn")
    if fp8 != (k_descale is not None and v_descale is not None) or (not fp8 and (k_descale, v_descale) != (None, None)):
        raise ValueError("attention_window: k_descale and v_descale go with e4m3 arenas, and only with them")
    if band < 0 or (band > 0 and not causal):
        raise ValueError(f"attention_window: band must be >= 0 and needs causal=True, got band={band} causal={causal}")
    with torch.cuda.device(k.device):
        if fp8:
            p, f, keep = _fill_decode(q, k, v, num_heads, scale, pad_mask, causal, k_descale, v_descale)
        else:
            p, keep = _fill_attn_params(_rows_contiguous(q), _rows_contiguous(k), _rows_contiguous(v), num_heads, scale,
                                        pad_mask, causal, None, 0, "auto")
            f = None
        p.impl = _lib.PCV_IMPL_AUTO
        out = _new_output(p, q.dtype, k.device)
        rows = _dev_rows(bounds, p.M, p.B, 2, "attention_window")
        entry = "pcv_attn_cached_window" + ("_fp8" if fp8 else "")
        ws = _workspace(p, k.device, entry, C.byref(p))
        check(getattr(_lib.lib(), entry)(*(C.byref(s) for s in (p, f, rows) if s is not None), int(band), _stream()),
              entry)
    del ws, keep
    return out


def kv_append_at(k_arena: torch.Tensor, v_arena: torch.Tensor, k_new: torch.Tensor, v_new: torch.Tensor,
                 row: torch.Tensor, k_inv_scale=None, v_inv_scale=None) -> None:
    """Write the new rows k_new / v_new (B, n, C) to rows ``row[0] .. row[0] + n - 1`` of the arenas (B, capacity, C), the
    row read from device memory when the kernel runs (pcv_kv_append_at); rows that would land before row 0 or at or
    past capacity are skipped.  ``row`` (B, >= 1) gives batch row b its own first row ``row[b, 0]``.
    ``float8_e4m3fn`` arenas store ``clamp(x * inv_scale, +-448)`` rounded to e4m3 (pcv_kv_append_at_fp8, per-channel
    ``k_inv_scale`` / ``v_inv_scale`` as in :func:`kv_append_fp8`)."""
    _require_cuda(k_arena, v_arena, k_new, v_new, row)
    fp8 = k_arena.dtype == F8
    if v_arena.dtype != k_arena.dtype or k_arena.shape[:2] != v_arena.shape[:2]:
        raise ValueError("kv_append_at: the K and V arenas must agree in dtype, batch and capacity")
    if not fp8 and (k_new.dtype != k_arena.dtype or v_new.dtype != k_arena.dtype):
        raise ValueError(f"kv_append_at: new rows {k_new.dtype} / {v_new.dtype} into a {k_arena.dtype} arena")
    if k_arena.stride(-1) != 1 or v_arena.stride(-1) != 1:
        raise ValueError("kv_append_at: arenas need unit channel stride")
    _launch_kv_append(None, None, _rows_contiguous(k_new), _rows_contiguous(v_new), k_arena, v_arena, False, False,
                      (k_inv_scale, v_inv_scale) if fp8 else None,
                      _dev_rows(row, k_arena.shape[1], k_arena.shape[0], 1, "kv_append_at"))


def rotary_apply_at(x: torch.Tensor, num_heads: int, table: torch.Tensor, rows: torch.Tensor, out: torch.Tensor,
                    y_inv_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out`` <- x (B, n, H*d) bf16 / fp16 rotated at the angle rows ``rows[0] + i`` of ``table`` (capacity, rotate_dim)
    (:func:`rotary_angle_table`), the rows read from device memory when the kernel runs (pcv_rotary_apply_at / _fp8).
    Row i goes to ``out[:, rows[0] + i]`` when ``rows[1] != 0`` (a key into a rotated-key arena of at least capacity
    rows), else to ``out[:, i]``.  Rows whose table row ``rows[0] + i`` is negative or at or past ``table.shape[0]``
    are skipped: their output row is not written.  ``rows`` (B, >= 2) gives batch row b its own ``rows[b, 0:2]``.  An
    e4m3 ``out`` stores the codes of the rotated rows times ``y_inv_scale[h]`` (H,).
    Bit-equal to :func:`rotary_at` / the rotated-key shadow of :func:`rotated_cache_keys` at the same positions."""
    _require_cuda(x, table, rows, out)
    x = _rows_contiguous(x)
    if out.stride(-1) != 1 or out.shape[0] != x.shape[0] or out.shape[2] != x.shape[2]:
        raise ValueError("rotary_apply_at: `out` must be (B, rows, H*d) like x with unit channel stride")
    if table.dim() != 2 or table.dtype != torch.float32 or table.stride(-1) != 1:
        raise ValueError("rotary_apply_at: the angle table must be a (capacity, rotate_dim) float32 tensor")
    fp8 = out.dtype == F8
    if not fp8 and out.dtype != x.dtype:
        raise ValueError(f"rotary_apply_at: `out` {out.dtype} must be x's dtype {x.dtype} or float8_e4m3fn")
    p = _rotary_params(x, out, num_heads, table[None], False, _pcv_dtype(x.dtype))
    f = _lib.RotaryFp8(x_descale=None, y_inv_scale=y_inv_scale.data_ptr()) if fp8 else None
    with torch.cuda.device(x.device):
        _launch_rotary(p, f, _dev_rows(rows, table.shape[0], x.shape[0], 2, "rotary_apply_at"))
    return out


# --------------------------------------------------------------------------------------------------
# token sampling (pcv_sample): temperature, top-k and top-p with the 🤗 warpers' semantics, drawn on the device from a
# counter-based stream keyed by (seed of the batch row, batch row, position), so it can be recorded in a CUDA graph.
# --------------------------------------------------------------------------------------------------
#: The largest vocabulary :func:`sample_tokens` takes.
SAMPLE_MAX_VOCAB = _lib.SAMPLE_MAX_VOCAB


def _sample_counters(seeds: torch.Tensor, positions: torch.Tensor, lead: tuple, what: str):
    _require_cuda(seeds, positions)
    if seeds.dtype != torch.int64 or tuple(seeds.shape) != lead[:1]:
        raise ValueError(f"{what}: seeds must be a ({lead[0]},) int64 CUDA tensor (one per batch row), got "
                         f"{tuple(seeds.shape)} {seeds.dtype}")
    if positions.dtype != torch.int32 or tuple(positions.shape) != lead:
        raise ValueError(f"{what}: positions must be a {lead} int32 CUDA tensor (one per logits row), got "
                         f"{tuple(positions.shape)} {positions.dtype}")
    return seeds.contiguous(), positions.contiguous()


def sample_tokens(logits: torch.Tensor, seeds: torch.Tensor, positions: torch.Tensor, temperature: float = 1.0,
                  top_k: int = 0, top_p: float = 1.0, logprobs: bool = False):
    """One token per logits row, drawn on the device (pcv_sample): ``logits / temperature``, then top-k, then top-p, then
    softmax + multinomial — the semantics of 🤗's ``TemperatureLogitsWarper`` -> ``TopKLogitsWarper`` ->
    ``TopPLogitsWarper``, except that a tie group straddling the top-p cut is kept whole.  ``temperature=0`` is greedy
    (the first maximal index); ``top_k=0`` and ``top_p=1`` turn those filters off.  The three values are taken in fp32.

    logits: (B, V) or (B, k, V) bf16 / fp16 / fp32, V <= :data:`SAMPLE_MAX_VOCAB`; seeds: (B,) int64 CUDA, one per batch
    row; positions: (B,) or (B, k) int32 CUDA, the counter of every row's draw.  A row's token is a pure function of
    its logits, the three values, its seed, its batch row and its position (nothing is read back to the host, so the
    call can be recorded in a CUDA graph).  Returns int64 tokens of the logits' leading shape and, with ``logprobs``,
    their fp32 log-probabilities under the filtered distribution (0 when greedy).  Arguments the kernel does not take
    raise ``ValueError`` with its reason before any launch."""
    _require_cuda(logits)
    if logits.dim() not in (2, 3) or logits.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError(f"sample_tokens: logits must be (B, V) or (B, k, V) bf16 / fp16 / fp32, got "
                         f"{tuple(logits.shape)} {logits.dtype}")
    lead = tuple(logits.shape[:-1])
    seeds, positions = _sample_counters(seeds, positions, lead, "sample_tokens")
    V = logits.shape[-1]
    rows = (logits if logits.stride(-1) == 1 else logits.contiguous()).reshape(-1, V)
    tokens = torch.empty(lead, dtype=torch.int64, device=logits.device)
    lp = torch.empty(lead, dtype=torch.float32, device=logits.device) if logprobs else None
    p = _lib.SampleParams()
    p.logits, p.stride_row, p.R, p.V = rows.data_ptr(), rows.stride(0), rows.shape[0], V
    p.dtype = _lib.PCV_F32 if logits.dtype == torch.float32 else _pcv_dtype(logits.dtype)
    p.rows_per_batch = 1 if logits.dim() == 2 else logits.shape[1]
    p.seeds, p.positions = seeds.data_ptr(), positions.data_ptr()
    p.temperature, p.top_p = float(temperature), float(top_p)
    p.top_k = min(int(top_k), 2 ** 31 - 1)
    p.tokens, p.logprobs = tokens.data_ptr(), (lp.data_ptr() if lp is not None else None)
    lib = _lib.lib()
    if not lib.pcv_sample_supported(C.byref(p)):
        raise ValueError(f"sample_tokens: {lib.pcv_last_error().decode()}")
    with torch.cuda.device(logits.device):
        check(lib.pcv_sample(C.byref(p), _stream()), "pcv_sample")
    return (tokens, lp) if logprobs else tokens


def sample_uniforms(seeds: torch.Tensor, positions: torch.Tensor) -> torch.Tensor:
    """The 64 random bits (as int64) of the draw of every row of :func:`sample_tokens` with these seeds (B,) and
    positions (B,) or (B, k) — pcv_sample_uniforms."""
    lead = tuple(positions.shape)
    if len(lead) not in (1, 2):
        raise ValueError(f"sample_uniforms: positions must be (B,) or (B, k), got {lead}")
    seeds, positions = _sample_counters(seeds, positions, lead, "sample_uniforms")
    out = torch.empty(lead, dtype=torch.int64, device=positions.device)
    with torch.cuda.device(positions.device):
        check(_lib.lib().pcv_sample_uniforms(out.data_ptr(), seeds.data_ptr(), positions.data_ptr(), positions.numel(),
                                             1 if len(lead) == 1 else lead[1], _stream()), "pcv_sample_uniforms")
    return out


# --------------------------------------------------------------------------------------------------
# speculative sampling (pcv_spec_verify): the rejection rule with a draft model's probabilities, on the sampler's integer
# masses, with accept and residual bits from two counter-based streams of their own.
# --------------------------------------------------------------------------------------------------
#: The most drafts :func:`spec_verify` decides per batch row in one call.
SPEC_MAX_DRAFTS = _lib.SPEC_MAX_DRAFTS
_SPEC_STREAMS = {"accept": 0, "residual": 1}


def _sampling_values(vals, what: str):
    if not isinstance(vals, (tuple, list)) or len(vals) != 3:
        raise ValueError(f"spec_verify: {what} must be a (temperature, top_k, top_p) triple, got {vals!r}")
    t, k, p = vals
    return float(t), min(int(k), 2 ** 31 - 1), float(p)


def spec_verify(target_logits: torch.Tensor, draft_logits: torch.Tensor, tokens: torch.Tensor, seeds: torch.Tensor,
                positions: torch.Tensor, sampling=(1.0, 0, 1.0), draft_sampling=(1.0, 0, 1.0)):
    """One round of speculative sampling for every batch row, on the device (pcv_spec_verify).

    Row b fed ``tokens[b]`` = t_0 .. t_G (B, G+1) int64 to both models, t_1 .. t_G drawn by the draft.
    ``target_logits`` (B, G+1, V): the target's logits after each t_i; ``draft_logits`` (B, G, V), of the same dtype
    (bf16 / fp16 / fp32): the logits the draft drew t_{i+1} from.  ``sampling`` and ``draft_sampling`` are the
    (temperature, top_k, top_p) triples of the two models, as :func:`sample_tokens` takes them; p and q are the two
    filtered distributions.  Draft t_{i+1} is accepted with probability min(1, p/q) (to 2^-64, in exact integer
    arithmetic on the sampler's masses); the first rejected one is replaced by a draw from max(0, p - q), and when every
    draft is accepted a bonus token is drawn from the last target row.  ``seeds`` (B,) int64 and ``positions`` (B, G+1)
    int32 are the counters: the accept and residual bits of target row i use (seeds[b], b, positions[b, i]) on two
    streams independent of :func:`sample_tokens`' own, so the draft may share the target's seeds.

    Returns ``(tokens, accepted)``: (B, G+1) int64 with the n_b accepted drafts, then the correction or bonus token, then
    -1; and (B,) int32 n_b.  Nothing is read back to the host, so the call can be recorded in a CUDA graph.  Arguments
    the kernel does not take raise ``ValueError`` with its reason before any launch."""
    _require_cuda(target_logits, draft_logits, tokens)
    if target_logits.dim() != 3 or target_logits.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError(f"spec_verify: target_logits must be (B, G+1, V) bf16 / fp16 / fp32, got "
                         f"{tuple(target_logits.shape)} {target_logits.dtype}")
    B, G1, V = target_logits.shape
    if tuple(draft_logits.shape) != (B, G1 - 1, V) or draft_logits.dtype != target_logits.dtype:
        raise ValueError(f"spec_verify: draft_logits must be ({B}, {G1 - 1}, {V}) {target_logits.dtype} like the target "
                         f"rows, got {tuple(draft_logits.shape)} {draft_logits.dtype}")
    if tuple(tokens.shape) != (B, G1) or tokens.dtype != torch.int64:
        raise ValueError(f"spec_verify: tokens must be ({B}, {G1}) int64 (t_0 .. t_G), got {tuple(tokens.shape)} "
                         f"{tokens.dtype}")
    seeds, positions = _sample_counters(seeds, positions, (B, G1), "spec_verify")
    t, k, p_ = _sampling_values(sampling, "sampling")
    dt, dk, dp = _sampling_values(draft_sampling, "draft_sampling")
    target = target_logits if target_logits.stride(-1) == 1 else target_logits.contiguous()
    draft = draft_logits if draft_logits.stride(-1) == 1 else draft_logits.contiguous()
    tokens = tokens.contiguous()
    out = torch.empty(B, G1, dtype=torch.int64, device=target.device)
    accepted = torch.empty(B, dtype=torch.int32, device=target.device)
    p = _lib.SpecVerifyParams()
    p.target, p.t_stride_b, p.t_stride_row = target.data_ptr(), target.stride(0), target.stride(1)
    p.draft, p.d_stride_b, p.d_stride_row = draft.data_ptr(), draft.stride(0), draft.stride(1)
    if G1 == 2:   # a dimension of size 1 may carry any stride: the kernel never steps along it
        p.d_stride_row = max(p.d_stride_row, V)
    if B == 1:
        p.t_stride_b, p.d_stride_b = max(p.t_stride_b, V), max(p.d_stride_b, V)
    p.tokens, p.seeds, p.positions = tokens.data_ptr(), seeds.data_ptr(), positions.data_ptr()
    p.B, p.G, p.V = B, G1 - 1, V
    p.dtype = _lib.PCV_F32 if target.dtype == torch.float32 else _pcv_dtype(target.dtype)
    p.draft_dtype = p.dtype
    p.temperature, p.top_k, p.top_p = t, k, p_
    p.draft_temperature, p.draft_top_k, p.draft_top_p = dt, dk, dp
    p.out_tokens, p.accepted = out.data_ptr(), accepted.data_ptr()
    lib = _lib.lib()
    if not lib.pcv_spec_verify_supported(C.byref(p)):
        raise ValueError(f"spec_verify: {lib.pcv_last_error().decode()}")
    with torch.cuda.device(target.device):
        check(lib.pcv_spec_verify(C.byref(p), _stream()), "pcv_spec_verify")
    return out, accepted


def spec_uniforms(seeds: torch.Tensor, positions: torch.Tensor, stream: str = "accept") -> torch.Tensor:
    """The 64 bits (as int64) of :func:`spec_verify`'s ``stream`` ("accept" or "residual") at these seeds (B,) and
    positions (B,) or (B, k) — pcv_spec_uniforms."""
    if stream not in _SPEC_STREAMS:
        raise ValueError(f"spec_uniforms: stream must be 'accept' or 'residual', got {stream!r}")
    lead = tuple(positions.shape)
    if len(lead) not in (1, 2):
        raise ValueError(f"spec_uniforms: positions must be (B,) or (B, k), got {lead}")
    seeds, positions = _sample_counters(seeds, positions, lead, "spec_uniforms")
    out = torch.empty(lead, dtype=torch.int64, device=positions.device)
    with torch.cuda.device(positions.device):
        check(_lib.lib().pcv_spec_uniforms(out.data_ptr(), seeds.data_ptr(), positions.data_ptr(), positions.numel(),
                                           1 if len(lead) == 1 else lead[1], _SPEC_STREAMS[stream], _stream()),
              "pcv_spec_uniforms")
    return out


# --------------------------------------------------------------------------------------------------
# beam search (pcv_beam_step, pcv_kv_gather_rows): 🤗's beam step on device-resident state, and the KV gather of the
# generated rows by parent, both recordable in a CUDA graph.
# --------------------------------------------------------------------------------------------------
#: The most beams and EOS ids :func:`beam_step` takes.
BEAM_MAX_BEAMS = _lib.BEAM_MAX_BEAMS
BEAM_MAX_EOS = _lib.BEAM_MAX_EOS


def early_stopping_code(early_stopping) -> int:
    """pcv_early_stopping of 🤗's ``early_stopping``: the bools False / True or the string "never", nothing else (🤗
    tests ``early_stopping is True`` and ``== "never"``, so a string "True" would not mean True there)."""
    if early_stopping is False or early_stopping is True:
        return int(early_stopping)
    if isinstance(early_stopping, str) and early_stopping == "never":
        return 2
    raise ValueError(f"early_stopping must be False, True or 'never', got {early_stopping!r}")


def beams_to_keep(num_beams: int, n_eos: int) -> int:
    return max(2, n_eos + 1) * num_beams


class BeamState:
    """The device state of :func:`beam_step` for B items of K beams and ``n_eos`` EOS ids: running and finished scores,
    finished flags, token histories (B, K, hist_len) filled with ``fill``, the per-item heuristic and done flags, the
    counters [generated count, max_length, every item done, 0], and the step's scratch and outputs (``tokens`` (B*K, 1)
    int64, ``parents`` (B*K,) int32).  ``reset(max_length)`` re-initialises every buffer in place."""

    def __init__(self, B: int, K: int, n_eos: int, hist_len: int, fill: int, device):
        keep = beams_to_keep(K, n_eos)
        self.B, self.K, self.n_eos, self.hist_len, self.fill = B, K, n_eos, hist_len, int(fill)
        f32, i32, i64 = torch.float32, torch.int32, torch.int64
        self.running = torch.empty(B, K, dtype=f32, device=device)
        self.finished = torch.empty(B, K, dtype=f32, device=device)
        self.finished_flags = torch.empty(B, K, dtype=i32, device=device)
        self.running_hist = torch.empty(B, K, hist_len, dtype=i64, device=device)
        self.finished_hist = torch.empty(B, K, hist_len, dtype=i64, device=device)
        self.hist_scratch = torch.empty(B, 2 * K, hist_len, dtype=i64, device=device)
        self.item_flags = torch.empty(B, 2, dtype=i32, device=device)
        self.counters = torch.empty(4, dtype=i32, device=device)
        self.cand_scores = torch.empty(B * K, keep, dtype=f32, device=device)
        self.cand_index = torch.empty(B * K, keep, dtype=i32, device=device)
        self.tokens = torch.zeros(B * K, 1, dtype=i64, device=device)
        self.parents = torch.zeros(B * K, dtype=i32, device=device)

    def reset(self, max_length: int) -> None:
        """Start a search of ``max_length`` generated tokens: eager in-place fills, no synchronisation."""
        self.running.fill_(-1e9)
        self.running[:, 0].fill_(0.0)
        self.finished.fill_(-1e9)
        self.finished_flags.zero_()
        self.running_hist.fill_(self.fill)
        self.finished_hist.fill_(self.fill)
        self.item_flags[:, 0].fill_(1)
        self.item_flags[:, 1].fill_(0)
        self.counters.zero_()
        self.counters[1:2].fill_(int(max_length))   # fill_ with a host scalar: a kernel argument, no copy or sync


def beam_step(logits: torch.Tensor, state: BeamState, eos=(), length_penalty: float = 1.0, early_stopping=False,
              logprobs: bool = False):
    """One step of 🤗's beam search (``do_sample=False``) on the device (pcv_beam_step), in place
    on ``state``: logits (B*K, V) bf16 / fp16 / fp32, V <= :data:`SAMPLE_MAX_VOCAB`, beam k of item b in row b*K + k.
    Returns ``(state.tokens, state.parents)``: the (B*K, 1) int64 next tokens and the (B*K,) int32 global beam row each
    beam continues.  Nothing is read back to the host, so the call can be recorded in a CUDA graph: the generated count
    and max_length live in ``state.counters``.  With ``logprobs=True`` the rows are fp32 log-probabilities already
    (:func:`process_logits` with ``log_softmax=True``: 🤗's processors run on the log-softmax) and the step starts from
    them (pcv_beam_step_logprobs).  Arguments the kernel does not take raise ``ValueError`` with its reason before any
    launch."""
    _require_cuda(logits)
    if logits.dim() != 2 or logits.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError(f"beam_step: logits must be (B*K, V) bf16 / fp16 / fp32, got {tuple(logits.shape)} "
                         f"{logits.dtype}")
    eos = list(eos)
    if logits.shape[0] != state.B * state.K or len(eos) != state.n_eos:
        raise ValueError(f"beam_step: the state is for {state.B}x{state.K} beams and {state.n_eos} EOS ids, got "
                         f"{logits.shape[0]} logits rows and {len(eos)} EOS ids")
    rows = logits if logits.stride(-1) == 1 else logits.contiguous()
    p = _lib.BeamStepParams()
    p.logits, p.stride_row = rows.data_ptr(), rows.stride(0) if rows.shape[0] > 1 else rows.shape[1]
    p.B, p.K, p.V = state.B, state.K, rows.shape[1]
    p.dtype = _lib.PCV_F32 if rows.dtype == torch.float32 else _pcv_dtype(rows.dtype)
    if len(eos) > BEAM_MAX_EOS:
        raise ValueError(f"beam_step: at most {BEAM_MAX_EOS} EOS ids, got {len(eos)}")
    p.n_eos = len(eos)
    for i, e in enumerate(eos):
        p.eos[i] = max(-2 ** 31, min(int(e), 2 ** 31 - 1))
    p.length_penalty = float(length_penalty)
    p.early_stopping = early_stopping_code(early_stopping)
    p.hist_len = state.hist_len
    for f in ("running", "finished", "finished_flags", "running_hist", "finished_hist", "hist_scratch", "item_flags",
              "counters", "cand_scores", "cand_index"):
        setattr(p, {"running": "running_scores", "finished": "finished_scores"}.get(f, f), getattr(state, f).data_ptr())
    p.next_tokens, p.parents = state.tokens.data_ptr(), state.parents.data_ptr()
    lib = _lib.lib()
    entry = "pcv_beam_step_logprobs" if logprobs else "pcv_beam_step"
    if not getattr(lib, entry + "_supported")(C.byref(p)):
        raise ValueError(f"beam_step: {lib.pcv_last_error().decode()}")
    with torch.cuda.device(logits.device):
        check(getattr(lib, entry)(C.byref(p), _stream()), entry)
    return state.tokens, state.parents


class KvGatherTable:
    """The device table of :func:`kv_gather_rows`: ``entries`` is a list of ``(arena, first_row, bounds_col)`` with arena
    a (R, capacity, C) tensor (any dtype, 16-byte rows) whose generated rows start at ``first_row``, and ``bounds_col``
    the int32 of a beam row's bounds that holds its current row.  Each arena needs a scratch of (R, capacity -
    first_row, C): taken from ``reuse`` (an earlier table, e.g. of the previous prefill's arenas) where one of that
    shape, dtype and device is at the same position, else allocated.  The scratch only carries rows within one
    :func:`kv_gather_rows` call, so tables on one stream may share it; the device table is uploaded again only when
    its bytes differ from ``reuse``'s."""

    def __init__(self, entries, reuse: Optional["KvGatherTable"] = None):
        if not entries:
            raise ValueError("KvGatherTable: no arenas")
        self.scratch, self.arenas = [], []
        table = (_lib.KvGatherEntry * len(entries))()
        R = entries[0][0].shape[0]
        for e, (arena, first, col) in zip(table, entries):
            _require_cuda(arena)
            row_bytes = arena.shape[2] * arena.element_size()
            if (arena.dim() != 3 or arena.shape[0] != R or not arena.is_contiguous() or row_bytes % 16
                    or arena.data_ptr() % 16):
                raise ValueError(f"KvGatherTable: arenas must be contiguous (R={R}, capacity, C) tensors with 16-byte "
                                 f"aligned rows, got {tuple(arena.shape)} {arena.dtype}")
            if not 0 <= first < arena.shape[1] or col < 0:
                raise ValueError(f"KvGatherTable: first_row={first} must be in [0, {arena.shape[1]}) and bounds_col "
                                 f"={col} >= 0")
            rows = arena.shape[1] - first
            i = len(self.scratch)
            old = reuse.scratch[i] if reuse is not None and i < len(reuse.scratch) else None
            shape = (R, rows, arena.shape[2])
            if old is not None and tuple(old.shape) == shape and old.dtype == arena.dtype and old.device == arena.device:
                s = old
            else:
                s = torch.empty(shape, dtype=arena.dtype, device=arena.device)
            e.arena, e.scratch = arena.data_ptr(), s.data_ptr()
            e.arena_stride_b, e.scratch_stride_b = arena.stride(0) * arena.element_size(), rows * row_bytes
            e.row_bytes, e.first_row, e.bounds_col, e.max_rows = row_bytes, int(first), int(col), rows
            self.scratch.append(s)
            self.arenas.append(arena)
        self.R = R
        self.n = len(entries)
        self.packed = bytes(table)
        dev = entries[0][0].device
        if reuse is not None and reuse.packed == self.packed and reuse.table.device == dev:
            self.table, self._host = reuse.table, reuse._host
            return
        raw = torch.frombuffer(bytearray(self.packed), dtype=torch.uint8).pin_memory()   # asynchronous: no sync
        self.table = raw.to(dev, non_blocking=True)
        self._host = raw   # alive until the copy has run


def kv_gather_rows(table: KvGatherTable, parents: torch.Tensor, bounds: torch.Tensor, last_rows: int = 0) -> None:
    """Every beam row i with ``parents[i] != i`` takes its parent's rows [first_row, cur) of every arena of ``table``,
    cur = ``bounds[i, bounds_col]`` read on the device when the kernel runs (pcv_kv_gather_rows).  Cycles and
    many-to-one moves read the rows as they were before the call; every other byte is untouched.  ``parents`` (R,) int32
    CUDA; ``bounds`` (R, >= 1) int32 CUDA with unit stride in its last dim.  ``last_rows`` > 0 moves only the newest
    ``last_rows`` of those rows (contrastive search: 1, the row the step just appended).  Recordable in a CUDA graph."""
    n = _as_int(last_rows)
    if n is None or n < 0 or n > 2 ** 31 - 1:
        raise ValueError(f"kv_gather_rows: last_rows must be an integer >= 0 (0: every generated row), got {last_rows!r}")
    _require_cuda(parents, bounds)
    if parents.dtype != torch.int32 or tuple(parents.shape) != (table.R,) or not parents.is_contiguous():
        raise ValueError(f"kv_gather_rows: parents must be a contiguous ({table.R},) int32 tensor, got "
                         f"{tuple(parents.shape)} {parents.dtype}")
    if bounds.dtype != torch.int32 or bounds.dim() != 2 or bounds.shape[0] != table.R or bounds.stride(-1) != 1:
        raise ValueError(f"kv_gather_rows: bounds must be a ({table.R}, cols) int32 tensor with unit column stride")
    p = _lib.KvGatherParams()
    p.table, p.n_entries, p.R, p.parents = table.table.data_ptr(), table.n, table.R, parents.data_ptr()
    p.last_rows = n
    r = _lib.DevRows()
    r.bounds, r.capacity, r.bounds_stride_b = bounds.data_ptr(), bounds.shape[1], bounds.stride(0)
    lib = _lib.lib()
    if not lib.pcv_kv_gather_rows_supported(C.byref(p), C.byref(r)):
        raise ValueError(f"kv_gather_rows: {lib.pcv_last_error().decode()}")
    with torch.cuda.device(parents.device):
        check(lib.pcv_kv_gather_rows(C.byref(p), C.byref(r), _stream()), "pcv_kv_gather_rows")


def _as_int(x):
    """x as an int when it is integer-like and not a bool, else None."""
    if isinstance(x, bool):
        return None
    try:
        return operator.index(x)
    except TypeError:
        return None


# --------------------------------------------------------------------------------------------------
# contrastive search (pcv_contrastive_candidates, pcv_contrastive_rank): the candidates, the degeneration-penalty ranking
# and the context of hidden rows on the device, recordable in a CUDA graph; the KV select is kv_gather_rows(last_rows=1).
# --------------------------------------------------------------------------------------------------
#: The largest top_k, hidden width and EOS count :func:`contrastive_step` takes.
CONTRASTIVE_MAX_K = _lib.CONTRASTIVE_MAX_K
CONTRASTIVE_MAX_HIDDEN = _lib.CONTRASTIVE_MAX_HIDDEN
CONTRASTIVE_MAX_EOS = _lib.CONTRASTIVE_MAX_EOS


class ContrastiveState:
    """The device state of contrastive search for B items of K candidates with hidden width D: the context of hidden
    rows (B, cap, D) in ``dtype`` and their fp64 squared norms (negative: a padding row), the candidates of the last
    :func:`contrastive_candidates` (``probs`` (B, K) fp64, ``cand`` (B, K) int32), ``sel`` (B,) int32, ``unfinished``
    (B,) int32, the emitted tokens ``history`` (B, hist_len) int64 filled with ``fill``, the counters [context length,
    generated count, every item finished, 0], the next inputs ``tokens`` (B*K, 1) int64 and ``parents`` (B*K,) int32.
    ``reset(hidden, pad)`` loads the prompt's context and re-initialises every buffer in place."""

    def __init__(self, B: int, K: int, D: int, cap: int, hist_len: int, fill: int, dtype: torch.dtype, device):
        self.B, self.K, self.D, self.cap, self.hist_len, self.fill, self.dtype = B, K, D, cap, hist_len, int(fill), dtype
        f64, i32, i64 = torch.float64, torch.int32, torch.int64
        splits = -(-cap // _lib.CONTRASTIVE_ROWS_PER_CTA)
        self.context = torch.zeros(B, cap, D, dtype=dtype, device=device)
        self.norm2 = torch.zeros(B, cap, dtype=f64, device=device)
        self.partial = torch.empty(B, splits, K, dtype=f64, device=device)
        self.probs = torch.zeros(B, K, dtype=f64, device=device)
        self.cand = torch.zeros(B, K, dtype=i32, device=device)
        self.sel = torch.zeros(B, dtype=i32, device=device)
        self.unfinished = torch.ones(B, dtype=i32, device=device)
        self.history = torch.empty(B, hist_len, dtype=i64, device=device)
        self.counters = torch.zeros(4, dtype=i32, device=device)
        self.tokens = torch.zeros(B * K, 1, dtype=i64, device=device)
        self.parents = torch.zeros(B * K, dtype=i32, device=device)

    def reset(self, hidden: torch.Tensor, pad: Optional[torch.Tensor] = None) -> None:
        """Start a search whose context is the prompt's hidden rows ``hidden`` (B, L, D), L <= cap, with ``pad`` (B, L)
        (non-zero: a padding position, which the penalty skips).  Eager in-place ops, no synchronisation."""
        B, L = hidden.shape[0], hidden.shape[1] if hidden.dim() == 3 else -1
        if hidden.dim() != 3 or B != self.B or hidden.shape[2] != self.D or not 1 <= L <= self.cap:
            raise ValueError(f"ContrastiveState.reset: hidden must be ({self.B}, 1 .. {self.cap}, {self.D}), got "
                             f"{tuple(hidden.shape)}")
        if pad is not None and tuple(pad.shape) != (B, L):
            raise ValueError(f"ContrastiveState.reset: pad must be ({B}, {L}), got {tuple(pad.shape)}")
        self.context[:, :L].copy_(hidden)
        n2 = self.context[:, :L].double().square().sum(-1)
        self.norm2[:, :L].copy_(n2 if pad is None else torch.where(pad != 0, -1.0, n2))
        self.sel.zero_()
        self.unfinished.fill_(1)
        self.history.fill_(self.fill)
        self.counters.zero_()
        self.counters[0:1].fill_(int(L))   # fill_ with a host scalar: a kernel argument, no copy or sync


def _logits_rows(logits: torch.Tensor, state: ContrastiveState, what: str) -> torch.Tensor:
    _require_cuda(logits)
    if (logits.dim() != 2 or logits.shape[0] != state.B * state.K
            or logits.dtype not in (torch.bfloat16, torch.float16, torch.float32)):
        raise ValueError(f"{what}: logits must be ({state.B * state.K}, V) bf16 / fp16 / fp32 (B*K rows), got "
                         f"{tuple(logits.shape)} {logits.dtype}")
    return logits if logits.stride(-1) == 1 else logits.contiguous()


def _candidates_params(rows: torch.Tensor, state: ContrastiveState) -> "_lib.ContrastiveCandidatesParams":
    p = _lib.ContrastiveCandidatesParams()
    p.logits, p.stride_row = rows.data_ptr(), rows.stride(0) if rows.shape[0] > 1 else rows.shape[1]
    p.B, p.K, p.V = state.B, state.K, rows.shape[1]
    p.dtype = _lib.PCV_F32 if rows.dtype == torch.float32 else _pcv_dtype(rows.dtype)
    p.sel, p.probs, p.cand, p.next_tokens = (state.sel.data_ptr(), state.probs.data_ptr(), state.cand.data_ptr(),
                                             state.tokens.data_ptr())
    lib = _lib.lib()
    if not lib.pcv_contrastive_candidates_supported(C.byref(p)):
        raise ValueError(f"contrastive_candidates: {lib.pcv_last_error().decode()}")
    return p


def contrastive_candidates(logits: torch.Tensor, state: ContrastiveState) -> torch.Tensor:
    """The K candidates of every item from logits row b*K + ``state.sel[b]`` (pcv_contrastive_candidates): the K largest
    values, value descending then index ascending on ties, with their fp64 softmax probabilities in ``state.probs``.
    ``logits`` (B*K, V) bf16 / fp16 / fp32, V <= :data:`SAMPLE_MAX_VOCAB`.  Returns ``state.tokens`` (B*K, 1) int64,
    candidate j of item b at row b*K + j.  Recordable in a CUDA graph; arguments the kernel does not take raise
    ``ValueError`` before any launch."""
    p = _candidates_params(_logits_rows(logits, state, "contrastive_candidates"), state)
    with torch.cuda.device(logits.device):
        check(_lib.lib().pcv_contrastive_candidates(C.byref(p), _stream()), "pcv_contrastive_candidates")
    return state.tokens


def contrastive_step(logits: torch.Tensor, hidden: torch.Tensor, state: ContrastiveState, alpha: float, eos=(),
                     process: Optional[dict] = None):
    """One step of contrastive search after the model ran candidate j of item b at row b*K + j: ranks the candidates of
    the last :func:`contrastive_candidates` by ``(1 - alpha) p_j - alpha * max cos(context, h_j)`` in fp64, emits the
    best one (``state.fill`` once the item has emitted an EOS id) into ``state.history``, appends its hidden row to the
    context (pcv_contrastive_rank), then takes the next candidates from its logits row.  ``logits`` (B*K, V) and
    ``hidden`` (B*K, D) or (B*K, 1, D) of ``state.dtype``: the candidate pass's outputs.  Returns ``(state.tokens,
    state.parents)``: the next inputs and the batch row each row continues (for ``kv_gather_rows(..., last_rows=1)``).
    ``process``, if given, holds the keyword arguments of :func:`process_logits` (``row_map`` excepted: it is
    ``state.sel``): 🤗's logits processors run on the selected rows between the ranking and the candidates, when
    ``state.sel`` and ``state.history`` hold this step's selection, and the candidates are taken from the fp32 rows
    they write (``process["out"]``, (B*K, V) fp32, allocated when absent).  Nothing is read back to the host, so the
    call can be recorded in a CUDA graph; arguments the kernels do not take raise ``ValueError`` before any launch."""
    rows = _logits_rows(logits, state, "contrastive_step")
    _require_cuda(hidden)
    BK, D = state.B * state.K, state.D
    h = hidden.reshape(BK, D) if hidden.dim() == 3 and hidden.shape[1] == 1 else hidden
    if h.dim() != 2 or tuple(h.shape) != (BK, D) or h.dtype != state.dtype or h.stride(-1) != 1:
        raise ValueError(f"contrastive_step: hidden must be ({BK}, {D}) or ({BK}, 1, {D}) {state.dtype} with unit "
                         f"stride in its last dim, got {tuple(hidden.shape)} {hidden.dtype}")
    eos = list(eos)
    if len(eos) > CONTRASTIVE_MAX_EOS:
        raise ValueError(f"contrastive_step: at most {CONTRASTIVE_MAX_EOS} EOS ids, got {len(eos)}")
    a = float(alpha)
    p = _lib.ContrastiveRankParams()
    p.hidden, p.hidden_stride_row = h.data_ptr(), h.stride(0) if BK > 1 else D
    p.context, p.context_norm2 = state.context.data_ptr(), state.norm2.data_ptr()
    p.probs, p.cand = state.probs.data_ptr(), state.cand.data_ptr()
    p.alpha, p.pad_token = a, state.fill
    p.B, p.K, p.D = state.B, state.K, D
    p.hidden_dtype = {torch.bfloat16: _lib.PCV_BF16, torch.float16: _lib.PCV_F16}.get(state.dtype, -1)
    p.cap, p.hist_len, p.n_eos = state.cap, state.hist_len, len(eos)
    for i, e in enumerate(eos):
        p.eos[i] = max(-2 ** 31, min(int(e), 2 ** 31 - 1))
    p.partial, p.sel, p.unfinished = state.partial.data_ptr(), state.sel.data_ptr(), state.unfinished.data_ptr()
    p.history, p.counters, p.parents = state.history.data_ptr(), state.counters.data_ptr(), state.parents.data_ptr()
    lib = _lib.lib()
    if not lib.pcv_contrastive_rank_supported(C.byref(p)):
        raise ValueError(f"contrastive_step: {lib.pcv_last_error().decode()}")
    pp = None
    if process is not None:
        pp, rows = _process_params(rows, row_map=state.sel, **process)
    q = _candidates_params(rows, state)
    with torch.cuda.device(logits.device):
        check(lib.pcv_contrastive_rank(C.byref(p), _stream()), "pcv_contrastive_rank")
        if pp is not None:
            check(lib.pcv_logits_process(C.byref(pp), _stream()), "pcv_logits_process")
        check(lib.pcv_contrastive_candidates(C.byref(q), _stream()), "pcv_contrastive_candidates")
    return state.tokens, state.parents


def tcgen05_supported(q, k, v, num_heads: int, pad_mask=None, causal: bool = False) -> bool:
    """True when pcv_attn_fwd would pick the tcgen05 kernel for these operands."""
    q, k, v, _ = _prep(q, k, v, num_heads=num_heads, pad=True)  # the forward's padding rule
    with torch.cuda.device(k.device):
        p, keep = _fill_attn_params(q, k, v, num_heads, 1.0, pad_mask, causal, None, 0, "auto")
        dummy = torch.empty(16, device=k.device)
        p.out = dummy.data_ptr()
        return bool(_lib.lib().pcv_attn_supported_tcgen05(C.byref(p)))


# --------------------------------------------------------------------------------------------------
# fused K/V producer (SURVEY.md §8(f)1): LayerNorm folded around ONE tcgen05 GEMM that writes K and V
# --------------------------------------------------------------------------------------------------
def ln_stats(x: torch.Tensor, eps: float) -> torch.Tensor:
    """Row statistics of nn.LayerNorm over the last dim of x (..., C): (rows, 2) float32 = (mean, rstd)."""
    _require_cuda(x)
    x2 = _rows2d(x)
    stats = torch.empty(x2.shape[0], 2, dtype=torch.float32, device=x.device)
    p = LnStatsParams()
    p.x, p.stats = x2.data_ptr(), stats.data_ptr()
    p.x_stride_row, p.rows, p.C, p.eps = x2.stride(0), x2.shape[0], x2.shape[1], float(eps)
    p.dtype = _pcv_dtype(x2.dtype)
    with torch.cuda.device(x.device):
        check(_lib.lib().pcv_ln_stats(C.byref(p), _stream()), "pcv_ln_stats")
    return stats


def _rows2d(x: torch.Tensor) -> torch.Tensor:
    """(..., C) -> (rows, C) view with ONE row stride (copies only if the leading dims are not collapsible)."""
    if x.dim() == 2:
        return x if x.stride(1) == 1 else x.contiguous()
    x2 = x if x.stride(-1) == 1 else x.contiguous()
    try:
        return x2.view(-1, x2.shape[-1])
    except RuntimeError:
        return x2.reshape(-1, x2.shape[-1])


def fold_ln_linear(norm_weight, norm_bias, weights, biases, dtype: torch.dtype):
    """Fold a LayerNorm's affine part into the Linear layers that follow it (host-side, once per set of weights).

    ``weights``: list of (n_i, C) Linear weights applied to LN(x); ``biases``: matching list (entries may be None).
    Returns ``(w_cat (sum n_i, C) in `dtype`, col_st (sum n_i, 2) float32)`` with
    ``w_cat = gamma * W`` (rounded), ``s = rowsum(w_cat)`` of the ROUNDED weights and ``t = W @ beta + bias``, so that
    ``LN(x) W^T + b == rstd * (x w_cat^T - mean * s) + t`` (include/pcv_attn.h, pcv_kvproj_params).
    ``norm_weight`` / ``norm_bias`` None = no LayerNorm (``w_cat = W``, ``t = bias``)."""
    w = torch.cat([wi.detach().float() for wi in weights], dim=0)
    n, Cin = w.shape
    b = torch.cat([(torch.zeros(wi.shape[0], device=w.device) if bi is None else bi.detach().float())
                   for wi, bi in zip(weights, biases)])
    if norm_weight is not None:
        t = b + (w @ norm_bias.detach().float() if norm_bias is not None else 0.0)
        w = w * norm_weight.detach().float()[None, :]
    else:
        t = b
    w_cat = w.to(dtype).contiguous()
    s = w_cat.float().sum(dim=1)
    col_st = torch.stack([s, t], dim=1).contiguous()
    return w_cat, col_st


E4M3_MAX = 448.0  # largest finite float8_e4m3fn


def fp8_descales(norm_weight, norm_bias, weight, bias, num_heads: int, per_channel: bool = False) -> torch.Tensor:
    """FP8 dequantisation factors of ``y = LN(x) W^T + b`` derived from the weights alone (once per set of weights).

    For a LayerNorm'd row ``||x_hat||_2 <= sqrt(C)``, so output column n obeys
    ``|y_n| <= sqrt(C) * ||gamma * W_n||_2 + |t_n|`` with ``t`` the folded bias of :func:`fold_ln_linear`.  Returns that
    bound / 448 per head (``(H,)``: the max over the head's channels, for q and k) or per channel (``(H, d)``, for v),
    float32.  Quantising ``y / descale`` to e4m3 then never saturates.  ``norm_weight`` None = no LayerNorm: the bound
    is not valid then, so it is refused."""
    if norm_weight is None:
        raise ValueError("fp8_descales: the bound needs the LayerNorm in front of the projection")
    w, col_st = fold_ln_linear(norm_weight, norm_bias, [weight], [bias], torch.float32)
    n, cin = w.shape
    if n % num_heads:
        raise ValueError(f"fp8_descales: {n} output channels are not divisible by {num_heads} heads")
    bound = math.sqrt(cin) * w.double().norm(dim=1) + col_st[:, 1].double().abs()
    bound = bound.view(num_heads, n // num_heads)
    if not per_channel:
        bound = bound.amax(dim=1)
    # a channel with an all-zero weight row and bias is exactly zero: any positive descale quantises it exactly
    return (bound / E4M3_MAX).clamp_min(torch.finfo(torch.float32).tiny).float().contiguous()


def fp8_pair_descale(channel_descale: torch.Tensor, rotate_dim: int = 0) -> torch.Tensor:
    """Per-head K descale (H,) of an FP8 KV cache from the per-channel descales (H, d) of :func:`fp8_descales`.

    A rotary channel mixes its pair, ``a cos - b sin``, so under rotation channels 2p and 2p+1 of the first
    ``rotate_dim`` channels are bounded by the pair norm ``sqrt(b_2p^2 + b_2p+1^2)`` of their single-channel bounds, not
    by either alone; the other channels by their own bound.  The per-head maximum of these bounds holds for the rows
    before and after rotation, so one descale serves a cache and its rotated shadow."""
    b = channel_descale.double()
    if rotate_dim:
        if rotate_dim % 2 or rotate_dim > b.shape[1]:
            raise ValueError(f"fp8_pair_descale: rotate_dim {rotate_dim} must be even and <= {b.shape[1]}")
        pair = b[:, :rotate_dim].reshape(b.shape[0], -1, 2).norm(dim=-1)
        b = torch.cat([pair.repeat_interleave(2, dim=1), b[:, rotate_dim:]], dim=1)
    return b.amax(dim=1).float().contiguous()


def fp8_dequantize(x8: torch.Tensor, descale: torch.Tensor, num_heads: int, dtype: torch.dtype) -> torch.Tensor:
    """(..., H*d) e4m3 codes -> ``codes * descale`` in ``dtype`` (descale (H,) per head or (H, d) per channel)."""
    xs = x8.float().reshape(*x8.shape[:-1], num_heads, x8.shape[-1] // num_heads)
    d = descale.float().to(x8.device)
    d = d[:, None] if d.dim() == 1 else d
    return (xs * d).reshape(x8.shape).to(dtype)


def _fill_decode(q, k, v, num_heads, scale, pad_mask, causal, k_descale=None, v_descale=None):
    """(AttnParams, DecodeFp8 or None, tensors to keep alive) of a decode launch.  bf16 / fp16 K / V rows are taken like
    :func:`attention` takes them (f None); e4m3 rows, or given descales, are those of :func:`attention_decode_fp8`."""
    if k.dtype != F8 and v.dtype != F8 and k_descale is None and v_descale is None:
        q, k, v, _ = _prep(q, k, v)
        p, keep = _fill_attn_params(q, k, v, num_heads, scale, pad_mask, causal, None, 0, "decode")
        return p, None, keep
    _require_cuda(q, k, v, k_descale, v_descale, pad_mask)
    if k.dtype != F8 or v.dtype != F8:
        raise ValueError(f"attention_decode_fp8: k8 / v8 must be torch.float8_e4m3fn, got {k.dtype} / {v.dtype}")
    q = _rows_contiguous(q if q.dtype in (torch.bfloat16, torch.float16) else q.to(torch.bfloat16))
    k, v = _rows_contiguous(k), _rows_contiguous(v)
    p, keep = _fill_attn_params(q, k, v, num_heads, scale, pad_mask, causal, None, 0, "decode")
    kd, vd = k_descale.float().contiguous(), v_descale.float().contiguous()
    if kd.shape != (p.H,) or vd.shape != (p.H, p.dv):
        raise ValueError(f"attention_decode_fp8: descales must be (H,) and (H, dv) = ({p.H},), ({p.H}, {p.dv})")
    f = _lib.DecodeFp8()
    f.k_descale, f.v_descale = kd.data_ptr(), vd.data_ptr()
    return p, f, keep + (q, kd, vd)


#: Query rows up to which an e4m3-cache call runs the streaming decode kernel; more rows (up to 64) take the
#: tensor-core kernel of pcv_attn_cached_fp8.
DECODE_MAX_ROWS = 4


def _fp8_entry(p, f, rows) -> str:
    """The entry point of a decode launch: pcv_attn_cached_fp8 for e4m3 rows of more than DECODE_MAX_ROWS query rows
    without a window (its impl is AUTO), else pcv_attn_decode(_window)(_fp8)."""
    if f is not None and rows is None and p.N > DECODE_MAX_ROWS:
        p.impl = _lib.PCV_IMPL_AUTO
        return "pcv_attn_cached_fp8"
    return "pcv_attn_decode" + ("_window" if rows is not None else "") + ("_fp8" if f is not None else "")


def _run_decode(p, f, rows, device) -> None:
    """Size and attach the workspace of the decode launch ``p`` and enqueue it: e4m3 K / V rows when ``f`` (DecodeFp8)
    is given, the key window read from device memory when ``rows`` (DevRows) is (pcv_attn_decode_fp8, _window,
    _window_fp8, or pcv_attn_cached_fp8 for 5 to 64 query rows on e4m3 rows)."""
    entry = _fp8_entry(p, f, rows)
    sizer = "pcv_attn_decode_window" if rows is not None else "pcv_attn_decode_fp8"  # the four decode entries' workspace
    ws = _workspace(p, device, entry if entry == "pcv_attn_cached_fp8" else sizer, C.byref(p))
    check(getattr(_lib.lib(), entry)(*(C.byref(s) for s in (p, f, rows) if s is not None), _stream()), entry)
    del ws


def attention_decode_fp8_supported(q, k8, v8, k_descale, v_descale, num_heads: int, scale: float = 1.0,
                                   pad_mask=None, causal: bool = False) -> bool:
    """Whether :func:`attention_decode_fp8` covers these operands (no launch; reason in ``_lib.lib().pcv_last_error()``)."""
    with torch.cuda.device(k8.device):
        p, f, keep = _fill_decode(q, k8, v8, num_heads, scale, pad_mask, causal, k_descale, v_descale)
        dummy = torch.empty(64, device=k8.device)
        p.out = dummy.data_ptr()
        p.o_stride_b, p.o_stride_n, p.o_stride_h = p.N * p.H * p.dv, p.H * p.dv, p.dv
        entry = _fp8_entry(p, f, None)
        return bool(getattr(_lib.lib(), entry + "_supported")(C.byref(p), C.byref(f)))


def attention_decode_fp8(q, k8, v8, k_descale, v_descale, num_heads: int, scale: float, pad_mask=None,
                         causal: bool = False) -> torch.Tensor:
    """Attention of 1 to 64 query rows on an FP8 (e4m3) KV cache.

    q: (B or 1, N <= 64, H*dqk) bf16 / fp16; k8: (B, M, H*dqk), v8: (B, M, H*dv) ``torch.float8_e4m3fn`` rows standing for
    ``k8 * k_descale[h]`` and ``v8[..., h, c] * v_descale[h, c]`` (float32 (H,) and (H, dv)).  Masks as in
    :func:`attention`.  Returns (B, N, H*dv) in q's dtype.  Up to DECODE_MAX_ROWS (4) query rows run the streaming
    decode kernel (pcv_attn_decode_fp8), whose probabilities stay fp32; 5 to 64 rows the tensor-core kernel
    (pcv_attn_cached_fp8), which converts the e4m3 tiles to q's dtype in shared memory and rounds P to q's dtype before
    P V, as :func:`attention` does.  Head dims: multiples of 16, at most 256.  No autograd: this is an inference path."""
    with torch.cuda.device(k8.device):
        p, f, keep = _fill_decode(q, k8, v8, num_heads, scale, pad_mask, causal, k_descale, v_descale)
        out = _new_output(p, _compute_dtype(q.dtype), k8.device)
        _run_decode(p, f, None, k8.device)
    del keep
    return out


def _fill_kvproj(x2, w_cat, col_st, n_k, n_v, stats, k_out, v_out, cta_group=0, ln_eps=0.0) -> KvProjParams:
    p = KvProjParams()
    p.x, p.w, p.col_st = x2.data_ptr(), w_cat.data_ptr(), col_st.data_ptr()
    p.row_stats = None if stats is None else stats.data_ptr()
    p.k_out = None if k_out is None else k_out.data_ptr()
    p.v_out = None if v_out is None else v_out.data_ptr()
    p.x_stride_row = x2.stride(0)
    p.k_stride_row = 0 if k_out is None else k_out.stride(0)
    p.v_stride_row = 0 if v_out is None else v_out.stride(0)
    p.rows, p.C, p.n_k, p.n_v = x2.shape[0], x2.shape[1], n_k, n_v
    p.dtype = _pcv_dtype(x2.dtype)
    p.cta_group = cta_group
    p.ln_eps = float(ln_eps)
    return p


def _check_folded(fn: str, x: torch.Tensor, w_cat: torch.Tensor, col_st: torch.Tensor, n: int) -> None:
    if w_cat.dtype != x.dtype or w_cat.shape != (n, x.shape[-1]) or not w_cat.is_contiguous():
        raise ValueError(f"{fn}: w_cat must be a contiguous (n_k + n_v, C) tensor in x's dtype")
    if col_st.dtype != torch.float32 or col_st.shape != (n, 2) or not col_st.is_contiguous():
        raise ValueError(f"{fn}: col_st must be a contiguous (n_k + n_v, 2) float32 tensor")


def _producer_stats(x2: torch.Tensor, eps: Optional[float], mode: str):
    """``(row statistics, ln_eps)`` of the producer's LayerNorm (``eps`` None: none): pcv_ln_stats, or in-kernel.
    The kernel computes statistics in-kernel only for ``ln_eps > 0`` (without statistics it reads ``ln_eps = 0`` as "no
    LayerNorm"), so a LayerNorm with ``eps = 0`` takes pcv_ln_stats whatever the mode.  With statistics, ``ln_eps`` is
    the eps they were computed with: the kernel writes the folded bias for their zero-variance rows."""
    if eps is None:
        return None, 0.0
    if eps > 0.0 and mode == "fused":
        return None, eps
    return ln_stats(x2, eps), eps


def _project_rows(x2: torch.Tensor, w_cat, col_st, n_k: int, n_v: int, stats, ln_eps=0.0, cta_group: int = 0):
    """pcv_kv_project of x2 (rows, C): new (rows, n_k) and (rows, n_v) tensors in x2's dtype (None for a width of 0)."""
    k_out = torch.empty(x2.shape[0], n_k, dtype=x2.dtype, device=x2.device) if n_k else None
    v_out = torch.empty(x2.shape[0], n_v, dtype=x2.dtype, device=x2.device) if n_v else None
    p = _fill_kvproj(x2, w_cat, col_st, n_k, n_v, stats, k_out, v_out, cta_group, ln_eps)
    check(_lib.lib().pcv_kv_project(C.byref(p), _stream()), "pcv_kv_project")
    return k_out, v_out


def kv_project_supported(x: torch.Tensor, n_k: int, n_v: int) -> bool:
    """True when ``kv_project`` covers (x, n_k, n_v): CUDA bf16/fp16 rows, widths/strides TMA can address."""
    if not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16) or x.numel() == 0:
        return False
    C_in = x.shape[-1]
    return C_in % 8 == 0 and n_k % 64 == 0 and n_v % 8 == 0 and (n_k + n_v) > 0


#: ``stats``: "separate" = pcv_ln_stats first (two-pass statistics; x is read twice, at the copy bandwidth), "fused" =
#: statistics computed inside the GEMM kernel from the staged tiles (x crosses HBM once).  The default is the numerically
#: more conservative two-pass variant.
kv_project_config = {"stats": "separate"}


def kv_project(x: torch.Tensor, w_cat: torch.Tensor, col_st: torch.Tensor, n_k: int, n_v: int,
               eps: Optional[float] = 1e-5, cta_group: int = 0, stats: Optional[str] = None):
    """K, V = LN(x) Wk^T + bk, LN(x) Wv^T + bv for x (..., C) through pcv_kv_project (statistics in-kernel or by
    pcv_ln_stats, see ``kv_project_config``).

    ``w_cat`` / ``col_st`` come from :func:`fold_ln_linear`; ``eps=None`` skips the LayerNorm (plain projection).
    Returns contiguous (..., n_k) and (..., n_v) tensors in x's dtype (``None`` for a width of 0)."""
    _require_cuda(x, w_cat, col_st)
    _check_folded("kv_project", x, w_cat, col_st, n_k + n_v)
    lead = x.shape[:-1]
    x2 = _rows2d(x)
    with torch.cuda.device(x.device):
        st, ln_eps = _producer_stats(x2, eps, kv_project_config["stats"] if stats is None else stats)
        k_out, v_out = _project_rows(x2, w_cat, col_st, n_k, n_v, st, ln_eps, cta_group)
    return tuple(None if o is None else o.view(*lead, o.shape[1]) for o in (k_out, v_out))


def fp8_quantize(x: torch.Tensor, descale: torch.Tensor, num_heads: int) -> torch.Tensor:
    """(..., H*d) values -> e4m3 codes of ``x / descale`` (descale (H,) per head or (H, d) per channel), rounded to
    nearest even and saturated at +-448.  A torch reference of the producer's e4m3 epilogue for tests and tools; the
    module's FP8 route quantises inside :func:`kv_project_fp8` instead."""
    H = num_heads
    xs = x.float().reshape(*x.shape[:-1], H, x.shape[-1] // H)
    d = descale.float().to(x.device)
    d = d[:, None] if d.dim() == 1 else d
    return (xs / d).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).reshape(x.shape)


def fp8_transpose_v(v8: torch.Tensor, num_heads: int, m_pad: Optional[int] = None) -> torch.Tensor:
    """(B, M, H*dv) e4m3 -> V^T (B, H, dv, M_pad) e4m3, keys contiguous and in order (M_pad: M rounded up to 16; the
    pad keys are zero and never read).  The layout :func:`attention_fp8` takes and :func:`kv_project_fp8` writes."""
    B, M, Cv = v8.shape
    dv = Cv // num_heads
    m_pad = (M + 15) // 16 * 16 if m_pad is None else m_pad
    vt = torch.zeros(B, num_heads, dv, m_pad, dtype=torch.uint8, device=v8.device)
    vt[..., :M] = v8.view(torch.uint8).reshape(B, M, num_heads, dv).permute(0, 2, 3, 1)
    return vt.view(torch.float8_e4m3fn)


def _fill_kvproj_fp8(x2, w_cat, col_st, inv_scale, n_k, n_v, stats, k8, vt8, keys_per_batch, v_head_dim, ln_eps):
    p = _fill_kvproj(x2, w_cat, col_st, n_k, n_v, stats, k8, None, 0, ln_eps)
    f = _lib.KvProjFp8()
    f.inv_scale = inv_scale.data_ptr()
    if vt8 is not None:
        f.vt_out = vt8.data_ptr()
        f.vt_stride_b, f.vt_stride_h, f.vt_stride_c = vt8.stride(0), vt8.stride(1), vt8.stride(2)
    f.keys_per_batch = int(keys_per_batch)
    f.v_head_dim = int(v_head_dim)
    return p, f


def kv_project_fp8_supported(x: torch.Tensor, n_k: int, n_v: int, num_heads: int) -> bool:
    """Whether :func:`kv_project_fp8` covers x (..., C) with these widths (no launch)."""
    if not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16) or x.dim() < 2:
        return False
    x2 = _rows2d(x)
    rows = x2.shape[0]
    p = KvProjParams()
    p.x = p.w = p.col_st = x2.data_ptr()
    p.k_out = x2.data_ptr() if n_k else None
    p.x_stride_row, p.k_stride_row, p.rows = x2.stride(0), n_k, rows
    p.C, p.n_k, p.n_v, p.dtype = x2.shape[1], n_k, n_v, _pcv_dtype(x.dtype)
    f = _lib.KvProjFp8()
    f.inv_scale = x2.data_ptr()
    dv = n_v // num_heads if n_v else 16
    m = x.shape[-2] if x.dim() >= 3 else rows
    f.vt_out = x2.data_ptr() if n_v else None
    mp = (m + 15) // 16 * 16
    f.vt_stride_c, f.vt_stride_h, f.vt_stride_b = mp, mp * dv, mp * dv * num_heads
    f.keys_per_batch, f.v_head_dim = m, dv
    with torch.cuda.device(x.device):
        return bool(_lib.lib().pcv_kv_project_fp8_supported(C.byref(p), C.byref(f)))


def kv_project_fp8(x: torch.Tensor, w_cat: torch.Tensor, col_st: torch.Tensor, inv_scale: torch.Tensor, n_k: int,
                   n_v: int, num_heads: int, eps: Optional[float] = 1e-5):
    """The fused producer with e4m3 outputs (pcv_kv_project_fp8): ``LN(x) W^T + b`` of x (B, M, C), column n
    multiplied by ``inv_scale[n]`` (float32, n_k + n_v; 1 / the descales of :func:`fp8_descales`) and rounded to e4m3.

    Returns ``(k8, vt8)``: k8 (B, M, n_k) e4m3 rows (or None), vt8 the V columns transposed, (B, H, n_v / H, M_pad)
    e4m3 as :func:`attention_fp8` takes them (or None).  With n_v = 0 this produces q.  No extra pass over the data:
    the LayerNorm statistics come from the GEMM kernel (or pcv_ln_stats) as in :func:`kv_project`."""
    _require_cuda(x, w_cat, col_st, inv_scale)
    if x.dim() != 3:
        raise ValueError("kv_project_fp8: x must be (B, M, C)")
    _check_folded("kv_project_fp8", x, w_cat, col_st, n_k + n_v)
    inv = inv_scale.float().contiguous()
    if inv.shape != (n_k + n_v,):
        raise ValueError("kv_project_fp8: inv_scale must be (n_k + n_v,)")
    B, M, _ = x.shape
    x2 = _rows2d(x)
    dv = n_v // num_heads if n_v else 16
    with torch.cuda.device(x.device):
        st, ln_eps = _producer_stats(x2, eps, kv_project_config["stats"])
        k8 = torch.empty(B * M, n_k, dtype=torch.float8_e4m3fn, device=x.device) if n_k else None
        vt8 = None
        if n_v:
            m_pad = (M + 15) // 16 * 16
            vt8 = torch.empty(B, num_heads, dv, m_pad, dtype=torch.float8_e4m3fn, device=x.device)  # pad keys: never read
        p, f = _fill_kvproj_fp8(x2, w_cat, col_st, inv, n_k, n_v, st, k8, vt8, M, dv, ln_eps)
        check(_lib.lib().pcv_kv_project_fp8(C.byref(p), C.byref(f), _stream()), "pcv_kv_project_fp8")
    return (None if k8 is None else k8.view(B, M, n_k)), vt8


# --------------------------------------------------------------------------------------------------
# training through the LayerNorm -> Linear chain: the fused producer forward + pcv_ln_linear_bwd
# --------------------------------------------------------------------------------------------------
def _gemm_rows(t: torch.Tensor, n: int) -> torch.Tensor:
    """(..., n) -> (rows, n) with unit column stride, a row stride that is a multiple of 8 elements and covers the row,
    and 16-byte alignment (copied if not: a gradient broadcast along the rows has row stride 0)."""
    t2 = t.reshape(-1, n)
    if t2.stride(1) != 1 or t2.stride(0) < n or t2.stride(0) % 8 or t2.data_ptr() % 16:
        t2 = t2.contiguous() if not t2.is_contiguous() else t2.clone()
    return t2


def ln_linear_backward(x: torch.Tensor, stats: torch.Tensor, w: torch.Tensor, gamma: Optional[torch.Tensor],
                       beta: Optional[torch.Tensor], grad_k: Optional[torch.Tensor], grad_v: Optional[torch.Tensor],
                       n_k: int, n_v: int, needs=(True, True, True, True, True)):
    """Gradients of ``[k | v] = LN(x) W^T + b`` (LN(x) = (x - mean) * rstd * gamma + beta) through pcv_ln_linear_bwd.

    x (rows, C) 16-bit with ``stats`` (rows, 2) f32 from :func:`ln_stats`; w the UNFOLDED (n_k + n_v, C) weights; gamma /
    beta (C) or None; grad_k (rows, n_k), grad_v (rows, n_v) (None for a width of 0).  ``needs`` selects
    (grad_x, grad_w, grad_b, grad_gamma, grad_beta); unneeded ones come back as None.  Bitwise reproducible."""
    _require_cuda(x, stats, w, gamma, beta, grad_k, grad_v)
    dt = x.dtype
    rows, Cin = x.shape
    if w.dtype != dt or w.shape != (n_k + n_v, Cin) or not w.is_contiguous():
        raise ValueError("ln_linear_backward: w must be a contiguous (n_k + n_v, C) tensor in x's dtype")
    for name, t in (("gamma", gamma), ("beta", beta)):
        if t is not None and (t.dtype != dt or t.shape != (Cin,) or not t.is_contiguous()):
            raise ValueError(f"ln_linear_backward: {name} must be a contiguous (C,) tensor in x's dtype")
    gk = _gemm_rows(grad_k.to(dt), n_k) if n_k else None
    gv = _gemm_rows(grad_v.to(dt), n_v) if n_v else None
    dev = x.device
    out = [torch.empty(rows, Cin, dtype=dt, device=dev) if needs[0] else None,
           torch.empty(n_k + n_v, Cin, dtype=dt, device=dev) if needs[1] else None,
           torch.empty(n_k + n_v, dtype=dt, device=dev) if needs[2] else None,
           torch.empty(Cin, dtype=dt, device=dev) if needs[3] else None,
           torch.empty(Cin, dtype=dt, device=dev) if needs[4] else None]
    if all(o is None for o in out):
        return tuple(out)
    ptr = lambda t: None if t is None else t.data_ptr()
    p = _lib.LnLinearBwdParams()
    p.x, p.x_stride_row, p.row_stats = x.data_ptr(), x.stride(0), stats.data_ptr()
    p.w, p.gamma, p.beta = w.data_ptr(), ptr(gamma), ptr(beta)
    p.grad_k, p.grad_v = ptr(gk), ptr(gv)
    p.gk_stride_row = gk.stride(0) if gk is not None else 0
    p.gv_stride_row = gv.stride(0) if gv is not None else 0
    p.grad_x, p.grad_w, p.grad_b, p.grad_gamma, p.grad_beta = (ptr(o) for o in out)
    p.rows, p.C, p.n_k, p.n_v, p.dtype = rows, Cin, n_k, n_v, _pcv_dtype(dt)
    with torch.cuda.device(dev):
        ws = _workspace(p, dev, "pcv_ln_linear_bwd", C.byref(p))  # noqa: F841 (kept until the launch is enqueued)
        check(_lib.lib().pcv_ln_linear_bwd(C.byref(p), _stream()), "pcv_ln_linear_bwd")
    return tuple(out)


class _LnLinear(torch.autograd.Function):
    """[k | v] = LN(x) W^T + b: forward by pcv_ln_stats + the fused producer (y is never materialised), backward by
    pcv_ln_linear_bwd.  Saves x, the row statistics and the parameters."""

    @staticmethod
    def forward(ctx, x, gamma, beta, w, b, w_cat, col_st, n_k: int, n_v: int, eps: float):
        lead = x.shape[:-1]
        x2 = _rows2d(x)
        with torch.cuda.device(x.device):
            st = ln_stats(x2, eps)
            k_out, v_out = _project_rows(x2, w_cat, col_st, n_k, n_v, st, eps)
        ctx.save_for_backward(x2, st, w, gamma, beta)
        ctx.dims = (x.shape, n_k, n_v, b is not None)
        outs = [o.view(*lead, o.shape[1]) for o in (k_out, v_out) if o is not None]
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        x2, st, w, gamma, beta = ctx.saved_tensors
        shape, n_k, n_v, has_b = ctx.dims
        ni = ctx.needs_input_grad
        rows = x2.shape[0]
        g = list(grads)
        for i, n in enumerate(d for d in (n_k, n_v) if d):
            if g[i] is None:
                g[i] = torch.zeros(rows, n, dtype=x2.dtype, device=x2.device)
        gk = g[0] if n_k else None
        gv = (g[1] if n_k else g[0]) if n_v else None
        needs = (ni[0], ni[3], ni[4] and has_b, ni[1] and gamma is not None, ni[2] and beta is not None)
        dx, dw, db, dgamma, dbeta = ln_linear_backward(x2, st, w, gamma, beta, gk, gv, n_k, n_v, needs)
        return (None if dx is None else dx.view(shape)), dgamma, dbeta, dw, db, None, None, None, None, None


def ln_linear(x: torch.Tensor, norm_weight: Optional[torch.Tensor], norm_bias: Optional[torch.Tensor], weights, biases,
              n_k: int, n_v: int, eps: float = 1e-5, w_cat: Optional[torch.Tensor] = None,
              col_st: Optional[torch.Tensor] = None):
    """Differentiable ``LN(x) [W_k; W_v]^T + [b_k; b_v]`` of x (..., C) on this package's kernels: the forward is
    :func:`kv_project` with separate statistics, the backward :func:`ln_linear_backward`.  ``weights`` / ``biases``
    are the Linear layers' tensors (biases may be None) whose concatenation has n_k + n_v rows; ``norm_weight`` /
    ``norm_bias`` the LayerNorm's (None = no affine part).  ``w_cat`` / ``col_st``: the folded weights of
    :func:`fold_ln_linear` when the caller caches them.  Returns (k, v), v None when n_v == 0."""
    _require_cuda(x)
    dt = x.dtype
    if w_cat is None or col_st is None:
        w_cat, col_st = fold_ln_linear(norm_weight, norm_bias, list(weights), list(biases), dt)
    w = torch.cat([wi.to(dt) for wi in weights], dim=0) if len(weights) > 1 else weights[0].to(dt)
    if all(bi is None for bi in biases):
        b = None
    else:
        b = torch.cat([(torch.zeros(wi.shape[0], dtype=dt, device=x.device) if bi is None else bi.to(dt))
                       for wi, bi in zip(weights, biases)])
    gamma = None if norm_weight is None else norm_weight.to(dt)
    beta = None if norm_bias is None else norm_bias.to(dt)
    outs = _LnLinear.apply(x, gamma, beta, w.contiguous(), b, w_cat, col_st, n_k, n_v, float(eps))
    return (outs[0], outs[1]) if (n_k and n_v) else ((outs[0], None) if n_k else (None, outs[0]))


# --------------------------------------------------------------------------------------------------
# logits processors (pcv_logits_process): 🤗's repetition penalty, n-gram blocking and minimum new tokens on fp32 rows,
# with the token histories and their lengths on the device, recordable in a CUDA graph.
# --------------------------------------------------------------------------------------------------
#: The largest no_repeat_ngram_size and EOS count :func:`process_logits` takes.
PROCESS_MAX_NGRAM = _lib.PROCESS_MAX_NGRAM
PROCESS_MAX_EOS = _lib.PROCESS_MAX_EOS


def _history(what: str, ids, length, R: int, per: int, device):
    """(pointer, row stride, cap, length pointer, length stride, count) of one history segment."""
    _require_cuda(ids)
    if ids.dtype != torch.int64 or ids.dim() != 2 or ids.stride(1) != 1:
        raise ValueError(f"process_logits: {what} must be a (rows, cap) int64 tensor with unit column stride, got "
                         f"{tuple(ids.shape)} {ids.dtype}")
    need = -(-R // per)
    if ids.shape[0] < need:
        raise ValueError(f"process_logits: {what} has {ids.shape[0]} rows; {R} processed rows at {per} per history "
                         f"row read {need}")
    if ids.device != device:
        raise ValueError(f"process_logits: {what} is on {ids.device}, the logits on {device}")
    if isinstance(length, torch.Tensor):
        _require_cuda(length)
        if length.device != device:
            raise ValueError(f"process_logits: {what}_len is on {length.device}, the logits on {device}")
        if length.dtype != torch.int32 or length.numel() not in (1, R) or (length.numel() == R and R > 1 and (
                length.dim() != 1 or length.stride(0) != 1)):
            raise ValueError(f"process_logits: {what}_len must be an int32 tensor of 1 or ({R},) elements, got "
                             f"{tuple(length.shape)} {length.dtype}")
        return ids.data_ptr(), ids.stride(0), ids.shape[1], length.data_ptr(), 1 if length.numel() > 1 else 0, 0
    n = _as_int(length)
    if n is None or not 0 <= n <= ids.shape[1]:
        raise ValueError(f"process_logits: {what}_len must be an integer in [0, {ids.shape[1]}] or an int32 CUDA "
                         f"tensor, got {length!r}")
    return ids.data_ptr(), ids.stride(0), ids.shape[1], None, 0, n


def process_logits(logits: torch.Tensor, prefix: torch.Tensor, prefix_len, *, tail: Optional[torch.Tensor] = None,
                   tail_len: Optional[torch.Tensor] = None, rows_per_hist: int = 1, row_map: Optional[torch.Tensor] = None,
                   out: Optional[torch.Tensor] = None, log_softmax: bool = False, repetition_penalty: float = 1.0,
                   no_repeat_ngram_size: int = 0, min_new_tokens: int = 0, prompt_len: int = 0, eos=()) -> torch.Tensor:
    """🤗's ``RepetitionPenaltyLogitsProcessor`` -> ``NoRepeatNGramLogitsProcessor`` -> ``MinNewTokensLengthLogitsProcessor``
    on the device (pcv_logits_process), on fp32 rows; the rule is stated in ``include/pcv_attn.h``.

    ``logits`` (rows, V) bf16 / fp16 / fp32, V <= :data:`SAMPLE_MAX_VOCAB`.  Without ``row_map`` every row r is
    processed; with ``row_map`` (G,) int32 CUDA, row ``r * (rows // G) + row_map[r]`` of every group r of rows is.
    ``log_softmax=True`` processes the rows' fp32 log-softmax (the beam step's arithmetic) instead of the logits.
    Processed row r's history (🤗's ``input_ids``) is history row ``h = r // rows_per_hist``: ``prefix[h, :Lp]`` then
    ``tail[h, :Lt]``, int64 tensors with unit column stride; ``prefix_len`` is a host integer or an int32 CUDA tensor
    of one or one-per-processed-row elements, ``tail_len`` an int32 CUDA tensor of the same kind, both read when the
    kernel runs (clamped to the segment's width).  ``min_new_tokens`` counts from ``prompt_len``; it needs ``eos`` ids.
    Returns ``out`` (allocated as fp32 rows like ``logits`` when None) with the processed rows written and the others
    untouched.  Recordable in a CUDA graph; arguments the kernel does not take raise ``ValueError`` with its reason
    before any launch."""
    p, out = _process_params(logits, prefix, prefix_len, tail=tail, tail_len=tail_len, rows_per_hist=rows_per_hist,
                             row_map=row_map, out=out, log_softmax=log_softmax, repetition_penalty=repetition_penalty,
                             no_repeat_ngram_size=no_repeat_ngram_size, min_new_tokens=min_new_tokens,
                             prompt_len=prompt_len, eos=eos)
    with torch.cuda.device(out.device):
        check(_lib.lib().pcv_logits_process(C.byref(p), _stream()), "pcv_logits_process")
    return out


def _process_params(logits, prefix, prefix_len, *, tail=None, tail_len=None, rows_per_hist=1, row_map=None, out=None,
                    log_softmax=False, repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, prompt_len=0,
                    eos=()):
    """The checked ``pcv_logits_process_params`` of :func:`process_logits` and its output rows; no launch."""
    _require_cuda(logits, prefix)
    if logits.dim() != 2 or logits.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError(f"process_logits: logits must be (rows, V) bf16 / fp16 / fp32, got {tuple(logits.shape)} "
                         f"{logits.dtype}")
    rows = logits if logits.stride(-1) == 1 else logits.contiguous()
    n, V = rows.shape
    R, group = n, 1
    dev = rows.device
    if row_map is not None:
        _require_cuda(row_map)
        if row_map.device != dev:
            raise ValueError(f"process_logits: row_map is on {row_map.device}, the logits on {dev}")
        if row_map.dtype != torch.int32 or row_map.dim() != 1 or not row_map.is_contiguous() or row_map.numel() < 1 \
                or n % row_map.numel():
            raise ValueError(f"process_logits: row_map must be a contiguous (G,) int32 tensor with G dividing the {n} "
                             f"rows, got {tuple(row_map.shape)} {row_map.dtype}")
        R, group = row_map.numel(), n // row_map.numel()
    per = _as_int(rows_per_hist)
    if per is None or per < 1:
        raise ValueError(f"process_logits: rows_per_hist must be an integer >= 1, got {rows_per_hist!r}")
    if out is None:
        out = torch.empty(n, V, dtype=torch.float32, device=rows.device)
    elif not out.is_cuda or out.device != dev or out.dtype != torch.float32 or tuple(out.shape) != (n, V) or \
            out.stride(-1) != 1:
        raise ValueError(f"process_logits: out must be ({n}, {V}) fp32 with unit column stride, got "
                         f"{tuple(out.shape)} {out.dtype}")
    p = _lib.LogitsProcessParams()
    p.logits, p.stride_row = rows.data_ptr(), rows.stride(0) if n > 1 else V
    p.out, p.out_stride_row = out.data_ptr(), out.stride(0) if n > 1 else V
    p.row_map, p.row_group, p.R, p.V, p.rows_per_hist = (row_map.data_ptr() if row_map is not None else None), group, \
        R, V, per
    p.dtype = _lib.PCV_F32 if rows.dtype == torch.float32 else _pcv_dtype(rows.dtype)
    p.prefix, p.prefix_stride, p.prefix_cap, p.prefix_len, p.prefix_len_stride, p.prefix_count = _history(
        "prefix", prefix, prefix_len, R, per, dev)
    if tail is not None:
        _require_cuda(tail)
        if not isinstance(tail_len, torch.Tensor):
            raise ValueError("process_logits: a tail needs tail_len, an int32 CUDA tensor")
        p.tail, p.tail_stride, p.tail_cap, p.tail_len, p.tail_len_stride, _ = _history("tail", tail, tail_len, R, per,
                                                                                       dev)
    elif tail_len is not None:
        raise ValueError("process_logits: tail_len without a tail")
    theta, N, M, n0 = float(repetition_penalty), _as_int(no_repeat_ngram_size), _as_int(min_new_tokens), _as_int(prompt_len)
    if N is None or M is None or n0 is None or not -2 ** 31 <= min(N, M, n0) <= max(N, M, n0) < 2 ** 31:
        raise ValueError(f"process_logits: no_repeat_ngram_size, min_new_tokens and prompt_len must be int32 integers, "
                         f"got {no_repeat_ngram_size!r}, {min_new_tokens!r}, {prompt_len!r}")
    p.log_softmax, p.repetition_penalty, p.no_repeat_ngram, p.min_new_tokens, p.prompt_len = int(bool(log_softmax)), \
        theta, N, M, n0
    eos = list(eos)
    if len(eos) > PROCESS_MAX_EOS:
        raise ValueError(f"process_logits: at most {PROCESS_MAX_EOS} EOS ids, got {len(eos)}")
    p.n_eos = len(eos)
    for i, e in enumerate(eos):
        p.eos[i] = max(-2 ** 31, min(int(e), 2 ** 31 - 1))
    lib = _lib.lib()
    if not lib.pcv_logits_process_supported(C.byref(p)):
        raise ValueError(f"process_logits: {lib.pcv_last_error().decode()}")
    return p, out


# --------------------------------------------------------------------------------------------------
# prompt-lookup drafts (pcv_prompt_lookup): each batch row's n-gram drafts from its own history, found on the device;
# the round mode settles a verified round first.  Recordable in a CUDA graph.
# --------------------------------------------------------------------------------------------------
#: The largest num_output_tokens (G), max_matching_ngram_size (N) and EOS count :func:`prompt_lookup` takes.
LOOKUP_MAX_DRAFTS = _lib.LOOKUP_MAX_DRAFTS
LOOKUP_MAX_NGRAM = _lib.LOOKUP_MAX_NGRAM
LOOKUP_MAX_EOS = _lib.LOOKUP_MAX_EOS


def _row_ints(what: str, t, B: int, device, dtype=torch.int32):
    """The pointer and element stride of a (B,) tensor of ``dtype`` on ``device`` (any element stride)."""
    _require_cuda(t)
    if t.device != device or t.dtype != dtype or t.dim() != 1 or t.shape[0] != B:
        raise ValueError(f"prompt_lookup: {what} must be a ({B},) {dtype} tensor on {device}, got {tuple(t.shape)} "
                         f"{t.dtype} on {t.device}")
    return t.data_ptr(), t.stride(0)


def _lookup_params(ids, lengths, G, N, start, limit, eos, length_offset):
    """The checked ``pcv_prompt_lookup_params`` of a search; no launch."""
    _require_cuda(ids)
    if ids.dtype != torch.int64 or ids.dim() != 2 or ids.stride(1) != 1:
        raise ValueError(f"prompt_lookup: ids must be a (B, cap) int64 tensor with unit column stride, got "
                         f"{tuple(ids.shape)} {ids.dtype}")
    B, cap = ids.shape
    dev = ids.device
    p = _lib.PromptLookupParams()
    p.ids, p.ids_stride, p.B, p.cap = ids.data_ptr(), ids.stride(0) if B > 1 else cap, B, cap
    p.length, stride = _row_ints("lengths", lengths, B, dev)
    p.length_stride = stride
    if start is not None:
        p.start, _ = _row_ints("start", start, B, dev)
        if start.stride(0) != 1:
            raise ValueError("prompt_lookup: start must be contiguous")
    if limit is not None:
        p.limit, _ = _row_ints("limit", limit, B, dev)
        if limit.stride(0) != 1:
            raise ValueError("prompt_lookup: limit must be contiguous")
    g, n, off = _as_int(G), _as_int(N), _as_int(length_offset)
    if g is None or n is None or off is None or not -2 ** 31 <= min(g, n, off) <= max(g, n, off) < 2 ** 31:
        raise ValueError(f"prompt_lookup: num_output_tokens, max_matching_ngram_size and length_offset must be int32 "
                         f"integers, got {G!r}, {N!r}, {length_offset!r}")
    p.G, p.N, p.length_offset = g, n, off
    eos = list(eos)
    if len(eos) > LOOKUP_MAX_EOS or any(_as_int(e) is None or not -2 ** 63 <= e < 2 ** 63 for e in eos):
        raise ValueError(f"prompt_lookup: at most {LOOKUP_MAX_EOS} int64 EOS ids, got {eos!r}")
    p.n_eos = len(eos)
    for i, e in enumerate(eos):
        p.eos[i] = int(e)
    return p


def _launch_lookup(p) -> None:
    lib = _lib.lib()
    if not lib.pcv_prompt_lookup_supported(C.byref(p)):
        raise ValueError(f"prompt_lookup: {lib.pcv_last_error().decode()}")
    check(lib.pcv_prompt_lookup(C.byref(p), _stream()), "pcv_prompt_lookup")


def prompt_lookup(ids: torch.Tensor, lengths: torch.Tensor, num_output_tokens: int = 10,
                  max_matching_ngram_size: int = 2, *, start: Optional[torch.Tensor] = None,
                  limit: Optional[torch.Tensor] = None, eos=(), length_offset: int = 0):
    """Prompt-lookup drafts of every batch row (pcv_prompt_lookup): 🤗's ``PromptLookupCandidateGenerator.get_candidates``
    (no logits processor) on each row alone, with G = ``num_output_tokens`` and N = ``max_matching_ngram_size``; the
    rule is stated in ``include/pcv_attn.h``.

    ``ids`` (B, cap) int64 CUDA with unit column stride.  Row b's history is ``ids[b, start[b] : L_b]`` with
    ``L_b = lengths[b] + length_offset`` (``lengths`` a (B,) int32 CUDA tensor of any element stride, read when the
    kernel runs) and ``start`` (B,) int32 its left-padding count (None: 0).  ``limit`` (B,) int32 caps each row's
    draft (None: G); ``eos`` cuts a draft before its first EOS id.  Returns ``(drafts, counts)``: (B, G) int64, the
    draft then the history's last id as filler, and (B,) int32 draft lengths.  Nothing is read back to the host;
    recordable in a CUDA graph.  Arguments the kernel does not take raise ``ValueError`` before any launch."""
    p = _lookup_params(ids, lengths, num_output_tokens, max_matching_ngram_size, start, limit, eos, length_offset)
    drafts = torch.empty(p.B, max(p.G, 1), dtype=torch.int64, device=ids.device)
    counts = torch.empty(p.B, dtype=torch.int32, device=ids.device)
    p.drafts, p.drafts_stride, p.counts = drafts.data_ptr(), p.G, counts.data_ptr()
    _launch_lookup(p)
    return drafts, counts


def prompt_lookup_round(ids: torch.Tensor, lengths: torch.Tensor, length_offset: int, fed: torch.Tensor,
                        draws: torch.Tensor, next_tokens: torch.Tensor, state: torch.Tensor, num_output_tokens: int,
                        max_matching_ngram_size: int, *, start: Optional[torch.Tensor] = None, eos=()) -> None:
    """Round mode of :func:`prompt_lookup`: settle the speculative round that fed ``fed`` (B, k) int64 (t_0, the
    drafts, filler) and drew ``draws`` (B, k) int64, then search the next drafts; the rule is stated in
    ``include/pcv_attn.h``.  ``state`` (4, B) int32 CUDA, contiguous: [accepted (out), counts (in: the drafts fed;
    out: the next), unfinished, left].  ``next_tokens`` (B, >= G+1) int64 with unit column stride takes the next t_0
    in column 0 and the next drafts in columns 1 .. G; row L_b - 1 of ``ids`` (``L_b = lengths[b] + length_offset +
    n_b``) takes t_0.  In place, no host read; recordable in a CUDA graph."""
    p = _lookup_params(ids, lengths, num_output_tokens, max_matching_ngram_size, start, None, eos, length_offset)
    B, dev = p.B, ids.device
    k = fed.shape[1] if fed.dim() == 2 else 0
    for what, t in (("fed", fed), ("draws", draws)):
        _require_cuda(t)
        if t.device != dev or t.dtype != torch.int64 or tuple(t.shape) != (B, k) or not t.is_contiguous():
            raise ValueError(f"prompt_lookup_round: {what} must be a contiguous ({B}, k) int64 tensor on {dev}, got "
                             f"{tuple(t.shape)} {t.dtype}")
    _require_cuda(next_tokens, state)
    if next_tokens.device != dev or next_tokens.dtype != torch.int64 or next_tokens.dim() != 2 or \
            next_tokens.shape[0] != B or next_tokens.shape[1] < p.G + 1 or next_tokens.stride(1) != 1:
        raise ValueError(f"prompt_lookup_round: next_tokens must be a ({B}, >= {p.G + 1}) int64 tensor with unit "
                         f"column stride on {dev}")
    if state.device != dev or state.dtype != torch.int32 or tuple(state.shape) != (4, B) or not state.is_contiguous():
        raise ValueError(f"prompt_lookup_round: state must be a contiguous (4, {B}) int32 tensor on {dev}")
    p.k, p.fed, p.draws = k, fed.data_ptr(), draws.data_ptr()
    p.t0, p.t0_stride = next_tokens.data_ptr(), next_tokens.stride(0) if B > 1 else next_tokens.shape[1]
    p.drafts, p.drafts_stride = next_tokens.data_ptr() + 8, p.t0_stride
    p.accepted, p.counts, p.unfinished, p.left = (state[i].data_ptr() for i in range(4))
    _launch_lookup(p)
