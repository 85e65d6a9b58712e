"""Torch oracle of the FP8 attention forward (ops.attention_fp8): quantisation helpers and an fp64 emulation that
rounds the probabilities exactly where the kernel does.

The kernel rounds each probability as e4m3(P * 2^8), with P taken relative to the running row maximum of the work
segment at the end of the probability's 128-key tile; a segment is a range of key tiles of one (b, h, 128-row query
tile) in the work plan (``_lib.debug_plan``), and split segments are merged exactly.  The emulation walks the same
plan, so it rounds the same values; what is left between the two is fp32 accumulation and ex2.approx."""
from __future__ import annotations

import math

import torch

from perceiver_io_b200 import _lib, ops

F8 = torch.float8_e4m3fn
E4M3_MAX = 448.0
FLT_MAX = torch.finfo(torch.float32).max
LOG2E = 1.0 / math.log(2.0)


quantize = ops.fp8_quantize
make_vt = ops.fp8_transpose_v


def per_head_descale(x: torch.Tensor, num_heads: int, per_channel: bool = False) -> torch.Tensor:
    """amax / 448 of (..., H*d) values per head (H,) or per channel (H, d): data-derived scales for the tests."""
    a = x.float().abs().reshape(-1, num_heads, x.shape[-1] // num_heads).amax(dim=0)
    a = a if per_channel else a.amax(dim=1)
    return (a / E4M3_MAX).clamp_min(1e-12)


def score_scale(scale: float, q_descale: torch.Tensor, k_descale: torch.Tensor) -> torch.Tensor:
    """(H,) factor from q.k to the log2-domain score, formed in fp32 as the kernel forms it."""
    sl2 = torch.tensor(scale * LOG2E, dtype=torch.float32)  # TcParams::scale_log2 (scale * log2(e) in fp32)
    return (sl2 * q_descale.float().cpu() * k_descale.float().cpu()).double()


def round_p(p: torch.Tensor) -> torch.Tensor:
    """The kernel's rounding of a probability in [0, 1]: e4m3(P * 2^8) / 2^8."""
    return (p * 256.0).float().to(F8).double() / 256.0


def emulate(q8, k8, vt8, q_descale, k_descale, v_descale, num_heads: int, scale: float, pad_mask=None,
            causal: bool = False, m_total=None, m_offset: int = 0, workers: int = 132):
    """fp64 emulation of one pcv_attn_fwd_fp8 call on the plan for `workers` CTAs.

    Returns a dict of (B, H, N[, dv]) float64 tensors: the merged state ``o`` / ``m`` / ``l`` (log2 domain, as
    part_o / part_m / part_l), ``out = o / l``, and ``pv_abs`` = sum_j p_j |v_j| of the exact (unrounded) normalised
    probabilities, the scale of the test gates."""
    H = num_heads
    dev = k8.device
    Bq, N, Cq = q8.shape
    B, M, _ = k8.shape
    dqk = Cq // H
    dv = vt8.shape[2]
    m_total = M if m_total is None else m_total
    T = (M + 127) // 128
    Mt = T * 128
    q = q8.double().reshape(Bq, N, H, dqk).permute(0, 2, 1, 3).expand(B, H, N, dqk)
    k = k8.double().reshape(B, M, H, dqk).permute(0, 2, 1, 3)
    t = (q @ k.transpose(-1, -2)) * score_scale(scale, q_descale, k_descale).to(dev)[None, :, None, None]
    masked = torch.zeros(B, 1, N, M, dtype=torch.bool, device=dev)
    if pad_mask is not None:
        masked |= pad_mask.to(dev).bool()[:, None, None, :]
    if causal:
        shift = (m_total - N) - m_offset
        masked |= (torch.arange(M, device=dev)[None, :] > torch.arange(N, device=dev)[:, None] + shift)[None, None]
    t = t.masked_fill(masked, -FLT_MAX)
    t = torch.cat([t, torch.full((B, H, N, Mt - M), -math.inf, dtype=torch.float64, device=dev)], dim=-1)
    v8 = torch.zeros(B, H, Mt, dv, dtype=torch.float64, device=dev)
    v8[:, :, :M] = vt8[..., :M].double().transpose(-1, -2)
    vdesc = v_descale.double().to(dev)  # (H, dv)

    o = torch.zeros(B, H, N, dv, dtype=torch.float64, device=dev)
    m = torch.full((B, H, N), -math.inf, dtype=torch.float64, device=dev)
    l = torch.zeros(B, H, N, dtype=torch.float64, device=dev)
    _, segs = _lib.debug_plan(B, H, N, M, workers=workers, rows_per_unit=128)
    for (_, b, h, q0, _, t0, t1, _) in segs:
        q1 = min(q0 + 128, N)
        x = t[b, h, q0:q1, t0 * 128:t1 * 128].reshape(q1 - q0, t1 - t0, 128)
        m_run = torch.cummax(x.amax(dim=-1), dim=1).values  # running maximum after each tile
        mref = torch.where(m_run == -math.inf, torch.zeros_like(m_run), m_run)
        p = torch.exp2(x - mref[..., None])
        w = torch.exp2(mref - mref[:, -1:])  # rescale of each tile's terms to the segment's final reference
        seg_l = (p.sum(dim=-1) * w).sum(dim=1)
        vt = v8[b, h, t0 * 128:t1 * 128].reshape(t1 - t0, 128, dv)
        seg_o = (torch.einsum("rtk,tkc->rtc", round_p(p), vt) * w[..., None]).sum(dim=1)
        seg_m = mref[:, -1]
        m_old = m[b, h, q0:q1]
        m_new = torch.maximum(m_old, seg_m)
        a_old, a_seg = torch.exp2(m_old - m_new), torch.exp2(seg_m - m_new)
        o[b, h, q0:q1] = o[b, h, q0:q1] * a_old[:, None] + seg_o * a_seg[:, None]
        l[b, h, q0:q1] = l[b, h, q0:q1] * a_old + seg_l * a_seg
        m[b, h, q0:q1] = m_new
    o = o * vdesc[None, :, None, :]  # the kernel's epilogue: v_descale of the channel (2^-8 is in round_p)
    pe = torch.softmax(t[..., :M] / LOG2E, dim=-1) if M else None
    vdeq = v8[:, :, :M] * vdesc[None, :, None, :]
    pv_abs = pe @ vdeq.abs()
    return {"o": o, "m": m, "l": l, "out": o / l[..., None], "pv_abs": pv_abs}
