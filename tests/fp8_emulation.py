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
    # TcParams::scale_log2: the fp32 scale times the fp32 kLog2e, in fp32
    sl2 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    return (sl2 * q_descale.float().cpu() * k_descale.float().cpu()).double()


def round_p(p: torch.Tensor) -> torch.Tensor:
    """The kernel's rounding of a probability in [0, 1]: e4m3(P * 2^8) / 2^8."""
    return (p * 256.0).float().to(F8).double() / 256.0


U32 = 2.0 ** -24     # unit roundoff of fp32
EX2_REL = 2.0 ** -21  # relative error allowed for ex2.approx.ftz.f32 (2 ulp, with a factor 2 of margin)
MUTANTS = ("tile_max", "final_max", "no_prescale", "vd_next_channel", "vd_prev_pass", "qd_next_head")


def _round_e4m3(y: torch.Tensor) -> torch.Tensor:
    """Round-to-nearest-even e4m3 of fp64 values through fp32, as the kernel's cvt.rn.satfinite.e4m3x2.f32 sees them."""
    return y.float().to(F8).double()


def emulate(q8, k8, vt8, q_descale, k_descale, v_descale, num_heads: int, scale: float, pad_mask=None,
            causal: bool = False, m_total=None, m_offset: int = 0, workers: int = 132, mutant=None):
    """fp64 emulation of one pcv_attn_fwd_fp8 call on the plan for `workers` CTAs.

    Returns a dict of (B, H, N[, dv]) float64 tensors: the merged state ``o`` / ``m`` / ``l`` (log2 domain, as
    part_o / part_m / part_l), ``out = o / l``, and ``pv_abs`` = sum_j p_j |v_j| of the exact (unrounded) normalised
    probabilities, the scale of the test gates.  The terms of the per-element gate of fp8_fwd_variants.element_gate:
      - ``pv_hat`` = sum_j p^_j |v_j| / l with the rounded (and rescaled) probabilities p^ the numerator takes;
      - ``flip`` = sum_j s_j |v_j| / l over the probabilities whose e4m3 rounding can change under the kernel's
        exponent error (s_j the change of the rounded value, 0 elsewhere);
      - ``rho`` (B, H, N): the largest relative error of an fp32 probability of the row (exponent argument and ex2);
      - ``rho_w`` (B, H, N): the relative error of the fp32 rescale factors (running maximum and split merge);
      - ``nadd`` (B, H, N): the depth of the fp32 denominator sum.
    `mutant` (one of MUTANTS) emulates a kernel with that defect, for the tests that show the gate rejects it."""
    H = num_heads
    dev = k8.device
    Bq, N, Cq = q8.shape
    B, M, _ = k8.shape
    dqk = Cq // H
    dv = vt8.shape[2]
    m_total = M if m_total is None else m_total
    T = (M + 127) // 128
    Mt = T * 128
    if mutant is not None and mutant not in MUTANTS:
        raise KeyError(mutant)
    if mutant == "qd_next_head":
        q_descale = torch.roll(q_descale, -1, dims=0)
    if mutant == "vd_next_channel":
        v_descale = torch.roll(v_descale, -1, dims=1)
    if mutant == "vd_prev_pass":
        v_descale = torch.cat([v_descale[:, :128], v_descale[:, :-128]], dim=1)
    q = q8.double().reshape(Bq, N, H, dqk).permute(0, 2, 1, 3).expand(B, H, N, dqk)
    k = k8.double().reshape(B, M, H, dqk).permute(0, 2, 1, 3)
    c = score_scale(scale, q_descale, k_descale).to(dev)[None, :, None, None]
    t = (q @ k.transpose(-1, -2)) * c
    masked = torch.zeros(B, 1, N, M, dtype=torch.bool, device=dev)
    if pad_mask is not None:
        masked |= pad_mask.to(dev).bool()[:, None, None, :]
    if causal:
        shift = (m_total - N) - m_offset
        masked |= (torch.arange(M, device=dev)[None, :] > torch.arange(N, device=dev)[:, None] + shift)[None, None]
    t = t.masked_fill(masked, -FLT_MAX)
    live = torch.cat([(~masked).expand(B, H, N, M),
                      torch.zeros(B, H, N, Mt - M, dtype=torch.bool, device=dev)], dim=-1)
    t = torch.cat([t, torch.full((B, H, N, Mt - M), -math.inf, dtype=torch.float64, device=dev)], dim=-1)
    v8 = torch.zeros(B, H, Mt, dv, dtype=torch.float64, device=dev)
    v8[:, :, :M] = vt8[..., :M].double().transpose(-1, -2)
    vdesc = v_descale.double().to(dev)  # (H, dv)

    o = torch.zeros(B, H, N, dv, dtype=torch.float64, device=dev)
    m = torch.full((B, H, N), -math.inf, dtype=torch.float64, device=dev)
    l = torch.zeros(B, H, N, dtype=torch.float64, device=dev)
    pvh, flip = torch.zeros_like(o), torch.zeros_like(o)
    rho, rho_w = torch.zeros_like(l), torch.zeros_like(l)
    nadd = torch.full_like(l, 2.0)  # the quad reduction of the per-thread sums
    _, segs = _lib.debug_plan(B, H, N, M, workers=workers, rows_per_unit=128)
    for (_, b, h, q0, _, t0, t1, _) in segs:
        q1, nt = min(q0 + 128, N), t1 - t0
        x = t[b, h, q0:q1, t0 * 128:t1 * 128].reshape(q1 - q0, nt, 128)
        lv = live[b, h, q0:q1, t0 * 128:t1 * 128].reshape(q1 - q0, nt, 128)
        tile_max = x.amax(dim=-1)
        m_run = torch.cummax(tile_max, dim=1).values  # running maximum after each tile
        mref = torch.where(m_run == -math.inf, torch.zeros_like(m_run), m_run)
        if mutant == "tile_max":
            pref = torch.where(tile_max == -math.inf, torch.zeros_like(tile_max), tile_max)
        elif mutant == "final_max":
            pref = mref[:, -1:].expand_as(mref)
        else:
            pref = mref
        p = torch.exp2(x - pref[..., None])
        w = torch.exp2(pref - mref[:, -1:])  # rescale of each tile's terms to the segment's final reference
        seg_l = (p.sum(dim=-1) * w).sum(dim=1)
        y = p * 256.0
        pr = _round_e4m3(p) if mutant == "no_prescale" else _round_e4m3(y) / 256.0
        vt = v8[b, h, t0 * 128:t1 * 128].reshape(nt, 128, dv)
        seg_o = (torch.einsum("rtk,tkc->rtc", pr, vt) * w[..., None]).sum(dim=1)
        # exponent error (log2 units) of a live probability: the fp32 row maximum, the fp32 s * c of a row that holds a
        # masked key in the tile, the fp32 fmaf(s, c, -m); masked and past-M probabilities are exactly 0 or 1
        mfin = torch.where(mref <= -FLT_MAX, torch.zeros_like(mref), mref)
        arg = torch.where(lv, x - mref[..., None], torch.zeros_like(x))
        xs = torch.where(lv, x, torch.zeros_like(x))
        rel = torch.where(lv, torch.expm1(math.log(2.0) * U32 * (mfin.abs()[..., None] + xs.abs() + arg.abs()))
                          + EX2_REL, torch.zeros_like(x))
        r0 = _round_e4m3(y)
        step = torch.maximum((_round_e4m3(y * (1.0 + rel)) - r0).abs(), (_round_e4m3(y * (1.0 - rel)) - r0).abs())
        va = vt.abs()
        seg_pvh = (torch.einsum("rtk,tkc->rtc", pr, va) * w[..., None]).sum(dim=1)
        seg_flip = (torch.einsum("rtk,tkc->rtc", step / 256.0, va) * w[..., None]).sum(dim=1)
        # a rescale factor per tile and one merge weight per segment: ex2 of a difference of two fp32 maxima, a multiply
        mabs = mfin.abs().amax(dim=1)
        seg_rho_w = (nt + 1) * (math.log(2.0) * 3 * U32 * mabs + EX2_REL + 2 * U32)
        seg_m = mref[:, -1]
        m_old = m[b, h, q0:q1]
        m_new = torch.maximum(m_old, seg_m)
        a_old, a_seg = torch.exp2(m_old - m_new), torch.exp2(seg_m - m_new)
        o[b, h, q0:q1] = o[b, h, q0:q1] * a_old[:, None] + seg_o * a_seg[:, None]
        pvh[b, h, q0:q1] = pvh[b, h, q0:q1] * a_old[:, None] + seg_pvh * a_seg[:, None]
        flip[b, h, q0:q1] = flip[b, h, q0:q1] * a_old[:, None] + seg_flip * a_seg[:, None]
        l[b, h, q0:q1] = l[b, h, q0:q1] * a_old + seg_l * a_seg
        m[b, h, q0:q1] = m_new
        rho[b, h, q0:q1] = torch.maximum(rho[b, h, q0:q1], rel.amax(dim=(1, 2)))
        rho_w[b, h, q0:q1] += seg_rho_w
        # per tile: a pair sum, a chain of 8, the two chains, the running sum and its rescale; per segment a merge
        nadd[b, h, q0:q1] += 12 + 2 * nt
    vd = vdesc[None, :, None, :]
    o = o * vd  # the kernel's epilogue: v_descale of the channel (2^-8 is in the rounded probabilities)
    pe = torch.softmax(t[..., :M] / LOG2E, dim=-1) if M else None
    vdeq = v8[:, :, :M] * vd
    pv_abs = pe @ vdeq.abs()
    return {"o": o, "m": m, "l": l, "out": o / l[..., None], "pv_abs": pv_abs, "pv_hat": pvh * vd / l[..., None],
            "flip": flip * vd / l[..., None], "rho": rho, "rho_w": rho_w, "nadd": nadd}
