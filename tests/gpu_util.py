"""Helpers shared by the -m gpu parity tests: the oracle is evaluated in fp64 on the SAME bf16-rounded
operands the kernel sees; tolerance is stated relative to the largest reference magnitude."""
import math
from typing import NamedTuple

import numpy as np
import torch

from oracle import mha_oracle as O


def bf16_round(t):
    return t.to(torch.bfloat16).to(torch.float64)


def oracle_core(q, k, v, H, scale, pad=None, causal=False):
    """q (Bq,N,H*d), k (B,M,H*d), v (B,M,H*dv) bf16/any on any device -> (B,N,H*dv) fp64 CPU."""
    qc, kc, vc = (t.detach().cpu().to(torch.float64) for t in (q, k, v))
    B = kc.shape[0]
    qh = O.split_heads(qc.expand(B, -1, -1), H)
    out = O.core_attention(qh, O.split_heads(kc, H), O.split_heads(vc, H), scale,
                           None if pad is None else pad.cpu(), causal)
    return O.merge_heads(out)


def assert_close(got, ref, rel, what=""):
    """max |got-ref| <= rel * max|ref|   (rel: 1e-2 for bf16-operand tensor-core paths: P and the output
    are rounded to bf16 = 2^-9 relative each; 6e-3 for the fp32-math SIMT path: output rounding only)."""
    got = got.detach().double().cpu()
    ref = ref.detach().double().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{what}: non-finite values in kernel output"
    err = (got - ref).abs().max().item()
    bound = rel * max(ref.abs().max().item(), 1e-6)
    assert err <= bound, f"{what}: max err {err:.3e} > {bound:.3e}"
    return err


# --------------------------------------------------------------------------------------------------
# The stated parity gate (BASELINE.md §3, SURVEY.md §8(d)):
#     max|kernel - ref_fp64|  <=  2 * max|ref_bf16_eager - ref_fp64|  +  1e-3 * max|ref_fp64|
# ref_fp64 is the reference algorithm in float64 on the SAME bf16-rounded operands; ref_bf16_eager is
# what the reference's own eager code gives when run in bf16 (q*scale, einsum, masked_fill, softmax, einsum, each
# rounding to bf16 — modules.py:123-167).  Both are evaluated with plain torch ops on the device, so the gate
# is DERIVED per case instead of being a hard-coded relative tolerance.
# --------------------------------------------------------------------------------------------------
def torch_core(q, k, v, H, scale, pad=None, causal=False, dtype=torch.float64):
    """Reference algorithm (modules.py:123-167) with torch ops on q's device in `dtype`.
    q (Bq,N,H*d), k (B,M,H*d), v (B,M,H*dv) -> (B,N,H*dv) in `dtype`."""
    B, M = k.shape[0], k.shape[1]
    N = q.shape[1]
    qh = q.to(dtype).expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = k.to(dtype).reshape(B, M, H, -1).transpose(1, 2)
    vh = v.to(dtype).reshape(B, M, H, -1).transpose(1, 2)
    qh = qh * scale                                                      # :124
    attn = torch.einsum("bhic,bhjc->bhij", qh, kh)                       # :151
    neg = -torch.finfo(attn.dtype).max                                   # :152
    if pad is not None:
        attn.masked_fill_(pad.to(q.device).bool()[:, None, None, :], neg)    # :154-155
    if causal:
        cm = torch.ones(N, M, device=q.device, dtype=torch.bool).triu(M - N + 1)  # :135-140
        attn.masked_fill_(cm, neg)                                       # :157-158
    attn = attn.softmax(dim=-1)                                          # :160
    o = torch.einsum("bhij,bhjc->bhic", attn, vh)                        # :163
    return o.transpose(1, 2).reshape(B, N, -1)                           # :166-167


def derived_bound(ref64, eager):
    """(bound, eager_err, ref_max) of the stated gate for one case."""
    ref64 = ref64.double()
    eager_err = (eager.double().to(ref64.device) - ref64).abs().max().item()
    ref_max = ref64.abs().max().item()
    return 2.0 * eager_err + 1e-3 * max(ref_max, 1e-30), eager_err, ref_max


def assert_parity(got, q, k, v, H, scale, pad=None, causal=False, what="", eager_dtype=None, floor=0.0, per_row=False):
    """Check `got` against the fp64 reference with the DERIVED gate; returns (err, bound, eager_err).

    `floor`: lower limit of the bound for paths that add roundings the eager reference does not have (stated by
    the caller where used).  `per_row`: also apply the gate to every (b, h, n) row on its own (assert_rows)."""
    eager_dtype = q.dtype if eager_dtype is None else eager_dtype
    ref = torch_core(q, k, v, H, scale, pad, causal, torch.float64)
    eager = torch_core(q, k, v, H, scale, pad, causal, eager_dtype)
    bound, eager_err, ref_max = derived_bound(ref, eager)
    bound = max(bound, floor * ref_max)
    g = got.detach().double().to(ref.device)
    assert g.shape == ref.shape, (g.shape, ref.shape)
    assert torch.isfinite(g).all(), f"{what}: non-finite values in kernel output"
    err = (g - ref).abs().max().item()
    print(f"[parity] {what}: err {err:.3e}  bound {bound:.3e} (= 2 x eager {eager_err:.3e} + 1e-3 x max|ref| {ref_max:.3e})")
    assert err <= bound, f"{what}: max err {err:.3e} > derived bound {bound:.3e} (eager bf16 err {eager_err:.3e}, max|ref| {ref_max:.3e})"
    if per_row:
        assert_rows(g, ref, eager, H, what, floor)
    return err, bound, eager_err


def assert_rows(got, ref, eager, H, what="", floor=0.0):
    """The derived gate applied to every (b, h, n) output row separately:

        max_c |got - ref|  <=  max(2 * max_c |eager - ref| + 1e-3 * max_c |ref|,  floor * max_c |ref|)

    got / ref / eager are (B, N, H*dv).  One wrong key on one row moves that row by about |v| / (live keys); the
    whole-tensor gate is set by the largest rows of the case and does not see it.  Prints the worst ratio of error to
    bound and returns it."""
    B, N = ref.shape[0], ref.shape[1]
    r = ref.double().reshape(B, N, H, -1)
    g = got.double().to(r.device).reshape(B, N, H, -1)
    e = eager.double().to(r.device).reshape(B, N, H, -1)
    err = (g - r).abs().amax(-1)
    rmax = r.abs().amax(-1)
    bound = torch.maximum(2.0 * (e - r).abs().amax(-1) + 1e-3 * rmax, floor * rmax).clamp_min(1e-30)
    ratio = err / bound
    worst = ratio.argmax().item()
    b, n, h = worst // (N * H), (worst // H) % N, worst % H
    bad = int((ratio > 1).sum().item())
    print(f"[parity rows] {what}: worst err/bound {ratio.max().item():.3f} at (b={b}, h={h}, n={n}): "
          f"err {err[b, n, h].item():.3e} bound {bound[b, n, h].item():.3e} max|ref| {rmax[b, n, h].item():.3e}")
    assert bad == 0, (f"{what}: {bad} of {ratio.numel()} rows over their derived bound; worst (b={b}, h={h}, n={n}) "
                      f"err {err[b, n, h].item():.3e} > {bound[b, n, h].item():.3e}")
    return ratio.max().item()


# --------------------------------------------------------------------------------------------------
# The gradient gate of the attention backward tests.  Gradient rows differ in size by orders of magnitude (a padded
# key's dK row is 0, a key only late queries see has a small dK, a peaked row a small dQ), so a gate set by max|ref|
# does not see a wrong row of a small gradient.  assert_grads adds an element-wise gate scaled by the fp64 reference of
# the same gradient on magnitudes (grad_magnitudes).
#
# KAPPA, from the rounding points of the backward kernels (csrc/pcv_attn_bwd.cu), u = the 16-bit unit roundoff:
#   - P (times keep / (1 - p) under dropout) is rounded to 16 bits before P^T dO:         dV error  u * dV_abs;
#   - dS is rounded to 16 bits before dS^T Q and dS K:                                    dK, dQ    u * dK_abs, u * dQ_abs;
#   - delta = rowsum(dO * O) reads the 16-bit forward output, which carries the forward's own P rounding and its output
#     rounding, |O - O*| <= 2u sum_j p|v|; so |delta - delta*| <= 2u rowsum(P A) and dS moves by 2u P rowsum(P A),
#     which dS_abs holds:                                                                 dK, dQ    2u * abs;
#   - the gradient is rounded to 16 bits on output:                                       all       u * abs.
# That is 2u for dV and 4u for dK / dQ.  The rest is fp32 (the scores, ex2 of the fp32 statistics, the accumulations)
# and far below u.  KAPPA = 8 is twice the largest sum; the CPU emulation of this arithmetic (test_bwd_variants_cpu.py)
# stays at or below half of the bound it sets.  The backward shim (head dims above 192) keeps P and dS in fp32 and
# has only the delta and output terms.
#
# fp16 has subnormals below 2^-14 with spacing 2^-24: a rounded P or dS element there is off by up to 2^-24 whatever
# its size, so the gate adds 2^-24 times the sum of the magnitudes each such element multiplies (GradMagnitude.sub),
# plus one spacing for the output.  bf16 has the exponent range of fp32: its only absolute error is ex2's flush below
# 2^-126, which the same term with 2^-126 covers.
# --------------------------------------------------------------------------------------------------
KAPPA = 8.0
UNIT_ROUNDOFF = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
ABS_SPACING = {torch.bfloat16: 2.0 ** -126, torch.float16: 2.0 ** -24}
GRAD_FLOOR = 6e-3  # of max|ref|, the whole-tensor gate's floor: two 2^-9 roundings (P / dS, then the gradient)


class GradMagnitude(NamedTuple):
    """The element-wise scale of one gradient: `abs`, the fp64 gradient evaluated on magnitudes, and `sub`, the sum of
    magnitudes that multiplies one absolute spacing per rounded P / dS element (plus 1 for the output)."""
    abs: torch.Tensor
    sub: torch.Tensor


def grad_magnitudes(q, k, v, go, H, scale, pad=None, causal=False, keep=None, rp=1.0):
    """(dq, dk, dv) GradMagnitude of the attention backward, fp64 on q's device; shapes those of the gradients.

    With A = |dO| |V|^T and P the fp64 probabilities (P_d = P * keep * rp under dropout):
        dS_abs = P * (A_d + rowsum(P_d * A))   (0 where the score is filled; the second term bounds delta)
        dV_abs = P_d^T |dO|      dK_abs = scale * dS_abs^T |Q|      dQ_abs = scale * dS_abs |K| (summed over the batch
    for a batch-1 q).  `sub` takes 1 for each P / dS element and P * rowsum(A) for the forward's P inside delta."""
    f64 = torch.float64
    dev = q.device
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    qh = q.detach().to(f64).expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2).abs()
    kh = k.detach().to(f64).reshape(B, M, H, -1).transpose(1, 2)
    vh = v.detach().to(f64).reshape(B, M, H, -1).transpose(1, 2).abs()
    gh = go.detach().to(dev, f64).reshape(B, N, H, -1).transpose(1, 2).abs()
    s = (q.detach().to(f64).expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2) * scale) @ kh.transpose(-1, -2)
    filled = torch.zeros(B, 1, N, M, dtype=torch.bool, device=dev)
    if pad is not None:
        filled = filled | pad.to(dev).bool()[:, None, None, :]
    if causal:
        filled = filled | torch.ones(N, M, dtype=torch.bool, device=dev).triu(M - N + 1)
    P = s.masked_fill(filled, -torch.finfo(f64).max).softmax(-1)
    del s
    kr = None if keep is None else keep.to(dev, f64) * rp
    Pd = P if kr is None else P * kr
    A = gh @ vh.transpose(-1, -2)
    ds = P * ((A if kr is None else A * kr) + (Pd * A).sum(-1, keepdim=True))
    ds = ds.masked_fill(filled, 0.0)
    ds_sub = P * A.sum(-1, keepdim=True) + 1.0
    del A
    kh = kh.abs()
    dq = (scale * ds @ kh, scale * ds_sub @ kh + 1.0)
    dk = (scale * ds.transpose(-1, -2) @ qh, scale * ds_sub.transpose(-1, -2) @ qh + 1.0)
    dv = (Pd.transpose(-1, -2) @ gh, (gh.sum(-2, keepdim=True) + 1.0).expand(B, H, M, gh.shape[-1]))

    def merge(t, L):
        return t.transpose(1, 2).reshape(B, L, -1)

    dq = [merge(t, N) for t in dq]
    if q.shape[0] == 1 and B > 1:
        dq = [t.sum(0, keepdim=True) for t in dq]
    return (GradMagnitude(*dq), GradMagnitude(*(merge(t, M) for t in dk)), GradMagnitude(*(merge(t, M) for t in dv)))


def element_bound(absref, dtype):
    """The element-wise bound of assert_grads: KAPPA * u * absref.abs + spacing * absref.sub."""
    return KAPPA * UNIT_ROUNDOFF[dtype] * absref.abs + ABS_SPACING[dtype] * absref.sub


def assert_grads(got, ref64, eager, absref, dtype, what="", whole=True):
    """One gradient of the attention backward against its fp64 reference, with two gates:

      - the whole-tensor derived gate: max|got - ref| <= max(2 max|eager - ref| + 1e-3 max|ref|, GRAD_FLOOR max|ref|),
        eager being 16-bit autograd of the reference algorithm (its bound is the floor alone if eager overflowed).
        `whole=False` leaves it out: with at most two keys per row the gradients are small by cancellation (the dS of
        a row sum to 0), and the CPU emulation of the kernels' arithmetic already exceeds this gate there
        (test_bwd_variants_cpu.py), so eager's error is no yardstick;
      - the element-wise gate: |got - ref| <= KAPPA * u * absref.abs + spacing * absref.sub (see KAPPA).

    Prints the whole-tensor error and the worst element's err / bound; returns that worst ratio."""
    r = ref64.detach().double()
    g = got.detach().double().to(r.device)
    assert g.shape == r.shape, (what, g.shape, r.shape)
    assert torch.isfinite(g).all(), f"{what}: non-finite values in the gradient"
    bound, eager_err, ref_max = derived_bound(r, eager)
    if not math.isfinite(bound):
        bound = 0.0
    bound = max(bound, GRAD_FLOOR * ref_max)
    diff = (g - r).abs()
    err = diff.max().item()
    assert not whole or err <= bound, (f"{what}: max err {err:.3e} > whole-tensor bound {bound:.3e} (eager {eager_err:.3e}, "
                          f"max|ref| {ref_max:.3e})")
    eb = element_bound(absref, dtype).to(r.device)
    ratio = diff / eb
    flat = int(ratio.argmax().item())
    idx = tuple(int(i) for i in np.unravel_index(flat, tuple(ratio.shape)))
    worst = ratio[idx].item()
    bad = int((ratio > 1).sum().item())
    print(f"[grad elems] {what}: err {err:.3e} {'<=' if whole else 'whole-tensor gate off,'} {bound:.3e}; worst err/bound {worst:.3f} at {idx}: err "
          f"{diff[idx].item():.3e} bound {eb[idx].item():.3e} ref {r[idx].item():.3e} abs {absref.abs[idx].item():.3e}")
    assert bad == 0, (f"{what}: {bad} of {ratio.numel()} elements over their bound; worst at {idx} (b, row, channel): "
                      f"got {g[idx].item():.6e} ref {r[idx].item():.6e} bound {eb[idx].item():.3e}")
    return worst


def assert_grad_set(got, ref64, eager, mags, dtype, what="", whole=True):
    """assert_grads on (dq, dk, dv); returns {name: worst err / bound}."""
    return {name: assert_grads(g_, r_, e_, m_, dtype, f"{what} {name}", whole)
            for name, g_, r_, e_, m_ in zip(("dq", "dk", "dv"), got, ref64, eager, mags)}


FLT_MAX = torch.finfo(torch.float32).max


# --------------------------------------------------------------------------------------------------
# The element-wise gate of the streaming decode kernel (csrc/pcv_attn_decode.cu).  The kernel keeps P in fp32: its one
# 16-bit rounding is the output, so the derived gate (twice eager's error, which rounds P to 16 bits) is far wider than
# the kernel's own error, and a missing or leaked key in a long row fits inside it.  decode_element_bound follows the
# kernel's rounding points instead, u = the 16-bit unit roundoff, u32 = 2^-24:
#   - the output is rounded to 16 bits once:                                              u |o|
#   - the scores: q is scaled by scale * log2e (and k_descale for e4m3 rows), then dqk products are summed in fp32
#     (fma chains of 8 / 16 channels and a shuffle tree over the lanes): |dt_j| <= (dqk + 8) u32 A_j with
#     A_j = scale * log2e * sum_c |q_c k_c|.  A score error moves p_j by ln2 (dt_j - sum_k p_k dt_k) relative, so o moves by
#     at most ln2 (dqk + 8) u32 (sum_j p_j A_j |v_j| + (sum_j p_j A_j) (sum_j p_j |v_j|));
#   - ex2 (2 ulp = 2^-22 relative) and the fp32 accumulation of p and p v: each term passes through at most `depth`
#     roundings and ex2 factors (the keys and block rescales of one lane group, the lane-group shuffle tree, the warps
#     and the splits; decode_variants.serial_depth), on the numerator and the denominator alike:
#     2 depth (u32 + 2^-22) sum_j p_j |v_j|;
#   - fp16 outputs below 2^-14 are subnormal: one absolute spacing 2^-24.
# The bound is twice the sum of the relative terms plus the spacing.  The factor 2 is what lets the kernel's fp32 error
# use the space the output rounding leaves: |RN(x) - ref| <= u |ref| + (1 + u) |x - ref|.  The CPU emulation of the
# kernel's arithmetic in its split and lane-group order (test_decode_variants_cpu.py) stays at or below half of it.
# --------------------------------------------------------------------------------------------------
EX2_ULP = 2.0 ** -22


def decode_element_bound(q, k, v, H, scale, pad, causal, dtype, depth, ref=None):
    """(bound, ref) of the decode kernel's element-wise gate (see above), fp64 on k's device, (B, N, H*dv).  q (Bq, N,
    H*dqk), k (B, M, H*dqk), v (B, M, H*dv) are the operands the kernel computes on (e4m3 rows dequantised); `depth` the
    longest chain of fp32 roundings a probability passes through."""
    f64, dev = torch.float64, k.device
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    qh = q.detach().to(dev, f64).expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = k.detach().to(f64).reshape(B, M, H, -1).transpose(1, 2)
    vh = v.detach().to(dev, f64).reshape(B, M, H, -1).transpose(1, 2)
    dqk = qh.shape[-1]
    if ref is None:
        ref = torch_core(q.to(dev), k, v.to(dev), H, scale, pad, causal, f64)
    s = (qh * scale) @ kh.transpose(-1, -2)
    filled = torch.zeros(B, 1, N, M, dtype=torch.bool, device=dev)
    if pad is not None:
        filled = filled | pad.to(dev).bool()[:, None, None, :]
    if causal:
        filled = filled | torch.ones(N, M, dtype=torch.bool, device=dev).triu(M - N + 1)
    P = s.masked_fill(filled, -torch.finfo(f64).max).softmax(-1)
    A = (qh.abs() * (scale * 1.4426950408889634)) @ kh.abs().transpose(-1, -2)
    va = vh.abs()
    pv = P @ va
    pa = P * A
    score = math.log(2.0) * (dqk + 8) * 2.0 ** -24 * (pa @ va + pa.sum(-1, keepdim=True) * pv)
    accum = 2.0 * depth * (2.0 ** -24 + EX2_ULP) * pv
    e32 = (score + accum).transpose(1, 2).reshape(B, N, -1)
    u = UNIT_ROUNDOFF[dtype]
    sp = 2.0 ** -24 if dtype == torch.float16 else 0.0
    return 2.0 * (u * ref.abs() + e32) + sp, ref


def assert_decode_elements(got, q, k, v, H, scale, pad, causal, dtype, depth, what=""):
    """The decode kernel's output against fp64 attention on the same operands: the derived gate row by row
    (assert_parity(per_row=True)) and the element-wise gate of decode_element_bound.  Returns the worst element's
    err / bound."""
    # the row gate's floor is the one output rounding: on a row of few keys eager's error can be smaller by chance
    assert_parity(got, q, k, v, H, scale, pad, causal, what=what, eager_dtype=dtype, per_row=True,
                  floor=UNIT_ROUNDOFF[dtype])
    bound, ref = decode_element_bound(q, k, v, H, scale, pad, causal, dtype, depth)
    g = got.detach().double().to(ref.device)
    ratio = (g - ref).abs() / bound
    flat = int(ratio.argmax().item())
    idx = tuple(int(i) for i in np.unravel_index(flat, tuple(ratio.shape)))
    worst = ratio[idx].item()
    bad = int((ratio > 1).sum().item())
    print(f"[decode elems] {what}: worst err/bound {worst:.3f} at {idx}: got {g[idx].item():.6e} ref {ref[idx].item():.6e} "
          f"bound {bound[idx].item():.3e}")
    assert bad == 0, f"{what}: {bad} of {ratio.numel()} elements over their bound; worst at {idx}"
    return worst


def assert_partial_state(part, q, k, v, H, scale, pad=None, causal=False, m_total=None, m_offset=0, what=""):
    """attention_partial's (o, m, l) against oracle.mha_oracle.partial_state, evaluated in fp64 on the device on the
    same operands (log2 domain: m = row max of the scaled scores, l = sum 2^(t - m), o = sum 2^(t - m) v).

    - m: the kernel keeps the exact running max, so it is the oracle's up to the fp32 score rounding (abs 4e-3);
    - l: relative 2e-3 (ex2.approx and fp32 sums; a max off by 4e-3 would alone move l by 0.3 %);
    - o: elementwise within 2^-8 of sum p |v| (+ 1e-6 of it for the fp32 sums): the kernel rounds P to 16 bits before
      P V, and 2^-8 is the unit roundoff of bf16;
    - rows without a live key (the shard lies in the row's causal future, or the batch row is fully padded) follow the
      finite-fill semantics exactly: m = -FLT_MAX (the oracle's -DBL_MAX), l = the shard's key count, and o = the sum
      of the shard's V rows (fp32 accumulation: 2^-12 of sum |v|).  combine_partials weights such a shard by zero."""
    po_k, pm_k, pl_k = (t.detach().double() for t in part)
    dev = po_k.device
    B, M = k.shape[0], k.shape[1]
    qh = O.split_heads(q.detach().to(dev, torch.float64).expand(B, -1, -1), H)
    kh, vh = O.split_heads(k.detach().to(dev, torch.float64), H), O.split_heads(v.detach().to(dev, torch.float64), H)
    padd = None if pad is None else pad.to(dev)
    mt = M if m_total is None else m_total
    po, pm, pl = O.partial_state(qh, kh, vh, scale, padd, causal, mt, m_offset)
    pa = O.partial_state(qh, kh, vh.abs(), scale, padd, causal, mt, m_offset)[0]
    dead = pm == -torch.finfo(torch.float64).max
    live = ~dead
    assert torch.isfinite(po_k).all() and torch.isfinite(pl_k).all(), f"{what}: non-finite partial state"
    assert (pm_k[dead] == -FLT_MAX).all(), f"{what}: rows without a live key must have m = -FLT_MAX"
    l_dead = pl_k[dead]
    assert (l_dead == pl[dead]).all(), (f"{what}: rows without a live key must have l = {M} (one per masked key); got "
                                        f"{l_dead.min().item() if l_dead.numel() else None}..{l_dead.max().item() if l_dead.numel() else None}")
    o_dead_err = ((po_k - po).abs() - 2.0 ** -12 * pa)[dead]
    assert o_dead_err.numel() == 0 or o_dead_err.max().item() <= 0, f"{what}: o of rows without a live key != sum of V"
    m_err = (pm_k - pm)[live].abs().max().item() if live.any() else 0.0
    l_err = ((pl_k - pl).abs() / pl)[live].max().item() if live.any() else 0.0
    o_ratio = ((po_k - po).abs() / ((2.0 ** -8 + 1e-6) * pa).clamp_min(1e-30))[live].max().item() if live.any() else 0.0
    print(f"[partial] {what}: {int(dead.sum())} rows without a live key; live rows: |dm| {m_err:.2e}, "
          f"rel dl {l_err:.2e}, o err / (2^-8 sum p|v|) {o_ratio:.3f}")
    assert m_err <= 4e-3, f"{what}: row max off by {m_err:.3e} (log2 units)"
    assert l_err <= 2e-3, f"{what}: denominator off by {l_err:.3e} relative"
    assert o_ratio <= 1.0, f"{what}: numerator error {o_ratio:.3f} x 2^-8 sum p|v|"
    return int(dead.sum())


def torch_cross_attention(sd, x_q, x_kv, H, pad=None, dtype=torch.float64, device="cuda"):
    """CrossAttention.forward (reference modules.py:204-230 -> :113-170) restated with torch ops in `dtype` on
    `device` from a reference state_dict: the fp64 yardstick / the eager-bf16 yardstick of module-level cases."""
    import torch.nn.functional as F

    w = {k: v.to(device=device, dtype=dtype) for k, v in sd.items()}
    xq = x_q.to(device=device, dtype=dtype)
    xkv = x_kv.to(device=device, dtype=dtype)
    xq = F.layer_norm(xq, xq.shape[-1:], w["q_norm.weight"], w["q_norm.bias"], 1e-5)          # :220
    xkv = F.layer_norm(xkv, xkv.shape[-1:], w["kv_norm.weight"], w["kv_norm.bias"], 1e-5)     # :226
    a = "attention."
    q = F.linear(xq, w[a + "q_proj.weight"], w.get(a + "q_proj.bias"))                          # :113
    k = F.linear(xkv, w[a + "k_proj.weight"], w.get(a + "k_proj.bias"))                         # :114
    v = F.linear(xkv, w[a + "v_proj.weight"], w.get(a + "v_proj.bias"))                         # :115
    scale = (q.shape[-1] // H) ** -0.5                                                          # :73
    o = torch_core(q, k, v, H, scale, None if pad is None else pad.to(device), False, dtype)
    return F.linear(o, w[a + "o_proj.weight"], w.get(a + "o_proj.bias"))                        # :168


# --------------------------------------------------------------------------------------------------
# The element-wise gates of the LayerNorm-folded projection (csrc/pcv_kvproj.cu) and its backward (csrc/pcv_lnlin_bwd.cu).
# u = the output's unit roundoff (2^-8 bf16, 2^-11 fp16, 2^-4 e4m3), u32 = 2^-24.
#
# Producer, against the operand-exact reference rstd (x.w'^T - mean s) + t on the kernel's own w' (w_cat) and (s, t)
# (col_st), mean / rstd in fp64:
#   - the output is rounded once:                                                         u |ref|
#   - x.w' is C / 16 fp32 additions of exact k16 partial sums on the tensor core, and the epilogue adds four roundings
#     (mean s, the difference, rstd, + t):              (C / 16 + 16) u32 (rstd sum_c |x_c w'_c| + rstd mu_abs |s| + |t|)
#     mu_abs = mean |x| + |x_0| bounds the error of the mean, which sums |x| (two-pass) or |x - x_0| (in-kernel) in fp32;
#   - rstd's relative error scales rstd (x.w' - mean s) <= rstd (sum |x w'| + |mean| |s|): (C / 32 + 16) u32 for
#     pcv_ln_stats (a lane's serial sum, the shuffle tree, sqrt, divide); for the in-kernel one-pass statistics the C / 2
#     serial additions of each half row enter var + (mean - x_0)^2 and leave var, so their term is multiplied by
#     1 + ((mean - x_0) rstd)^2.
# The bound is 2 (u |ref| + E32) + one absolute spacing: |RN(y) - ref| <= u |ref| + (1 + u) |y - ref|.  The term
# rstd mu_abs |s| is the fold's cancellation: a row with |mean| >> std leaves x.w' - mean s to fp32 and multiplies what
# remains by rstd.  A zero-variance row is written as t exactly (pcv_kvproj.cu); a near-constant row keeps this term.
# Against module semantics (fp64 LayerNorm -> Linear on the 16-bit parameters) the fold's one rounding of gamma W adds
# u sum_c |x_hat_c| |gamma_c W_nc|: kernel error on one side, design error on the other.
# --------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24
E4M3_U = 2.0 ** -4


def proj_reference(x, w_cat, col_st, eps, fuse=False):
    """(ref, E32) of the producer: the operand-exact fp64 reference and the fp32 error term above (fp64, (rows, n)).
    eps None: no LayerNorm (out = x w^T + t)."""
    xd, wd = x.double(), w_cat.double().to(x.device)
    cs = col_st.double().to(x.device)
    s, t = cs[:, 0], cs[:, 1]
    C = xd.shape[1]
    xw = xd @ wd.T
    xwa = xd.abs() @ wd.abs().T
    if eps is None:
        return xw + t, (C / 16 + 16) * U32 * (xwa + t.abs())
    mean = xd.mean(1, keepdim=True)
    rstd = 1.0 / (xd.var(1, unbiased=False, keepdim=True) + eps).sqrt()
    ref = rstd * (xw - mean * s) + t
    mu_abs = xd.abs().mean(1, keepdim=True) + xd[:, :1].abs()
    e_gemm = (C / 16 + 16) * U32 * (rstd * xwa + rstd * mu_abs * s.abs() + t.abs())
    if fuse:
        rel = ((C / 2 + 8) / 2 * (1 + ((mean - xd[:, :1]) * rstd) ** 2) + 8) * U32
    else:
        rel = (C / 32 + 16) * U32
    return ref, e_gemm + rel * rstd * (xwa + mean.abs() * s.abs())


def _report(ratio, what, got, ref, bound, tag):
    flat = int(ratio.argmax().item())
    idx = tuple(int(i) for i in np.unravel_index(flat, tuple(ratio.shape)))
    worst = ratio[idx].item()
    bad = int((ratio > 1).sum().item())
    print(f"[{tag}] {what}: worst err/bound {worst:.3f} at {idx}: got {got[idx].item():.6e} ref {ref[idx].item():.6e} "
          f"bound {bound[idx].item():.3e}")
    assert bad == 0, (f"{what}: {bad} of {ratio.numel()} elements over their bound; worst at {idx}: got "
                      f"{got[idx].item():.6e} ref {ref[idx].item():.6e} bound {bound[idx].item():.3e}")
    return worst


def assert_proj_elements(got, ref, e32, dtype, what=""):
    """A 16-bit producer output against the operand-exact reference: |got - ref| <= 2 (u |ref| + E32) + spacing."""
    g = got.detach().double().to(ref.device)
    assert g.shape == ref.shape, (what, g.shape, ref.shape)
    assert torch.isfinite(g).all(), f"{what}: non-finite output"
    sp = 2.0 ** -24 if dtype == torch.float16 else 0.0
    bound = 2.0 * (UNIT_ROUNDOFF[dtype] * ref.abs() + e32) + sp
    return _report((g - ref).abs() / bound, what, g, ref, bound, "proj elems")


def assert_e4m3_codes(codes, ref, e32, inv_scale, what=""):
    """e4m3 producer codes against RN(ref * inv_scale): a code may differ from it only where a rounding midpoint lies
    within 2 E32 of ref, i.e. its value must lie between RN((ref - 2 E32) inv) and RN((ref + 2 E32) inv)."""
    f8 = torch.float8_e4m3fn
    inv = inv_scale.double().to(ref.device)
    q = lambda v: (v * inv).clamp(-448.0, 448.0).float().to(f8).view(torch.uint8)
    lo, hi, mid = q(ref - 2.0 * e32), q(ref + 2.0 * e32), q(ref)
    c = codes.detach().to(ref.device).view(torch.uint8)
    val = lambda u8: u8.view(f8).double()
    ok = (val(c) >= val(lo)) & (val(c) <= val(hi))
    exact = int((c == mid).sum().item())
    print(f"[e4m3 codes] {what}: {exact} of {c.numel()} codes equal RN(ref * inv); "
          f"{int((~ok).sum().item())} outside the midpoint band")
    if not bool(ok.all()):
        bad = (~ok).nonzero()[0].tolist()
        raise AssertionError(f"{what}: code {int(c[tuple(bad)])} at {bad} is neither RN of ref +- 2 E32 "
                             f"({int(lo[tuple(bad)])}, {int(hi[tuple(bad)])}); ref {ref[tuple(bad)].item():.6e}")
    return exact


def fold_term(x, gamma, w, eps, dtype):
    """u sum_c |x_hat_c| |gamma_c W_nc|: the one rounding of the folded weights gamma W (fp64, (rows, n))."""
    xd = x.double()
    xh = (xd - xd.mean(1, keepdim=True)) / (xd.var(1, unbiased=False, keepdim=True) + eps).sqrt()
    gw = (w.double() * gamma.double().to(w.device)[None, :]).abs()
    return UNIT_ROUNDOFF[dtype] * xh.abs() @ gw.to(xd.device).T


# --------------------------------------------------------------------------------------------------
# The backward's element-wise gate.  With x_hat rebuilt in fp32 from x and the statistics, its 16-bit rounding points
# (pcv_lnlin_bwd.cu) are: dx_hat = gamma dy is written to grad_x in 16 bits before the fixup reads it back; x_hat is
# rounded to 16 bits before the dW GEMM; every output is rounded once.  So dx and dW carry 2u of their magnitude
# gradient, db / dgamma / dbeta 1u.  The fp32 sums add `depth` u32 each: dx (n / 16 tensor-core adds, the column-tile
# partials, the fixup), dW (the rows of a split on the tensor core, the splits, the rank-1 term), db (a thread's serial
# sum over the rows of a split, the splits), dgamma / dbeta (two rows per thread, the shuffle tree, 8 warps, the row
# blocks of a range, the ranges).  The magnitudes are the closed-form gradient on |G|, |W|, |x_hat|, |gamma|, |beta|:
#   dy_a = |G| |W|, dxh_a = |gamma| dy_a, dx_a = rstd (dxh_a + (sum dxh_a + |x_hat| sum dxh_a |x_hat|) / C),
#   dW_a = (|x_hat|^T |G|) |gamma| + db_a |beta|, db_a = sum |G|, dgamma_a = sum dy_a |x_hat|, dbeta_a = sum dy_a.
# The bound is 2 (rounds u + depth u32) abs + spacing (fp16: 2^-24 times (1 + 2 rstd) for dx, whose dx_hat may be
# subnormal).
# --------------------------------------------------------------------------------------------------
def lnlin_magnitudes(x, stats, w, gamma, beta, G):
    """(dx, dW, db, dgamma, dbeta) magnitudes and (rstd) of the backward, fp64 on x's device."""
    xd = x.double()
    st = stats.double()
    rstd = st[:, 1:2]
    xh = ((xd - st[:, :1]) * rstd).abs()
    C = xd.shape[1]
    g = torch.ones(C, dtype=torch.float64, device=xd.device) if gamma is None else gamma.double().abs()
    b = torch.zeros(C, dtype=torch.float64, device=xd.device) if beta is None else beta.double().abs()
    Ga, Wa = G.double().abs(), w.double().abs()
    dy = Ga @ Wa
    dxh = dy * g
    dx = rstd * (dxh + (dxh.sum(1, keepdim=True) + xh * (dxh * xh).sum(1, keepdim=True)) / C)
    db = Ga.sum(0)
    dW = (xh.T @ Ga).T * g[None, :] + db[:, None] * b[None, :]
    return (dx, dW, db, (dy * xh).sum(0), dy.sum(0)), rstd


def lnlin_element_bounds(mags, rstd, dtype, rows, C, n, splits, m_blocks):
    u = UNIT_ROUNDOFF[dtype]
    rps = -(-rows // splits)
    depth = (n / 16 + C / 128 + 8, rps / 16 + splits + 8, rps / 2 + splits + 4, 16 + m_blocks / 8 + 8,
             16 + m_blocks / 8 + 8)
    rounds = (2, 2, 1, 1, 1)
    sp = 2.0 ** -24 if dtype == torch.float16 else 0.0
    out = []
    for i, (m, d, r) in enumerate(zip(mags, depth, rounds)):
        extra = sp * (1 + 2 * rstd) if i == 0 else sp
        out.append(2.0 * (r * u + d * U32) * m + extra)
    return out


def assert_lnlin_elements(got, ref, bounds, names, what=""):
    """Each requested backward output against fp64 autograd under its element bound; returns {name: worst}."""
    out = {}
    for name, g_, r_, b_ in zip(names, got, ref, bounds):
        if g_ is None:
            continue
        g = g_.detach().double().to(r_.device)
        assert g.shape == r_.shape, (what, name, g.shape, r_.shape)
        assert torch.isfinite(g).all(), f"{what} {name}: non-finite"
        out[name] = _report((g - r_.double()).abs() / b_, f"{what} {name}", g, r_.double(), b_, "lnlin elems")
    return out
