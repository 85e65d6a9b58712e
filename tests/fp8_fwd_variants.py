"""Variant matrix, schedule shapes, operand builders, exact probes and the per-element gate of the FP8 tensor-core
attention forward (ops.attention_fp8 -> launch_attn_tc_fp8 -> attn_fwd_fp8_kernel<NQB, NVB, BF16> in
perceiver_io_b200/csrc/pcv_attn_tc.cu, plus tc_combine_kernel when the plan splits), shared by its GPU test
(test_gpu_fp8_variants.py) and its CPU companion (test_fp8_variants_cpu.py).  Nothing here needs a GPU.

The dispatch, restated (launch_attn_tc_fp8 / launch_dispatch_fp8):
  - NQB = ceil(dqk / 128) Q / K boxes of 128 e4m3 channels (1..2);
  - V^T runs in passes of at most 128 channels (kMaxDvPass), each with NVB = ceil(dv_pass / 64) (1..2);
  - bf16 or fp16 output.
The ring (attn_fwd_body with FP8 = true): a key tile streams NQB K boxes and one V^T box (KVB = 1, 128 keys x 128
channels, the NVB 64-channel halves at byte offset 8192 v) through FwdCfg<NQB, NVB>::kSlots 16 KB slots."""
import itertools
import math

import torch

from fp8_emulation import score_scale
from fwd_variants import BF16, DTYPES, FP16, MAX_DV_PASS, SCHEDULE_SHAPES, TILE, check_schedule, nvb_passes  # noqa: F401

E4M3_CH = 128        # e4m3 channels per Q / K box
BOX_BYTES = 16384
SMEM_LIMIT = 227 * 1024
FLT_MAX = torch.finfo(torch.float32).max


def nqb8(dqk):
    """launch_attn_tc_fp8: nqb = (dqk + 127) / 128."""
    return (dqk + E4M3_CH - 1) // E4M3_CH


def variants_of(dqk, dv, dtype):
    """The (NQB, NVB, dtype) instantiations of attn_fwd_fp8_kernel one call launches."""
    return {(nqb8(dqk), nvb, dtype) for nvb in nvb_passes(dv)}


def reachable_variants():
    """Every instantiation the dispatch can reach: head dims in multiples of 16 (attn_tc_fp8_supported), dqk <= 256,
    dv <= 512."""
    out = set()
    for dqk, dv in itertools.product(range(16, 257, 16), range(16, 513, 16)):
        for dt in DTYPES:
            out |= variants_of(dqk, dv, dt)
    return out


def ring_slots(nqb, nvb):
    """FwdCfg<NQB, NVB>::kSlots: kFit = min(16, (kSmemLimit - NQB * kBoxBytes - 2048) / kBoxBytes) slots, rounded down
    to a multiple of NQB + NVB (the 16-bit kernel's boxes per tile, which the FP8 kernel shares the config of)."""
    fit = min(16, (SMEM_LIMIT - nqb * BOX_BYTES - 2048) // BOX_BYTES)
    return fit // (nqb + nvb) * (nqb + nvb)


def boxes_per_tile(nqb):
    """NQB K boxes + KVB = 1 V^T box: the pipelined schedule needs kSlots % (NQB + 1) == 0 (static_assert)."""
    return nqb + 1


def case_id(case):
    dqk, dv, dt = case
    return f"{dt}-qk{dqk}-v{dv}"


# ---- section 1: every instantiation, from head dims that are not multiples of 128 / 64 (zero-filled box tails) ----
# (dqk, dv, dtype).  qk 48 / 112 give NQB 1, 144 / 208 / 256 NQB 2; v 48 NVB 1, 112 NVB 2; v 176 runs an NVB 2 and an
# NVB 1 pass in one call, v 304 two NVB 2 passes and an NVB 1 pass, v 512 four NVB 2 passes.
VARIANT_CASES = [(dqk, dv, dt) for dt in DTYPES
                 for dqk, dv in ((48, 48), (112, 176), (144, 112), (208, 304), (256, 512))]
# B, N, M, H of section 1: 12 (b, h, query tile) units of 35 key tiles over 132 CTAs, so segments hold 3..4 tiles (the
# in-loop path, rescales of O) and split units merge in tc_combine_kernel; the last key tile is ragged.
SEC1 = (3, 200, 4400, 2)
# std of the live scores in log2 units: most probabilities fall below e4m3's normal range at 2^8 P, and a few keys
# dominate each row, so that rounding P against another maximum moves a row by more than the accumulation error
SEC1_SPREAD = 6.0

# ---- section 2: schedule shapes (fwd_variants.SCHEDULE_SHAPES), one case per (NQB, NVB), both output dtypes ----
SCHEDULE_CASES = [(112, 48, BF16), (48, 112, FP16), (208, 48, FP16), (144, 112, BF16)]

# ---- section 3: causal diagonal sweep (fwd_variants.DIAG_*) ----
DIAG_CASES = [(48, 112, BF16), (144, 48, FP16)]


def check_schedule8(shape_name, case, workers):
    """fwd_variants.check_schedule with the single-CTA plan and the FP8 ring: "ring" streams at least twice kSlots
    boxes through one segment."""
    dqk, dv, dt = case
    nq = nqb8(dqk)
    slots = ring_slots(nq, min(nvb_passes(dv)))
    return check_schedule(shape_name, (dqk, dv, dt, False), workers, boxes_per_tile=boxes_per_tile(nq), slots=slots)


def tiles_per_segment(B, H, N, M, workers):
    """(min, max, mean) key tiles per segment of the single-CTA plan."""
    from perceiver_io_b200 import _lib

    _, segs = _lib.debug_plan(B, H, N, M, workers=workers, rows_per_unit=TILE)
    n = [t1 - t0 for *_, t0, t1, _s in segs]
    return min(n), max(n), sum(n) / len(n)


# --------------------------------------------------------------------------------------------------
# operands (built on the CPU generator, then moved to `device`)
# --------------------------------------------------------------------------------------------------
def v_descale(H, dv):
    """(H, dv) powers of two, 2^-((5 c + 3 h) mod 11): channel c + 1, channel c - 128 (the previous pass) and head h + 1
    all differ by a factor of at least 2."""
    c = torch.arange(dv)[None, :]
    h = torch.arange(H)[:, None]
    return torch.exp2(-((5 * c + 3 * h) % 11).float())


def _to_f8(x, device):
    return x.float().to(torch.float8_e4m3fn).to(device)


def random_operands(B, N, M, H, dqk, dv, seed, Bq=None, poison=None, device="cuda", spread=SEC1_SPREAD):
    """(q8, k8, vt8, qd, kd, vd) with scores the tensor cores compute exactly: q / k codes are integers in [-4, 4], so
    every partial sum of q8 . k8 is an integer of magnitude <= 16 dqk <= 4096.  Each query is 2 u_h plus noise in
    [-2, 2], u_h a +-1 direction of its head, so a key 4 u_h scores about 8 dqk against every row, far above the live
    keys (std sqrt(40 dqk)).  `poison` (B, M) bool: those keys get 4 u_h and V codes +-448 (saturated e4m3).  q / k
    descales differ per head and put the live scores' std at `spread` log2 units; v descales are v_descale()."""
    g = torch.Generator().manual_seed(seed)
    Bq = B if Bq is None else Bq
    u = torch.randint(0, 2, (H, dqk), generator=g) * 2 - 1
    q = torch.randint(-2, 3, (Bq, N, H, dqk), generator=g) + 2 * u
    k = torch.randint(-4, 5, (B, M, H, dqk), generator=g)
    v = (torch.randn(B, M, H, dv, generator=g) * 64.0).clamp(-448.0, 448.0)
    if poison is not None:
        pz = poison[:, :, None, None]
        k = torch.where(pz, 4 * u, k)
        v = torch.where(pz, torch.where(torch.rand(B, M, H, dv, generator=g) < 0.5, -448.0, 448.0), v)
    c = spread / math.sqrt(40.0 * dqk)  # log2-domain factor per unit of q8 . k8
    d = math.sqrt(c / (dqk ** -0.5 * math.log2(math.e)))
    qd = d * (1.0 + 0.25 * torch.arange(H).float())
    kd = d / (1.0 + 0.25 * torch.arange(H).float()) * (1.0 + 0.1 * torch.arange(H).float())
    vt8 = _vt(_to_f8(v.reshape(B, M, H * dv), device), H)
    return (_to_f8(q.reshape(Bq, N, H * dqk), device), _to_f8(k.reshape(B, M, H * dqk), device), vt8,
            qd.to(device), kd.to(device), v_descale(H, dv).to(device))


def _vt(v8, H):
    from perceiver_io_b200 import ops

    return ops.fp8_transpose_v(v8, H)


# ---- exact probes ----
# Scores take the levels 0 and 16 only; with a log2-domain factor c >= 10.5 the gap is >= 168 > 160 log2 units, so every
# probability below the row maximum is exactly 0 after ex2.approx.ftz (and every merge weight after exp2f).
PROBE_C = 10.5
PROBE_SUM_LIMIT = 2 ** 12  # sum_j |v8_j| of a channel: 2^8 times it is a multiple of 2^8 below 2^20 (12 bits)


def needle_keys(M, dqk):
    """Key of channel c's needle: spread from key 0 (first tile) to M - 1 (last, ragged tile)."""
    return [round(c * (M - 1) / max(1, dqk - 1)) for c in range(dqk)]


def query_channel(N, H, dqk):
    """(N, H) the channel of row n's one-hot query."""
    return (torch.arange(N)[:, None] * 7 + torch.arange(H)[None, :] * 3) % dqk


def probe_operands(kind, B, N, M, H, dqk, dv, Bq=None, poison=None, device="cuda"):
    """Operands of the needle ("needle") or count ("count") probe.  Needle: row n's query is 4 on channel
    query_channel(n) and the needle key of that channel carries K code 4 there, so it scores 16 and every other live key
    0.  Count: q codes 0, so every live key scores 0.  `poison` keys carry K code 4 on every channel (they score 16
    against every needle query).  V codes are small integers (1..3 on live keys, 5..7 on poisoned ones) on the needle
    keys (every channel) and on a sparse pattern elsewhere, so the P V sums are exact integers (PROBE_SUM_LIMIT)."""
    Bq = B if Bq is None else Bq
    q = torch.zeros(Bq, N, H, dqk)
    if kind == "needle":
        q.scatter_(3, query_channel(N, H, dqk)[None, :, :, None].expand(Bq, N, H, 1), 4.0)
    elif kind != "count":
        raise KeyError(kind)
    k = torch.zeros(B, M, H, dqk)
    nk = needle_keys(M, dqk)
    k[:, nk, :, torch.arange(dqk)] = 4.0
    pz = torch.zeros(B, M, dtype=torch.bool) if poison is None else poison
    k = torch.where(pz[:, :, None, None], torch.full_like(k, 4.0), k)
    j = torch.arange(M)[None, :, None, None]
    c = torch.arange(dv)[None, None, None, :]
    h = torch.arange(H)[None, None, :, None]
    b = torch.arange(B)[:, None, None, None]
    period = max(1, math.ceil(7 * M / (PROBE_SUM_LIMIT // 2)))
    on = ((j * 13 + c * 7 + h) % period == 0)
    isneedle = torch.zeros(M, dtype=torch.bool)
    isneedle[nk] = True
    on = on | isneedle[None, :, None, None]
    code = 1 + (j + 3 * c + 5 * h + 7 * b) % 3 + 4 * pz[:, :, None, None]
    v = torch.where(on, code, 0).float()
    sl2 = score_scale(dqk ** -0.5, torch.ones(1), torch.ones(1)).item()
    base = torch.tensor([PROBE_C + 0.75 * i for i in range(H)], dtype=torch.float64) / sl2
    qd = (base.sqrt() * 1.25).float()
    kd = (base.sqrt() / 1.25).float()
    vt8 = _vt(_to_f8(v.reshape(B, M, H * dv), device), H)
    return (_to_f8(q.reshape(Bq, N, H * dqk), device), _to_f8(k.reshape(B, M, H * dqk), device), vt8, qd.to(device),
            kd.to(device), v_descale(H, dv).to(device))


def live_mask(B, N, M, pad_mask=None, causal=False, m_total=None, m_offset=0, device="cpu"):
    """(B, N, M) True where key j is live for row n (the kernel's padded / causal rule)."""
    live = torch.ones(B, N, M, dtype=torch.bool, device=device)
    if pad_mask is not None:
        live &= ~pad_mask.to(device).bool()[:, None, :]
    if causal:
        m_total = M if m_total is None else m_total
        shift = (m_total - N) - m_offset
        live &= ~(torch.arange(M, device=device)[None, :] > torch.arange(N, device=device)[:, None] + shift)[None]
    return live


def probe_expected(q8, k8, vt8, qd, kd, vd, H, scale, pad_mask=None, causal=False, m_total=None, m_offset=0):
    """The exact result of a probe call: every key at the row's top live score level has p = 1, every other p = 0; a
    row without a live key averages over all M keys (kMaskedScore is finite).  Returns (out fp32 before the 16-bit
    rounding, part_o, part_m, part_l) with out = fp32(sum v8 vd) * fp32(1 / count), part_o = sum v8 vd,
    part_m = fp32(s_max * c) (-FLT_MAX for a row without a live key), part_l = count; (B, H, N[, dv])."""
    dev = k8.device
    Bq, N, Cq = q8.shape
    B, M, _ = k8.shape
    dqk, dv = Cq // H, vt8.shape[2]
    q = q8.double().reshape(Bq, N, H, dqk).permute(0, 2, 1, 3).expand(B, H, N, dqk)
    k = k8.double().reshape(B, M, H, dqk).permute(0, 2, 1, 3)
    s = q @ k.transpose(-1, -2)  # exact integers
    live = live_mask(B, N, M, pad_mask, causal, m_total, m_offset, dev)[:, None].expand(B, H, N, M)
    smax = s.masked_fill(~live, -math.inf).amax(dim=-1)
    anylive = live.any(dim=-1)
    sel = torch.where(anylive[..., None], live & (s == smax[..., None]), torch.ones_like(live))
    v8 = vt8[..., :M].double().transpose(-1, -2)  # (B, H, M, dv)
    S = (sel.double() @ v8) * vd.double()[None, :, None, :]
    cnt = sel.sum(dim=-1)
    c = score_scale(scale, qd, kd).float().to(dev)  # fp32, as the kernel forms p.scale_log2 * qd * kd
    m = torch.where(anylive, (smax.float() * c[None, :, None]), torch.full_like(smax.float(), -FLT_MAX))
    inv = 1.0 / cnt.float()
    out = S.float() * inv[..., None]
    return out, S.float(), m, cnt.float()


def probe_gap_and_sums(q8, k8, vt8, qd, kd, H, scale):
    """(smallest gap in log2 units between the two score levels of any row, largest sum_j |v8_j| of a channel)."""
    Bq, N, Cq = q8.shape
    B, M, _ = k8.shape
    dqk = Cq // H
    q = q8.double().reshape(Bq, N, H, dqk).permute(0, 2, 1, 3)
    k = k8.double().reshape(B, M, H, dqk).permute(0, 2, 1, 3)
    levels = torch.unique(q.expand(B, -1, -1, -1) @ k.transpose(-1, -2))
    c = score_scale(scale, qd, kd)
    gap = (levels[1:] - levels[:-1]).min().item() * c.min().item() if len(levels) > 1 else math.inf
    sums = vt8[..., :M].double().abs().sum(dim=-1).max().item()
    return gap, sums, sorted(levels.tolist())


# --------------------------------------------------------------------------------------------------
# the per-element gate
# --------------------------------------------------------------------------------------------------
# A: relative precision of the FP8 wgmma's accumulation of P V against sum_j p^_j |v_j|.  Hopper's FP8 MMA keeps about
# 14 bits, but relative to the largest product of a k32 step (the products are aligned to it), so a step of 32 similar
# products can lose about 2^-8 of their sum.  Measured on one H100 SXM: up to 2.0e-3 (2^-9), in rows of one to three key
# tiles with flat scores; the published 2^-12 fails there by a factor of up to 6.
ACC_A = 2.0 ** -8
U_OUT = {BF16: 2.0 ** -8, FP16: 2.0 ** -11, None: 0.0}
OLD_GATE = 2.0 ** -6  # test_gpu_fp8.py: 2^-6 sum_j p_j |v_j|
U32 = 2.0 ** -24


def gate_terms(ref, out_dtype):
    """Per-element terms (B, H, N, dv) of the bound on |kernel - emulation| for one call (out_dtype None: the partial
    state, as part_o / part_l):
      - flip: probabilities whose e4m3 rounding the kernel's exponent error can change, one e4m3 step each;
      - acc:  A sum_j p^_j |v_j| vd / l, the FP8 wgmma accumulation;
      - den:  the fp32 denominator (its probabilities' relative error and the sum's depth) and the fp32 rescale factors;
      - out:  the 16-bit rounding of the output, and the fp32 multiplies of the epilogue."""
    absout = ref["out"].abs()
    flip = ref["flip"]
    acc = ACC_A * ref["pv_hat"]
    den = absout * (ref["rho"] + ref["nadd"] * U32)[..., None] + 2.0 * ref["rho_w"][..., None] * ref["pv_hat"]
    rest = flip + acc + den
    out = U_OUT[out_dtype] * (absout + rest) + 4 * U32 * absout
    if out_dtype == FP16:
        out = out + 2.0 ** -25  # half a subnormal step
    return {"flip": flip, "acc": acc, "den": den, "out": out}


def gate_report(got, ref, out_dtype):
    """(err / gate worst, measured A, worst share of each term) of `got` (B, H, N, dv) float64 against the emulation."""
    terms = gate_terms(ref, out_dtype)
    gate = sum(terms.values())
    err = (got - ref["out"]).abs()
    ratio = (err / gate.clamp_min(1e-300))
    worst = ratio.max().item()
    excess = (err - (gate - terms["acc"])).clamp_min(0.0) / ref["pv_hat"].clamp_min(1e-300)
    a_meas = excess.max().item()
    shares = {k: (v / gate.clamp_min(1e-300)).max().item() for k, v in terms.items()}
    return worst, a_meas, shares, err <= gate


def out_to_bhnd(out, H):
    """(B, N, H*dv) output -> (B, H, N, dv) float64."""
    B, N, C = out.shape
    return out.double().reshape(B, N, H, C // H).permute(0, 2, 1, 3)


def round_out(x, out_dtype):
    return x.to(torch.bfloat16 if out_dtype == BF16 else torch.float16).double()
