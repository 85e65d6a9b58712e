"""Variant matrix, schedule rules and CPU emulation of the tensor-core attention on an FP8 KV cache
(perceiver_io_b200/csrc/pcv_attn_cached.cu, pcv_attn_cached_fp8), shared by its GPU tests (test_gpu_cached_fp8.py) and
their CPU companion (test_cached_fp8_cpu.py).  Nothing here needs a GPU.

launch_attn_cached without device rows instantiates attn_cached_kernel<BF16, FP8 = true, WIN = false, NVB>:
  - BF16: bf16 or fp16 (the dtype of q and out, and of the converted K / V tiles);
  - NVB: the 64-channel boxes of a V row, ceil(dv / 64), 1 to 4.
The Q / K box count ceil(dqk / 64) is a runtime value (the number of Q K^T k-steps and the stage size).
Each rule below names the function of pcv_attn_cached.cu it restates."""
import itertools
import math

import torch

from gpu_util import ABS_SPACING, UNIT_ROUNDOFF, decode_element_bound, torch_core

BF16, FP16 = "bf16", "fp16"
DTYPES = (BF16, FP16)
DTYPE = {BF16: torch.bfloat16, FP16: torch.float16}
KEYS = 64                    # kKeys: keys per tile
MAX_ROWS = 64                # kMaxRows: query rows of the m64 tile
BOX = 64 * 128               # kBox
MAX_STAGES = 4               # kMaxStages
SMEM_LIMIT = 226 * 1024      # kSmemLimit
PAIR_BUDGET = 110 * 1024     # kPairBudget
MIN_TILES = 4                # plan_cached: at least 4 tiles (256 keys) per split
MAX_SPLITS = 256
SMS = 132                    # the H100 SXM's SM count; sm_count falls back to 132 without a device
FLT_MAX = torch.finfo(torch.float32).max
LOG2E = 1.4426950408889634


def device_sms():
    """The SM count plan_cached plans with: the current device's when there is one, else the fallback 132."""
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return SMS


# ---- the restated rules ----
def plan(B, H, M, dqk, dv, sms=SMS):
    """plan_cached: box counts, CTAs per SM, ring stages, dynamic shared memory and the split of the key tiles."""
    nkb, nvb = -(-dqk // 64), -(-dv // 64)
    per_sm = 2 if (nvb == 1 and nkb <= 3) else 1
    budget = PAIR_BUDGET if per_sm == 2 else SMEM_LIMIT
    fixed = nkb * BOX + 1024 + 2 * MAX_STAGES * 8
    stages = min(MAX_STAGES, (budget - fixed) // ((nkb + nvb) * BOX))
    tiles = -(-M // KEYS)
    bh = B * H
    want = max(1, -(-(2 * per_sm * sms) // bh))
    want = min(want, max(1, tiles // MIN_TILES), MAX_SPLITS)
    tps = -(-tiles // want)
    return dict(nkb=nkb, nvb=nvb, per_sm=per_sm, stages=stages, smem=fixed + stages * (nkb + nvb) * BOX,
                tiles=tiles, tiles_per_split=tps, nsplit=-(-tiles // tps))


def split_ranges(M, pl):
    """[kb, ke) of every split: whole tiles, the last split (and its last tile) ragged."""
    tps = pl["tiles_per_split"] * KEYS
    return [(s * tps, min(M, (s + 1) * tps)) for s in range(pl["nsplit"])]


def workspace_bytes(B, H, N, M, dqk, dv, sms=SMS):
    """workspace_of: ws_o, ws_m, ws_l of B*H*nsplit*N rows and B*H tickets, each 256-aligned."""
    a256 = lambda x: (x + 255) // 256 * 256  # noqa: E731
    rows = B * H * plan(B, H, M, dqk, dv, sms)["nsplit"] * N
    return a256(rows * dv * 4) + 2 * a256(rows * 4) + a256(B * H * 4)


def serial_depth(pl):
    """The longest chain of fp32 roundings and ex2 factors one probability passes through (element_bound):
    the sum over a tile's keys inside the MMA (counted as one rounding per key), one rescale per tile of the split, the
    merge over the splits, and the descale, quotient and output roundings."""
    return KEYS + pl["tiles_per_split"] + pl["nsplit"] + 4


def element_bound(q, k, v, H, scale, pad, causal, dtype, depth):
    """(bound, ref) of the kernel's element-wise gate, (B, N, H*dv) fp64 on k's device: gpu_util.decode_element_bound
    (the output rounding, the fp32 scores, ex2 and the fp32 sums along `depth`) plus the rounding of P.  The kernel rounds
    each probability to 16 bits before P V while its denominator sums the fp32 ones, which moves the output by at most
    u sum_j p_j |v_j| (relative u per p, p normalised), plus one absolute spacing per rounded p below the normal range
    (fp16 subnormals, ex2's flush for bf16): spacing sum_j |v_j|, as the row's largest p is 1 and its denominator at
    least 1.  Both enter the relative terms that decode_element_bound doubles.  q, k, v as in decode_element_bound (the
    e4m3 rows dequantised)."""
    bound, ref = decode_element_bound(q, k, v, H, scale, pad, causal, dtype, depth)
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    va = v.detach().to(k.device, torch.float64).abs()
    pv = torch_core(q.to(k.device), k, va, H, scale, pad, causal, torch.float64)               # sum_j p_j |v_j|
    vsum = va.reshape(B, M, H, -1).sum(1).reshape(B, 1, -1)                                     # sum_j |v_j|
    return bound + 2.0 * (UNIT_ROUNDOFF[dtype] * pv + ABS_SPACING[dtype] * vsum), ref


# ---- the instantiations ----
def variant_of(dt, dv):
    return (dt, -(-dv // 64))


def reachable_variants():
    """Every whole-cache instantiation launch_attn_cached can reach: head dims 16..256 in multiples of 16, both dtypes."""
    return {variant_of(dt, dv) for dt, dv in itertools.product(DTYPES, range(16, 257, 16))}


# (dqk, dv) per NVB: the smallest and the widest rows, dqk != dv both ways, GiantMIDI's 96 and the bench's 128
HEAD_DIMS = {1: [(16, 16), (192, 64)], 2: [(96, 96), (128, 80)], 3: [(64, 160)], 4: [(256, 256)]}


def _matrix():
    return [(dt, dqk, dv) for dt in DTYPES for dims in HEAD_DIMS.values() for dqk, dv in dims]


#: (dtype, dqk, dv): every reachable instantiation at least once
VARIANT_CASES = _matrix()


def case_id(case):
    dt, dqk, dv = case
    return f"{dt}-qk{dqk}-v{dv}"


#: query rows and cache lengths of the edge sweep; SPLIT_M is planned at B = 3, H = 2 as 3 splits of 5 tiles, the last
#: split 3 tiles and its last tile 37 keys
EDGE_N = (1, 5, 8, 63, 64)
EDGE_M = (1, 63, 64, 65)
EDGE_B, EDGE_H, SPLIT_M = 3, 2, 805


def edge_ms(N):
    return sorted(set(EDGE_M) | {N, SPLIT_M})


def edge_keys(M, pl, N, limit=60):
    """Keys under test for the count probe: the first and last key of every split, the first and last key of every
    tile of the first and last split, and the causal diagonals of the N rows (at most `limit`)."""
    marks = set()
    ranges = split_ranges(M, pl)
    for kb, ke in ranges:
        marks |= {kb, ke - 1}
    for kb, ke in (ranges[0], ranges[-1]):
        for t0 in range(kb, ke, KEYS):
            marks |= {t0, min(t0 + KEYS, ke) - 1}
    diag = [M - N + i for i in range(N)]
    marks |= set(diag[:8] + diag[-8:])
    marks = sorted(m for m in marks if 0 <= m < M)
    assert len(marks) <= limit, len(marks)
    return marks


# ---- the kernel's arithmetic on the CPU ----
def _rn(x, dtype):
    return x.to(dtype).to(torch.float32)


def emulate(q, k8, v8, kd, vd, H, scale, pad, causal, dt, sms=SMS):
    """The output of the whole-cache attn_cached_kernel restated in torch: fp32 scores from exact codes and the 16-bit q, the row
    maximum of round(s c), p = 2^(s c - m) with one rounding (fp64 then fp32), the fp32 running sums per 64-key tile,
    P rounded to the 16-bit type before P V, v_descale on the fp32 accumulator, the merge of the splits in split order
    and the rounding of o / l.  q (Bq, N, H*dqk) 16-bit, k8 / v8 (B, M, H*d) e4m3, kd (H,), vd (H, dv)."""
    dtype = DTYPE[dt]
    B, M = k8.shape[0], k8.shape[1]
    N = q.shape[1]
    qh = q.float().expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)          # (B, H, N, dqk)
    kh = k8.float().reshape(B, M, H, -1).transpose(1, 2)
    vh = v8.float().reshape(B, M, H, -1).transpose(1, 2)
    dqk, dv = qh.shape[-1], vh.shape[-1]
    pl = plan(B, H, M, dqk, dv, sms)
    c = (torch.tensor(scale * LOG2E, dtype=torch.float32) * kd.float().cpu())[None, :, None, None]   # (1, H, 1, 1)
    j = torch.arange(M)
    masked = torch.zeros(B, 1, N, M, dtype=torch.bool)
    if pad is not None:
        masked = masked | pad.cpu().bool()[:, None, None, :]
    if causal:
        masked = masked | (j[None, :] > (torch.arange(N)[:, None] + M - N))[None, None]
    s_all = qh.cpu() @ kh.cpu().transpose(-1, -2)                                   # fp32 scores (B, H, N, M)
    states = []
    for kb, ke in split_ranges(M, pl):
        m_run = torch.full((B, H, N, 1), -math.inf)
        l_run = torch.zeros(B, H, N, 1)
        o = torch.zeros(B, H, N, dv)
        for t0 in range(kb, ke, KEYS):
            t1 = min(t0 + KEYS, ke)
            s = s_all[..., t0:t1]
            mk = masked[..., t0:t1].expand_as(s)
            x = torch.where(mk, torch.tensor(-FLT_MAX), s * c)
            mn = torch.maximum(m_run, x.amax(-1, keepdim=True))
            alpha = torch.exp2(m_run - mn)
            ex = torch.where(mk, torch.tensor(-FLT_MAX, dtype=torch.float64) - mn.double(),
                             s.double() * c.double() - mn.double()).float()
            p = torch.exp2(ex.double()).float()
            l_run = l_run * alpha + p.sum(-1, keepdim=True)
            o = o * alpha + _rn(p, dtype) @ vh.cpu()[..., t0:t1, :]
            m_run = mn
        states.append((o * vd.float().cpu()[None, :, None, :], m_run, l_run))
    mm = torch.stack([m for _, m, _ in states]).amax(0)
    ov, ll = torch.zeros_like(states[0][0]), torch.zeros_like(states[0][2])
    for o, m, l in states:
        wt = torch.exp2(m - mm)
        ov = ov + o * wt
        ll = ll + l * wt
    return (ov / ll).to(dtype).transpose(1, 2).reshape(B, N, H * dv)


def random_operands(B, Bq, N, M, H, dqk, dv, dt, seed, device="cpu"):
    """(q, k8, v8, kd, vd): 16-bit q of unit scale, e4m3 codes of random rows spanning the e4m3 range, and descales
    that give the dequantised K unit-scale rows and V per-channel scales differing by channel."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = torch.randn(Bq, N, H * dqk, generator=g).to(DTYPE[dt])
    k8 = (torch.randn(B, M, H * dqk, generator=g) * 64).clamp(-448, 448).to(torch.float8_e4m3fn)
    v8 = (torch.randn(B, M, H * dv, generator=g) * 64).clamp(-448, 448).to(torch.float8_e4m3fn)
    kd = (torch.rand(H, generator=g) + 0.5) / 64
    vd = (torch.rand(H, dv, generator=g) + 0.5) / 64
    return tuple(t.to(device) for t in (q, k8, v8, kd, vd))


def left_pad(B, M, device="cpu"):
    """Batch row 0 unpadded, row 1 left-padded by a third of the keys, row 2 (if any) wholly padded."""
    pad = torch.zeros(B, M, dtype=torch.bool, device=device)
    if B > 1:
        pad[1, :M // 3] = True
    if B > 2:
        pad[2] = True
    return pad
