"""Variant matrix, schedule rules, mask semantics and CPU emulation of the banded-window tensor-core attention over a KV
arena (perceiver_io_b200/csrc/pcv_attn_cached.cu, pcv_attn_cached_window / _fp8), shared by its GPU tests
(test_gpu_window.py) and their CPU companion (test_window_cpu.py).  Nothing here needs a GPU.

launch_attn_cached with device rows instantiates attn_cached_kernel<BF16, FP8, WIN = true, NVB>:
  - BF16: bf16 or fp16 (the dtype of q and out, and of the K / V tiles in shared memory);
  - FP8: e4m3 arena rows (converted in shared memory) or rows of q's 16-bit type;
  - NVB: the 64-channel boxes of a V row, ceil(dv / 64), 1 to 4.
Each rule below names the function of pcv_attn_cached.cu it restates."""
import itertools
import math

import torch

from cached_fp8_variants import DTYPE, DTYPES, FLT_MAX, KEYS, LOG2E, SMS, _rn, element_bound
from cached_fp8_variants import plan as cached_plan

KINDS = ("16bit", "e4m3")


# ---- the restated rules ----
def plan(B, H, capacity, dqk, dv, sms=SMS):
    """plan_cached on M = capacity (the split count is fixed for the arena)."""
    return cached_plan(B, H, capacity, dqk, dv, sms)


def clamp_window(b0, b1, capacity):
    """The window the kernel reads: [max(b0, 0), min(b1, capacity)), empty when its length is <= 0."""
    return max(b0, 0), min(b1, capacity)


def split_tiles(b0, b1, capacity, nsplit):
    """attn_cached_kernel (WIN): the key range [kb, ke) of every split.  The window's 64-key tiles start at its begin;
    split s takes tiles [min(T, s tps), min(T, s tps + tps)) with tps = ceil(T / nsplit), T = ceil(length / 64)."""
    w0, wend = clamp_window(b0, b1, capacity)
    T = -(-max(wend - w0, 0) // KEYS)
    tps = -(-T // nsplit)
    out = []
    for s in range(nsplit):
        t0 = min(T, s * tps)
        t1 = min(T, t0 + tps)
        out.append((w0 + t0 * KEYS, min(wend, w0 + t1 * KEYS)) if t1 > t0 else (w0, w0))
    return out


def workspace_bytes(B, H, N, capacity, dqk, dv, sms=SMS):
    """workspace_of: ws_o, ws_m, ws_l of B*H*nsplit*N rows and B*H tickets, each 256-aligned."""
    a256 = lambda x: (x + 255) // 256 * 256  # noqa: E731
    rows = B * H * plan(B, H, capacity, dqk, dv, sms)["nsplit"] * N
    return a256(rows * dv * 4) + 2 * a256(rows * 4) + a256(B * H * 4)


def row_keys(i, N, b0, b1, capacity, band, causal):
    """(lo, hi, causal_fill): the keys query i attends, [lo, hi), and the first of them (or hi) that the causal mask
    fills.  Query i sits at r_i = end - N + i of the clamped window.  A band W > 0 keeps [r_i + 1 - W, r_i]: no causal
    fill, keys outside it are excluded.  W = 0 keeps the window, with keys past r_i filled when causal."""
    w0, wend = clamp_window(b0, b1, capacity)
    r = wend - N + i
    if wend <= w0:
        return w0, w0, w0
    if band > 0:
        lo, hi = max(w0, r + 1 - band), min(wend, r + 1)
        return lo, max(lo, hi), max(lo, hi)
    return w0, wend, (max(w0, min(wend, r + 1)) if causal else wend)


def depth(b0, b1, capacity, pl):
    """The serial depth of element_bound at the run-time split: KEYS + tiles per split + splits + 4."""
    w0, wend = clamp_window(b0, b1, capacity)
    T = -(-max(wend - w0, 0) // KEYS)
    return KEYS + -(-T // pl["nsplit"]) + pl["nsplit"] + 4


# ---- the instantiations ----
def variant_of(dt, kind, dv):
    return (dt, kind, -(-dv // 64))


def reachable_variants():
    """Every window instantiation launch_attn_cached can reach: head dims up to 256 in multiples of 8 (16-bit rows) or 16
    (e4m3 rows), both dtypes."""
    return {variant_of(dt, kind, dv) for dt, kind in itertools.product(DTYPES, KINDS)
            for dv in range(8 if kind == "16bit" else 16, 257, 8 if kind == "16bit" else 16)}


# (dqk, dv) per NVB: 16-bit rows also take head dims that are odd multiples of 8 (a zero-filled half k16 step)
HEAD_DIMS = {"16bit": {1: [(40, 24)], 2: [(128, 128)], 3: [(96, 136)], 4: [(256, 256)]},
             "e4m3": {1: [(16, 16)], 2: [(128, 80)], 3: [(64, 160)], 4: [(256, 256)]}}

#: (dtype, kind, dqk, dv): every reachable instantiation at least once
VARIANT_CASES = [(dt, kind, dqk, dv) for dt in DTYPES for kind in KINDS for dims in HEAD_DIMS[kind].values()
                 for dqk, dv in dims]


def case_id(case):
    dt, kind, dqk, dv = case
    return f"{dt}-{kind}-qk{dqk}-v{dv}"


# ---- the kernel's arithmetic on the CPU ----
def masks(N, b0, b1, capacity, band, causal, pad):
    """(keep, filled): (B, 1, N, capacity) bools — the keys query i attends, and those of them that take the fill."""
    B = pad.shape[0] if pad is not None else 1
    keep = torch.zeros(N, capacity, dtype=torch.bool)
    cfill = torch.zeros(N, capacity, dtype=torch.bool)
    for i in range(N):
        lo, hi, cf = row_keys(i, N, b0, b1, capacity, band, causal)
        keep[i, lo:hi] = True
        cfill[i, cf:hi] = True
    filled = cfill[None, None].expand(B, 1, N, capacity)
    if pad is not None:
        filled = filled | pad.cpu().bool()[:, None, None, :]
    return keep[None, None], filled & keep[None, None]


def emulate(q, k, v, kd, vd, H, scale, b0, b1, band, pad, causal, dt, sms=SMS):
    """The output of the window attn_cached_kernel restated in torch: fp32 scores of the 16-bit q and the exact K rows (e4m3 codes
    when kd is given), the row maximum of round(s c) over the attended keys, p = 2^(s c - m) with one rounding, fp32
    running sums per 64-key tile from the window's begin, no rescale while a row has no key, P rounded to the 16-bit
    type before P V, v_descale on the fp32 accumulator, the merge in split order with empty splits at weight 0, and
    o / l rounded (zero for a row without keys)."""
    dtype = DTYPE[dt]
    B, cap, N = k.shape[0], k.shape[1], q.shape[1]
    qh = q.float().cpu().expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = k.float().cpu().reshape(B, cap, H, -1).transpose(1, 2)
    vh = v.float().cpu().reshape(B, cap, H, -1).transpose(1, 2)
    dqk, dv = qh.shape[-1], vh.shape[-1]
    pl = plan(B, H, cap, dqk, dv, sms)
    c = torch.tensor(scale * LOG2E, dtype=torch.float32)
    if kd is not None:
        c = c * kd.float().cpu()[None, :, None, None]
    keep, filled = masks(N, b0, b1, cap, band, causal, pad)
    s_all = qh @ kh.transpose(-1, -2)
    states = []
    for kb, ke in split_tiles(b0, b1, cap, pl["nsplit"]):
        m_run = torch.full((B, H, N, 1), -math.inf)
        l_run = torch.zeros(B, H, N, 1)
        o = torch.zeros(B, H, N, dv)
        for t0 in range(kb, ke, KEYS):
            t1 = min(t0 + KEYS, ke)
            s = s_all[..., t0:t1]
            kp = keep[..., t0:t1].expand_as(s)
            fl = filled[..., t0:t1].expand_as(s)
            x = torch.where(kp, torch.where(fl, torch.tensor(-FLT_MAX), s * c), torch.tensor(-math.inf))
            mn = torch.maximum(m_run, x.amax(-1, keepdim=True))
            empty = mn == -math.inf
            alpha = torch.where(empty, torch.ones_like(mn), torch.exp2(m_run - torch.where(empty, 0.0, mn)))
            mnd = torch.where(empty, 0.0, mn).double()
            ex = torch.where(fl, torch.tensor(-FLT_MAX, dtype=torch.float64) - mnd, s.double() * c.double() - mnd).float()
            p = torch.where(kp, torch.exp2(ex.double()).float(), torch.zeros(()))
            l_run = l_run * alpha + p.sum(-1, keepdim=True)
            o = o * alpha + _rn(p, dtype) @ vh[..., t0:t1, :]
            m_run = mn
        states.append((o * vd.float().cpu()[None, :, None, :] if vd is not None else o, m_run, l_run))
    mm = torch.stack([m for _, m, _ in states]).amax(0)
    ov, ll = torch.zeros_like(states[0][0]), torch.zeros_like(states[0][2])
    for o, m, l in states:
        wt = torch.where(m == -math.inf, torch.zeros(()), torch.exp2(m - torch.where(mm == -math.inf, 0.0, mm)))
        ov = ov + o * wt
        ll = ll + l * wt
    out = torch.where(ll > 0, ov / torch.where(ll > 0, ll, 1.0), torch.zeros(()))
    return out.to(dtype).transpose(1, 2).reshape(B, N, H * dv)


def reference_and_bound(q, k, v, H, scale, b0, b1, band, pad, causal, dt, pl):
    """(ref, bound) (B, N, H*dv) fp64 on k's device: row by row, cached_fp8_variants.element_bound on the keys that
    row attends (row_keys), their fill as its pad mask, so excluded keys drop out of every sum.  k / v are the rows the
    kernel computes on (e4m3 rows dequantised).  A row without keys is zero, exactly."""
    B, cap, N = k.shape[0], k.shape[1], q.shape[1]
    dv = v.shape[2] // H
    ref = torch.zeros(B, N, H * dv, dtype=torch.float64, device=k.device)
    bound = torch.zeros_like(ref)
    dep = depth(b0, b1, cap, pl)
    for i in range(N):
        lo, hi, cf = row_keys(i, N, b0, b1, cap, band, causal)
        if hi <= lo:
            continue
        fill = torch.zeros(B, hi - lo, dtype=torch.bool, device=k.device)
        fill[:, cf - lo:] = True
        if pad is not None:
            fill = fill | pad[:, lo:hi].to(k.device).bool()
        bd, rf = element_bound(q[:, i:i + 1], k[:, lo:hi], v[:, lo:hi], H, scale, fill, False, DTYPE[dt], dep)
        ref[:, i:i + 1], bound[:, i:i + 1] = rf, bd
    return ref, bound


def random_operands(B, Bq, N, cap, H, dqk, dv, dt, kind, seed, device="cpu"):
    """(q, k, v, kd, vd, k64, v64): 16-bit q of unit scale; arenas of q's type (kd = vd = None) or e4m3 codes with
    descales as cached_fp8_variants.random_operands; and the fp64 rows they stand for."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    dtype = DTYPE[dt]
    q = torch.randn(Bq, N, H * dqk, generator=g).to(dtype)
    if kind == "16bit":
        k = torch.randn(B, cap, H * dqk, generator=g).to(dtype)
        v = torch.randn(B, cap, H * dv, generator=g).to(dtype)
        kd = vd = None
        k64, v64 = k.double(), v.double()
    else:
        k = (torch.randn(B, cap, H * dqk, generator=g) * 64).clamp(-448, 448).to(torch.float8_e4m3fn)
        v = (torch.randn(B, cap, H * dv, generator=g) * 64).clamp(-448, 448).to(torch.float8_e4m3fn)
        kd = (torch.rand(H, generator=g) + 0.5) / 64
        vd = (torch.rand(H, dv, generator=g) + 0.5) / 64
        k64 = (k.double().reshape(B, cap, H, -1) * kd.double()[:, None]).reshape(B, cap, -1)
        v64 = (v.double().reshape(B, cap, H, -1) * vd.double()).reshape(B, cap, -1)
    return tuple(t.to(device) if t is not None else None for t in (q, k, v, kd, vd, k64, v64))


# ---- exact probes (the operands are decode_variants.count_operands / needle_operands) ----
def key_sets(B, N, b0, b1, capacity, band, causal, pad, device="cpu"):
    """(in_range, live) (B, N, capacity) bools for decode_variants.count_expect / needle_expect: the keys each row
    attends (row_keys), and those of them that are neither padded nor past the causal diagonal.  A row whose attended
    keys are all filled is the average over all of them; a row that attends no key is zero."""
    rng = torch.zeros(N, capacity, dtype=torch.bool)
    unfilled = torch.zeros(N, capacity, dtype=torch.bool)
    for i in range(N):
        lo, hi, cf = row_keys(i, N, b0, b1, capacity, band, causal)
        rng[i, lo:hi] = True
        unfilled[i, lo:cf] = True
    in_range = rng.to(device)[None].expand(B, N, capacity)
    live = in_range & unfilled.to(device)[None] & ~pad.to(device).bool()[:, None, :]
    return in_range, live


def _edge_rows(N, per_side=3):
    return sorted(set(range(min(per_side, N))) | set(range(max(0, N - per_side), N)))


def split_edges(b0, b1, capacity, nsplit):
    """The first and last key of every non-empty split, and of the first and last tile of the first and last of them."""
    live = [(kb, ke) for kb, ke in split_tiles(b0, b1, capacity, nsplit) if ke > kb]
    marks = set()
    for kb, ke in live:
        marks |= {kb, ke - 1}
    for kb, ke in ({live[0], live[-1]} if live else ()):
        last = kb + (ke - 1 - kb) // KEYS * KEYS
        marks |= {kb, min(kb + KEYS, ke) - 1, last, ke - 1}
    return marks


def row_edges(i, N, b0, b1, capacity, band, causal):
    """Row i's mask edges: the first attended key and the one before it (the band's lower edge r_i + 1 - W, or the
    window's begin), the last attended key and the one after it, and the causal diagonal r_i and the key past it."""
    lo, hi, cf = row_keys(i, N, b0, b1, capacity, band, causal)
    return {lo - 1, lo, hi - 1, hi, cf - 1, cf}


def probe_marks(N, b0, b1, capacity, band, causal, nsplit, limit=60):
    """The keys whose V the count probe sets: the window's edges and the keys next to them, the split and tile edges
    (split_edges) and the mask edges of the first and last three rows (row_edges).  At most `limit`, so that S stays
    below 64 codes and one key more or less moves S / L by more than a 16-bit ulp."""
    w0, wend = clamp_window(b0, b1, capacity)
    marks = {w0 - 1, w0, wend - 1, wend} | split_edges(b0, b1, capacity, nsplit)
    for i in _edge_rows(N):
        marks |= row_edges(i, N, b0, b1, capacity, band, causal)
    marks = sorted(m for m in marks if 0 <= m < capacity)
    assert len(marks) <= limit, len(marks)
    return marks


def needle_candidates(N, b0, b1, capacity, band, causal, nsplit, pad):
    """cands[b][n]: the keys a needle of query row n of batch row b is placed on: its own mask edges (row_edges), the
    window's edges and the keys next to them, the split and tile edges, and the first and last padded key of the
    window."""
    w0, wend = clamp_window(b0, b1, capacity)
    shared = {w0 - 1, w0, wend - 1, wend} | split_edges(b0, b1, capacity, nsplit)
    out = []
    for b in range(pad.shape[0]):
        padded = pad[b, w0:wend].nonzero() if wend > w0 else pad[b, :0].nonzero()
        pb = {w0 + int(padded[0]), w0 + int(padded[-1])} if padded.numel() else set()
        out.append([sorted(c for c in shared | pb | row_edges(n, N, b0, b1, capacity, band, causal)
                           if 0 <= c < capacity) for n in range(N)])
    return out


def needles(B, H, N, cands, r):
    """(B, H, N) needle keys of round r: row n of batch row b walks its own list cands[b][n], H keys a round."""
    out = torch.zeros(B, H, N, dtype=torch.long)
    for b, h, n in itertools.product(range(B), range(H), range(N)):
        c = cands[b][n]
        out[b, h, n] = c[(r * H + h) % len(c)]
    return out


def needle_rounds(cands, H):
    """Rounds of `needles` that put a needle on every candidate of every row."""
    return max(-(-len(c) // H) for rows in cands for c in rows)
