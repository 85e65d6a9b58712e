"""Rules and exact probe rows of the kernels that scan one vocabulary row per 512-thread CTA: sample_kernel and
spec_verify_kernel (pcv_sample.cu), beam_rows_kernel (pcv_beam.cu), cs_candidates_kernel (pcv_contrastive.cu) and
process_kernel (pcv_process.cu), on the row primitives of pcv_vocab.cuh.  Shared by test_gpu_vocab_variants.py and its
CPU companion test_vocab_variants_cpu.py.  Nothing here needs a GPU.

The restated rules cite the line of pcv_vocab.cuh (or of the kernel's file) they restate:
  - kThreads = 512 threads, kWarps = 16 warps (:14-15);
  - warp_segment(V): warp w scans [w * seg, min(V, w * seg + seg)), seg = ceil(V / 512) * 32, so later warps may be
    empty and the last live one ragged (:44-48);
  - order_key: an order-preserving uint32 key, -0 folded onto +0 (:18-22); select_key: the k-th largest key by four
    8-bit passes from the top byte, each a count histogram of the keys that share the prefix chosen so far (:54-97);
  - collect_top: every key above the threshold, then the keys equal to it in warp-segment order, which is index order
    because the segments are contiguous and ascending (:138-177); top_rank orders them key descending, index ascending
    (:180-186);
  - beams_to_keep = max(2, E + 1) * K (pcv_beam.cu:35-37); a row keeps min(beams_to_keep, V) candidates and writes
    fillers (-inf, index -1) after them (pcv_beam.cu:69-86).

Every probe row is a float32 array whose values are representable in the dtype it was built for, so a bf16 / fp16
tensor of it holds the same values.  Each builder states the structure it claims; the CPU companion checks the claim."""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import numpy as np

from oracle import sample_oracle as S

THREADS = 512
WARPS = THREADS // 32
MAX_VOCAB = 32768
MASS_ONE = 1 << 40
DTYPES = ("bf16", "fp16", "fp32")
# every warp_segment shape: one live warp (20 ragged, 32 full), a second warp of one element (33), sixteen live warps
# with the last ragged (511, 32767) or full (512, 32768), nine live warps of which the last holds one element (513)
VOCABS = (20, 32, 33, 511, 512, 513, 16 * 2048 - 1, 32768)
# a draw counter whose t = hi64(bits * (2^40 + 32767)) lands in the run of 32767 mass-1 tokens (found by a search of
# uniform_bits over positions; test_vocab_variants_cpu checks it)
DENSE_DRAW = ((1, 0, 6320554), (1, 0, 11766342))


# ---- the restated rules -------------------------------------------------------------------------------------------------
def warp_segment(V: int, w: int):
    """[s0, s1) of warp w (:44-48); empty when s1 <= s0."""
    seg = (V + THREADS - 1) // THREADS * 32
    s0 = w * seg
    return s0, min(V, s0 + seg)


def segment_shape(V: int):
    """(live warps, size of the last live segment, segment size, empty warps) of warp_segment(V)."""
    segs = [warp_segment(V, w) for w in range(WARPS)]
    live = [s for s in segs if s[1] > s[0]]
    return len(live), live[-1][1] - live[-1][0], (V + THREADS - 1) // THREADS * 32, WARPS - len(live)


def order_key(x, fold_zero: bool = True) -> np.ndarray:
    """order_key (:18-22) of float32 values, as uint64 (the uint32 key)."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    if fold_zero:
        u = np.where(u == 0x80000000, np.uint64(0), u)
    neg = (u & np.uint64(0x80000000)) != 0
    return np.where(neg, ~u & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))


def select_key(x, k: int, fold_zero: bool = True):
    """select_key (:54-97): (the k-th largest key, [the (bin, still needed) chosen by each of the four passes])."""
    keys = order_key(x, fold_zero)
    prefix, need, passes = 0, k, []
    for shift in (24, 16, 8, 0):
        hi_mask = 0 if shift == 24 else (0xFFFFFFFF << (shift + 8)) & 0xFFFFFFFF
        live = keys[(keys & np.uint64(hi_mask)) == np.uint64(prefix)]
        hist = np.bincount(((live >> np.uint64(shift)) & np.uint64(255)).astype(np.int64), minlength=256)
        above = 0
        for d in range(255, -1, -1):       # the bin d with above(d) < need <= above(d) + h[d], from the top
            if above < need <= above + hist[d]:
                prefix |= d << shift
                need -= above
                passes.append((d, need))
                break
            above += int(hist[d])
    return prefix, passes


def deciding_pass(x, k: int) -> Optional[int]:
    """The select_key pass (1-4) whose histogram first separates the k-th from the (k+1)-th largest key: 1 + the high
    bytes they share; None when k >= V or the two keys are equal."""
    keys = np.sort(order_key(x))[::-1]
    if k >= keys.shape[0] or keys[k - 1] == keys[k]:
        return None
    diff = int(keys[k - 1]) ^ int(keys[k])
    return 4 - (diff.bit_length() - 1) // 8


def collect_top(x, nsel: int, eq_order: str = "warps", fold_zero: bool = True, lose_last: bool = False):
    """collect_top (:138-177) then top_rank (:180-186): the indices of the nsel largest keys, ranked.  The keys equal to
    the threshold are taken warp by warp in segment order (eq_order="warps"); the mutants take them "reversed" (highest
    index first) or with the warps in "reversed_warps" order, and ``lose_last`` drops the last element of the last live
    segment."""
    x = np.asarray(x, dtype=np.float32)
    V = x.shape[0]
    keys = order_key(x, fold_zero)
    if lose_last:
        keys = keys[:-1]
        V -= 1
        nsel = min(nsel, V)
    thr, _ = select_key(x[:V], nsel, fold_zero)
    gt = [i for i in range(V) if keys[i] > thr]
    segs = [warp_segment(V, w) for w in range(WARPS)]
    if eq_order == "reversed_warps":
        segs = segs[::-1]
    eq = [i for s0, s1 in segs for i in range(s0, s1) if keys[i] == thr]
    if eq_order == "reversed":
        eq = eq[::-1]
    taken = gt + eq[:nsel - len(gt)]
    return sorted(taken, key=lambda i: (-int(keys[i]), i))


def top_reference(x, nsel: int):
    """The nsel largest values, value descending and index ascending on ties (-0 == +0): a stable sort."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64) + 0.0
    return np.lexsort((np.arange(x.shape[0]), -x))[:nsel].tolist()


def beams_to_keep(K: int, E: int) -> int:
    return max(2, E + 1) * K


def row_candidates(acc, keep: int, fillers_first: bool = False):
    """beam_rows_kernel's scratch row (pcv_beam.cu:69-86): (scores, indices within the row) of the top min(keep, V) of
    the fp32 row ``acc``, then fillers (-inf, -1).  The mutant puts the fillers before the -inf candidates."""
    acc = np.asarray(acc, dtype=np.float32)
    nsel = min(keep, acc.shape[0])
    idx = top_reference(acc, nsel)
    if fillers_first:
        fin = [i for i in idx if np.isfinite(acc[i])]
        idx = fin + [-1] * (keep - nsel) + [i for i in idx if not np.isfinite(acc[i])]
    else:
        idx = idx + [-1] * (keep - nsel)
    scores = np.array([acc[i] if i >= 0 else -np.inf for i in idx], dtype=np.float32)
    return scores, np.array(idx, dtype=np.int64)


# ---- dtype grids --------------------------------------------------------------------------------------------------------
def _bits(dt):
    return 32 if dt == "fp32" else 16


def dkey(v, dt: str) -> int:
    """The order key of a value in the dtype's own bits (16 or 32), -0 folded onto +0."""
    nb = _bits(dt)
    f = np.float32(v)
    if dt == "fp32":
        u = int(f.view(np.uint32))
    elif dt == "fp16":
        u = int(np.float16(f).view(np.uint16))
    else:
        u = int(f.view(np.uint32)) >> 16
    sign = 1 << (nb - 1)
    u = 0 if u == sign else u
    return (~u & ((1 << nb) - 1)) if u & sign else u | sign


def dval(k: int, dt: str) -> np.float32:
    """The float32 value of the dtype key k."""
    nb = _bits(dt)
    sign = 1 << (nb - 1)
    u = k & (sign - 1) if k & sign else ~k & ((1 << nb) - 1)
    if dt == "fp32":
        return np.uint32(u).view(np.float32)
    if dt == "fp16":
        return np.float32(np.uint16(u).view(np.float16))
    return np.uint32(u << 16).view(np.float32)


def representable(x, dt: str) -> bool:
    x = np.asarray(x, dtype=np.float32)
    if dt == "fp32":
        return True
    if dt == "fp16":
        return bool(np.array_equal(x.astype(np.float16).astype(np.float32), x, equal_nan=True))
    return bool(np.all((x.view(np.uint32) & np.uint32(0xFFFF)) == 0))


def largest_finite(dt: str) -> np.float32:
    return {"fp32": np.finfo(np.float32).max, "fp16": np.float32(65504.0),
            "bf16": np.uint32(0x7F7F0000).view(np.float32)}[dt]


def min_subnormal(dt: str) -> np.float32:
    return dval((1 << (_bits(dt) - 1)) + 1, dt)


# ---- masses -------------------------------------------------------------------------------------------------------------
def masses(x, m):
    """(w, ambiguous) of sample_oracle: w = round(2^40 exp(x - m)), 0 below -29; ambiguous within 2^-9 of a half."""
    d = np.asarray(x, dtype=np.float32).astype(np.float64) - np.float64(np.float32(m))
    e = np.exp(d) * S.MASS_SCALE
    e[d < -29.0] = 0.0
    frac = e - np.floor(e)
    return np.rint(e).astype(np.uint64), (d >= -29.0) & (np.abs(frac - 0.5) < 2.0 ** -9)


class Probe(NamedTuple):
    name: str
    dtype: str
    x: np.ndarray       # the fp32 row
    k: int              # the selection size it targets (top_k, nsel)
    claim: dict         # the structure the builder states


def _fill(keys_lo: int, keys_hi: int, n: int, dt: str, rng) -> np.ndarray:
    """n values whose dtype keys lie in [keys_lo, keys_hi]."""
    if n <= 0:
        return np.zeros(0, np.float32)
    ks = rng.integers(keys_lo, keys_hi + 1, size=n)
    return np.array([dval(int(k), dt) for k in ks], dtype=np.float32)


def _unambiguous(x: np.ndarray, fixed, dt: str, lo_key: int, hi_key: int) -> np.ndarray:
    """Moves every token whose mass the device's exp could round the other way one dtype step down (up when that would
    leave the keys [lo_key, hi_key] it started in) until none is left; the row maximum and ``fixed`` stay."""
    fixed = set(fixed) | {int(np.argmax(x))}
    for _ in range(256):
        _, amb = masses(x, x.max())
        bad = [i for i in np.nonzero(amb)[0] if i not in fixed]
        if not bad:
            return x
        for i in bad:
            k = dkey(x[i], dt)
            x[i] = dval(k - 1 if k - 1 >= lo_key or k < lo_key else k + 1, dt)
    raise AssertionError("could not clear the mass slack")


# ---- radix probes -------------------------------------------------------------------------------------------------------
def radix_probe(V: int, k: int, byte: int, negative: bool, dt: str, seed: int) -> Probe:
    """The k-th and (k+1)-th largest dtype keys are consecutive and first differ in dtype key byte ``byte`` (a borrow
    across every lower byte, as 0x3f800000 -> 0x3f7fffff), near +-1.5; k - 1 values above the pair share its prefix up
    to that byte, V - k - 1 below.  Claims the fp32 keys' deciding pass (for fp32 rows: 4 - byte)."""
    rng = np.random.default_rng(seed)
    c = dkey(np.float32(-1.5 if negative else 1.5), dt)
    ka0 = c & ~((1 << (8 * byte)) - 1)
    top = byte == _bits(dt) // 8 - 1    # the top byte: keep the values finite and of one sign
    span = (1 << (_bits(dt) - 12) if top else min(1 << (8 * byte + 8), 1 << 20)) - 1
    for attempt in range(64):        # every mass must be exact: move the pair along byte `byte` until it is
        ka = ka0 + (attempt << (8 * byte))
        if (ka >> (8 * byte)) & 255 == 0:
            continue
        kb = ka - 1
        above = _fill(ka + 1, ka + span, k - 1, dt, rng)
        below = _fill(kb - span, kb - 1, V - k - 1, dt, rng) if k < V else np.zeros(0, np.float32)
        pair = [dval(ka, dt)] + ([dval(kb, dt)] if k < V else [])
        perm = rng.permutation(V)
        row = np.empty(V, np.float32)
        row[perm] = np.concatenate([above, np.array(pair, np.float32), below])
        ia, ib = int(perm[k - 1]), (int(perm[k]) if k < V else -1)
        row = _unambiguous(row, [ia, ib], dt, ka + 1, ka + span)
        if S.filter_row(row, 1.0, 0, 1.0).slack == 0:
            break
    else:
        raise AssertionError("no exact radix probe")
    assert representable(row, dt)
    claim = dict(pass_=deciding_pass(row, k) if k < V else None, negative=negative, kth=float(dval(ka, dt)))
    return Probe(f"radix V={V} k={k} byte={byte} {'neg' if negative else 'pos'}", dt, row, k, claim)


def radix_probes(V: int, dt: str):
    ks = sorted({1, min(2, V), V // 2, V - 1, V} - {0})
    out = []
    for k in ks:
        for byte in range(_bits(dt) // 8):
            for negative in (False, True):
                out.append(radix_probe(V, k, byte, negative, dt, seed=V * 131 + k * 7 + byte * 3 + negative))
    return out


def zero_probes(V: int, k: int, dt: str, seed: int):
    """Cuts at the sign change: (a) -0 and +0 tie at the k-th key (-0 at the lower index); (b) +min subnormal k-th, +0
    (k+1)-th; (c) +0 k-th, -min subnormal (k+1)-th.  k - 1 positive values above the cut, the rest negative."""
    assert 1 <= k and k + 1 <= V
    rng = np.random.default_rng(seed)
    sub = min_subnormal(dt)
    out = []
    for case, cut in (("-0/+0 tie", [np.float32(-0.0), np.float32(0.0)]), ("+sub/0", [sub, np.float32(0.0)]),
                      ("0/-sub", [np.float32(0.0), -sub])):
        above = np.abs(_fill(dkey(np.float32(0.25), dt), dkey(np.float32(1.0), dt), k - 1, dt, rng))
        below = -np.abs(_fill(dkey(np.float32(0.25), dt), dkey(np.float32(1.0), dt), V - k - 1, dt, rng))
        pos = rng.permutation(V)
        row = np.empty(V, np.float32)
        row[pos[:k - 1]] = above
        i0, i1 = sorted(pos[k - 1:k + 1].tolist())
        row[i0], row[i1] = cut
        row[pos[k + 1:]] = below
        row = _unambiguous(row, [i0, i1], dt, 0, 1 << _bits(dt))
        while S.filter_row(row, 1.0, 0, 1.0).slack:   # a cut value's own mass is inexact: lower the row maximum
            i = int(np.argmax(row))
            row[i] = dval(dkey(row[i], dt) - 1, dt)
        out.append(Probe(f"zero {case} V={V} k={k}", dt, row, k, dict(cut=case, at=(i0, i1))))
    return out


def max_probes(V: int, dt: str, seed: int):
    """The dtype's largest finite value is the largest key (k = 1), its predecessor the second; in fp32 rows also the
    fp16 and bf16 maxima, with larger fp32 values above them (k = V // 2)."""
    rng = np.random.default_rng(seed)
    out = []
    tops = [(dt, 1)] + ([("fp16", max(1, V // 2)), ("bf16", max(1, V // 2))] if dt == "fp32" else [])
    for which, k in tops:
        if k + 1 > V:
            continue
        top = largest_finite(which)
        kt = dkey(top, dt)
        above = _fill(kt + 1, kt + 4096, k - 1, dt, rng)
        below = _fill(kt - 2 - 4096, kt - 2, V - k - 1, dt, rng)
        pos = rng.permutation(V)
        row = np.empty(V, np.float32)
        row[pos[:k - 1]] = above
        row[pos[k - 1]] = top
        row[pos[k]] = dval(kt - 1, dt)
        row[pos[k + 1:]] = below
        row = _unambiguous(row, [int(pos[k - 1]), int(pos[k])], dt, kt + 1, kt + 4096)
        out.append(Probe(f"max {which} in {dt} V={V} k={k}", dt, row, k, dict(kth=float(top))))
    return out


def inf_probes(V: int, k: int, dt: str, seed: int):
    """-inf at the cut (k - 1 finite values, the rest -inf: a -inf tie group holds the k-th key) and below it (k
    finite, the rest -inf); the finite values integers in [-4, 4] (ties among them too)."""
    rng = np.random.default_rng(seed)
    out = []
    for n_fin, case in ((k - 1, "at"), (k, "below")):
        if n_fin >= V or n_fin < 0:
            continue
        row = np.full(V, -np.inf, np.float32)
        pos = rng.permutation(V)[:n_fin]
        row[pos] = rng.integers(-4, 5, size=n_fin).astype(np.float32)
        out.append(Probe(f"-inf {case} the cut V={V} k={k}", dt, row, k, dict(finite=n_fin)))
    return out


def tie_probes(V: int, nsel: int, dt: str, seed: int):
    """A tie group at the cut larger than the number still needed, straddling one warp-segment boundary, several, or
    the boundary to the empty segments (its members the last indices of the last live warp and the first of the one
    before).  Claims: the group's indices, how many it must give, and the segment boundaries it crosses."""
    rng = np.random.default_rng(seed)
    segs = [warp_segment(V, w) for w in range(WARPS)]
    starts = [s0 for s0, s1 in segs[1:] if s1 > s0]
    live = [s for s in segs if s[1] > s[0]]
    layouts = []
    if starts:
        b = starts[len(starts) // 2]
        layouts.append(("one boundary", [b - 2, b - 1, b, b + 1]))
    if len(starts) >= 3:
        layouts.append(("several boundaries", sorted({starts[0] - 1, starts[0], starts[1] - 1, starts[1], starts[2]})))
    if len(live) < WARPS and len(live) >= 2:
        s0 = live[-1][0]
        layouts.append(("the empty segments", sorted({s0 - 1, s0, V - 1})))
    out = []
    for case, group in layouts:
        group = [g for g in group if 0 <= g < V]
        need = max(1, len(group) // 2)
        n_above = nsel - need
        if n_above < 0 or n_above + len(group) > V:
            continue
        rest = [i for i in range(V) if i not in group]
        rng.shuffle(rest)
        row = np.empty(V, np.float32)
        row[group] = 1.0
        row[rest[:n_above]] = rng.integers(2, 9, size=n_above).astype(np.float32)
        row[rest[n_above:]] = rng.integers(-6, 1, size=len(rest) - n_above).astype(np.float32)
        bounds = [s for s in starts if group[0] < s <= group[-1]]
        out.append(Probe(f"tie across {case} V={V} nsel={nsel}", dt, row, nsel,
                         dict(group=group, need=need, crosses=bounds)))
    return out


# ---- top-p boundary probes ----------------------------------------------------------------------------------------------
def _below(v, dt):
    return dval(dkey(v, dt) - 1, dt)


def _largest_with_mass_at_most(R: int, m, below, dt: str):
    """The largest dtype value v < ``below`` with an exact mass w(v) <= R (w > 0), and w(v)."""
    v = _round_to(np.float64(m) + math.log(R / S.MASS_SCALE), dt) if R < MASS_ONE else below
    v = min(v, _below(below, dt))
    while True:
        w, amb = masses(np.array([v]), m)
        if 0 < w[0] <= R and not amb[0]:
            return v, int(w[0])
        v = _below(v, dt)


def _round_to(v, dt):
    """v as a value of the dtype (bf16: truncated), in float32."""
    if dt == "fp32":
        return np.float32(v)
    if dt == "fp16":
        return np.float32(np.float16(v))
    return np.uint32(int(np.float32(v).view(np.uint32)) & 0xFFFF0000).view(np.float32)


def top_p_probe(V: int, top_p: float, over: int, ng: int, dt: str, seed: int) -> Optional[Probe]:
    """A row whose group at the cut has W<= == cut + over (over 0: the group goes; 1: it stays, and with ng >= 2 it
    straddles the cut).  n0 top tokens at m ~ 1.25 * 2^-10 (n0 = 1 at top_p 0.5, 3 at 0.75, so the cut lands near 2^40),
    ng tokens of the group just below m, fillers below it making up W<= exactly (largest exact masses first, down to
    mass-1 tokens near d = -27.8), the rest at m - 60 (mass 0).  None when V is too small for the fillers."""
    rng = np.random.default_rng(seed)
    m = _round_to(1.25 * 2.0 ** -10, dt)
    n0 =1 if top_p == 0.5 else 3
    pf = float(np.float32(top_p))
    W = None
    for t in range(64):
        cand = MASS_ONE + t
        if cand - math.floor((1.0 - pf) * float(cand + n0 * MASS_ONE)) == over:
            W = cand
            break
    assert W is not None
    vg, wg = _largest_with_mass_at_most((W - 1) // ng, m, m, dt)
    vals = [m] * n0 + [vg] * ng
    R = W - ng * wg
    while R > 0:
        v, w = _largest_with_mass_at_most(R, m, vg, dt)
        c = R // w
        vals += [v] * c
        R -= c * w
        if len(vals) > V:
            return None
    row = np.full(V, _round_to(m - 60.0, dt), np.float32)
    pos = rng.permutation(V)[:len(vals)]
    row[pos] = np.array(vals, np.float32)
    f = S.filter_row(row, 1.0, 0, top_p)
    gi = int(np.nonzero(f.vals == vg)[0][0])
    return Probe(f"top-p {top_p} W<=cut+{over} ng={ng} V={V}", dt, row, 0,
                 dict(top_p=top_p, over=over, ng=ng, W=int(f.W[gi]), cut=f.cut, slack=f.slack, group=float(vg)))


def top_p_probes(V: int, dt: str):
    out = []
    for top_p in (0.5, 0.75):
        for over in (0, 1):
            for ng in (1, 2):
                p = top_p_probe(V, top_p, over, ng, dt, seed=V + int(top_p * 8) + 2 * over + 4 * ng)
                if p is not None:
                    out.append(p)
    return out


# ---- draw probes --------------------------------------------------------------------------------------------------------
def segment_draw_probe(V: int, w: int, dt: str):
    """The kept set is the last token of warp w's segment and the first of warp w+1's, at mass 2^40 each (x = 0), the
    rest at -60 (mass 0); with counters (seed 5, b, pos) searched so that each of the two is drawn.  Returns (probe,
    [(pos, token)] for the first and the second token at batch row b = 0)."""
    s0, s1 = warp_segment(V, w)
    t0, t1 = warp_segment(V, w + 1)
    assert s1 > s0 and t1 > t0 and s1 == t0
    row = np.full(V, -60.0, np.float32)
    row[[s1 - 1, t0]] = 0.0
    picks = {}
    for pos in range(64):
        t = (int(S.uniform_bits(np.uint64(5), 0, pos)) * 2 * MASS_ONE) >> 64
        picks.setdefault(s1 - 1 if t < MASS_ONE else t0, pos)
        if len(picks) == 2:
            break
    empty_after = warp_segment(V, w + 2)[1] <= warp_segment(V, w + 2)[0]
    return (Probe(f"segment draw V={V} warps {w}/{w + 1}", dt, row, 2, dict(tokens=(s1 - 1, t0), empty_after=empty_after)),
            sorted((p, t) for t, p in picks.items()))


def segment_draw_probes(dt: str):
    """Every boundary kind: inside sixteen live warps (1000, 32767, 32768), before the empty segments (33, 513)."""
    cases = [(1000, 3), (32767, 14), (32768, 7), (33, 0), (513, 7)]
    return [segment_draw_probe(V, w, dt) for V, w in cases]


def dense_draw_probe(dt: str) -> Probe:
    """32767 tokens of mass 1 (d ~ -27.8) and the top token last: t below 32767 picks token t itself (the first whose
    prefix t + 1 exceeds t); DENSE_DRAW holds counters that land there."""
    V = MAX_VOCAB
    m = np.float32(0.5)
    a = _round_to(np.float32(0.5 - 27.8), dt) if dt != "fp32" else np.float32(0.5 - 27.8)
    row = np.full(V, a, np.float32)
    row[-1] = m
    return Probe(f"dense mass-1 draw {dt}", dt, row, 0, dict(mass_one=V - 1))


# ---- zero-mass probes ---------------------------------------------------------------------------------------------------
def zero_mass_probes(V: int, dt: str):
    """(probe, temperature, expected token) of rows the sampler takes as greedy (their largest scaled value is not
    finite) and one that keeps its normal draw: every logit -inf (token 0); the dtype's largest finite value at two
    indices at T = 0.5, which overflows fp32 in bf16 and fp32 rows (the lower index); -inf except one token (that
    token, drawn normally with log-probability 0)."""
    out = []
    row = np.full(V, -np.inf, np.float32)
    out.append((Probe(f"all -inf V={V}", dt, row, 0, dict(greedy=True)), 1.0, 0))
    if dt != "fp16":
        big = np.float32(3e38) if dt == "fp32" else largest_finite("bf16")
        row = np.linspace(-3, 3, V).astype(np.float32)
        row = np.array([_round_to(v, dt) for v in row], np.float32) if dt != "fp32" else row
        i0, i1 = (V // 3, V - 1) if V > 3 else (V - 1, V - 1)
        row[[i1, i0]] = big
        out.append((Probe(f"{big:.3g} at T=0.5 V={V}", dt, row, 0, dict(greedy=True)), 0.5, min(i0, i1)))
    row = np.full(V, -np.inf, np.float32)
    j = (V * 2) // 3
    row[j] = -3.0
    out.append((Probe(f"one finite token V={V}", dt, row, 0, dict(greedy=False)), 1.0, j))
    return out


# ---- processor probes ---------------------------------------------------------------------------------------------------
def processor_cases(V: int, seed: int):
    """(name, histories (R lists of ids), kwargs of process_logits / process_oracle.process) at the processor's edges:
    the last seen word partial (V % 32 != 0 in PROCESS_VOCABS), histories longer than 512 (more than one stride of the
    loops), duplicates, ids -1 and V (matched, never written), L + 1 == N and L + 1 == N - 1, N = 1 and N = 8, and
    min_new_tokens at L - prompt_len == M - 1 and == M."""
    rng = np.random.default_rng(seed)
    tail_ids = [V - 1, V - 2, 32 * (V // 32)] if V % 32 else [V - 1]
    out = []
    long = rng.integers(0, min(V, 7), size=700).tolist() + tail_ids + [-1, V, 3, -1, V]
    out.append(("long history, duplicates, -1 and V", [long, long[::-1], long[:513]],
                dict(repetition_penalty=1.3, no_repeat_ngram_size=2)))
    out.append(("N = 1 bans the history", [long[:600] + tail_ids, [V, -1] * 300, tail_ids],
                dict(repetition_penalty=0.7, no_repeat_ngram_size=1)))
    # an n-gram whose banned next id is out of range: a write there would land in the row
    oob = [5, 6, -1, 5, 6, V, 5, 6]
    out.append(("banned ids -1 and V", [oob, oob[:5] + [5, 6], oob + [9] * 600 + [5, 6]], dict(no_repeat_ngram_size=3)))
    for N in (3, 8):
        h = rng.integers(0, 4, size=N + 5).tolist()
        out.append((f"N = {N} at L + 1 == N and N - 1, L == N", [h[:N - 1], h[:N - 2], h[:N], [7] * N, h + h],
                    dict(no_repeat_ngram_size=N)))
    base = rng.integers(0, V, size=40).tolist()
    for M in (1, 4):
        hists = [base[:30 + M - 1], base[:30 + M], base[:30 + M + 1], base[:30]]
        out.append((f"min_new_tokens={M} at its boundary", hists,
                    dict(min_new_tokens=M, prompt_len=30, eos=(0, V - 1), repetition_penalty=1.1)))
    return out


PROCESS_VOCABS = (33, 97, 32767)
