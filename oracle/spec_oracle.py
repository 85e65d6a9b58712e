"""CPU restatement (Python integers) of the device's speculative-sampling verifier, pcv_spec_verify
(perceiver_io_b200/csrc/pcv_sample.cu), on top of sample_oracle's filter and hash.

TEST INFRASTRUCTURE ONLY — nothing under perceiver_io_b200/ imports this file.

    masses          P_i / Zp_i: sample_oracle.filter_row's kept masses of target row i under the target's values (greedy,
                    temperature 0 or a max scaled value of +-inf: 2^40 at the first maximal index); Q_i / Zq_i: the same
                    for draft row i under the draft's values
    accept          t_{i+1} = x is accepted iff (u_a * Q_i(x) * Zp_i) >> 64 < P_i(x) * Zq_i
    n               the first rejected i, or G
    correction      R(y) = max(0, P(y) Zq - Q(y) Zp) on row n; the first index whose prefix sum of R exceeds
                    (u_r * ΣR) >> 64; ΣR = 0: the draw from P below
    bonus / P draw  the first index whose prefix P mass exceeds (u_r * Zp) >> 64
    streams         sample_oracle.uniform_bits' construction with other round keys: u_a (accept) and u_r (residual) at
                    (seed, b, positions[i])

Ambiguity.  As in sample_oracle, the device's fp64 exp can move a mass by 1 where 2^40 exp(d) lies near a half-integer
(``slack`` such tokens per row, U), so Z moves by at most U.  A verdict is flagged when such moves could cross:
  an acceptance comparison: |L - R| within (Zp + U_p) + Q(x) U_p + 1 + (Zq + U_q) + P(x) U_q (each term present only
  when its row has slack);
  a residual or draw boundary: every R(y) moves by at most |ΔP(y)| (Zq + U_q) + P(y) U_q + |ΔQ(y)| (Zp + U_p) + Q(y) U_p,
  so ΣR and every prefix by E = U_p (Zq + U_q) + Zp U_q + U_q (Zp + U_p) + Zq U_p, and t by E + 1; flagged when t lies
  within 2E + 2 of the drawn token's edges (2U + 16 for a draw from P, sample_oracle's rule), or ΣR <= E;
  a top-p cut, or the rows' own top-k / greedy / top-p flags of sample_oracle.sample_row with ``logit_err``.
With ``logit_err`` = e > 0 (the logits known to within e each) every mass ratio moves by a factor within exp(+-2e/T),
so the comparisons and boundaries above also take a relative margin eps = expm1(4e/T) of their magnitudes.
"""
import math
from typing import List, NamedTuple

import numpy as np

from oracle import sample_oracle as S

ONE = 1 << 40
_STREAM_HALVES = {
    "accept": ((0xD2511F53, 0xCD9E8D57, 0x428A2F98, 0x71374491, 0xB5C0FBCF),
               (0xCD9E8D57, 0xD2511F53, 0xE9B5DBA5, 0x3956C25B, 0x59F111F1)),
    "residual": ((0xD2511F53, 0xCD9E8D57, 0x923F82A4, 0xAB1C5ED5, 0xD807AA98),
                 (0xCD9E8D57, 0xD2511F53, 0x12835B01, 0x243185BE, 0x550C7DC3)),
}
_M32 = 0xFFFFFFFF


def stream_bits(seed, b, pos, stream: str) -> np.ndarray:
    """uint64 bits of the "accept" or "residual" stream at (seed, b, pos), broadcast as sample_oracle.uniform_bits."""
    seed = np.asarray(seed)
    seed = seed if seed.dtype == np.uint64 else seed.astype(np.int64).astype(np.uint64)
    b = np.asarray(b).astype(np.int64).astype(np.uint64) & np.uint64(_M32)
    pos = np.asarray(pos).astype(np.int64).astype(np.uint64) & np.uint64(_M32)
    with np.errstate(over="ignore"):
        word = ((b * np.uint64(0x9E3779B1) + pos) & np.uint64(_M32)) * np.uint64(0x85EBCA6B) & np.uint64(_M32)
        lo, hi = seed & np.uint64(_M32), seed >> np.uint64(32)
        halves = []
        for ca, cb, k0, k1, k2 in _STREAM_HALVES[stream]:
            x = S._round(word ^ lo, ca, k0)
            x = S._round(x ^ hi, cb, k1)
            halves.append(S._round(x, ca, k2))
    return (halves[1] << np.uint64(32)) | halves[0]


def _bits(seed: int, b: int, pos: int, stream: str) -> int:
    return int(stream_bits(np.uint64(seed & (2 ** 64 - 1)), b, pos, stream))


class Masses(NamedTuple):
    w: List[int]     # kept masses
    Z: int
    slack: int       # tokens whose mass the device's exp could round the other way
    cut_amb: bool    # the top-p cut lies within the slack of a tie-group boundary


def masses(logits, temperature: float, top_k: int, top_p: float) -> Masses:
    logits = np.asarray(logits, dtype=np.float32)
    tok = S.greedy_token(logits, temperature)
    if tok is not None:
        w = [0] * len(logits)
        w[tok] = ONE
        return Masses(w, ONE, 0, False)
    f = S.filter_row(logits, temperature, top_k, top_p)
    w = [int(v) for v in np.where(f.kept, f.w, np.uint64(0))]
    amb = bool(f.slack and f.cut >= 0 and np.any(np.abs(f.W.astype(np.float64) - f.cut) <= 2 * f.slack + 16))
    return Masses(w, f.z_kept, f.slack, amb)


def first_exceeding(weights: List[int], t: int):
    """(index, prefix before it, prefix through it) of the first index whose prefix sum exceeds t."""
    acc = 0
    for y, v in enumerate(weights):
        if acc + v > t:
            return y, acc, acc + v
        acc += v
    raise AssertionError("t is not below the total")


def residual(P: Masses, Q: Masses) -> List[int]:
    return [max(0, p * Q.Z - q * P.Z) for p, q in zip(P.w, Q.w)]


class Verdict(NamedTuple):
    tokens: List[int]    # (G+1): the accepted drafts, the correction or bonus token, -1
    n: int
    ambiguous: bool
    why: str


def _row_flags(logits, vals, logit_err: float) -> List[str]:
    if logit_err <= 0:
        return []
    d = S.sample_row(logits, *vals, seed=0, b=0, pos=0, logit_err=logit_err)
    return [w for w in d.why.split("; ") if w and not w.startswith("draw")]


def _eps(vals, logit_err: float) -> float:
    return math.expm1(4 * logit_err / vals[0]) if logit_err > 0 and vals[0] > 0 else 0.0


def verify_row(target_rows, draft_rows, tokens, sampling, draft_sampling, seed: int, b: int, positions,
               logit_err: float = 0.0) -> Verdict:
    """The device's verdict for one batch row: target_rows (G+1, V), draft_rows (G, V), tokens t_0 .. t_G, positions
    (G+1); ``logit_err`` applies to the target rows."""
    target_rows = np.asarray(target_rows, dtype=np.float32)
    draft_rows = np.asarray(draft_rows, dtype=np.float32)
    G, V = draft_rows.shape
    why: List[str] = []
    eps = _eps(sampling, logit_err)
    n = G
    for i in range(G):
        P = masses(target_rows[i], *sampling)
        Q = masses(draft_rows[i], *draft_sampling)
        why += [f"row {i}: {w}" for w in _row_flags(target_rows[i], sampling, logit_err)]
        if P.cut_amb or Q.cut_amb:
            why.append(f"row {i}: top-p cut within the mass slack")
        x = int(tokens[i + 1])
        px, qx = (P.w[x], Q.w[x]) if 0 <= x < V else (0, 0)
        L = (_bits(seed, b, int(positions[i]), "accept") * qx * P.Z) >> 64
        R = px * Q.Z
        margin = ((P.Z + P.slack if Q.slack else 0) + qx * P.slack + (Q.Z + Q.slack if P.slack else 0) + px * Q.slack
                  + (1 if P.slack or Q.slack else 0))
        margin += int(eps * max(L, R)) + (1 if eps else 0)
        if margin and abs(L - R) <= margin:
            why.append(f"row {i}: acceptance within the error")
        if L >= R:
            n = i
            break
    out = [int(t) for t in tokens[1:n + 1]]
    u = _bits(seed, b, int(positions[n]), "residual")
    P = masses(target_rows[n], *sampling)
    if n < G:
        Q = masses(draft_rows[n], *draft_sampling)
        Rw = residual(P, Q)
        SR = sum(Rw)
        E = P.slack * (Q.Z + Q.slack) + P.Z * Q.slack + Q.slack * (P.Z + P.slack) + Q.Z * P.slack
        E += int(2 * eps * P.Z * Q.Z)
        if E and SR <= E:
            why.append("residual sum within the error of 0")
        if SR > 0:
            t = (u * SR) >> 64
            tok, lo, hi = first_exceeding(Rw, t)
            if (E or eps) and (t - lo <= 2 * E + 2 or hi - 1 - t <= 2 * E + 2):
                why.append("residual draw within the error")
            out.append(tok)
            out += [-1] * (G - n)
            return Verdict(out, n, bool(why), "; ".join(why))
    if n == G:
        why += [f"row {G}: {w}" for w in _row_flags(target_rows[G], sampling, logit_err)]
        if P.cut_amb:
            why.append(f"row {G}: top-p cut within the mass slack")
    t = (u * P.Z) >> 64
    tok, lo, hi = first_exceeding(P.w, t)
    s = (2 * P.slack + 16 if P.slack else 0) + int(eps * P.Z)
    if s and (t - lo <= s or hi - 1 - t <= s):
        why.append("draw from P within the error")
    out.append(tok)
    out += [-1] * (G - n)
    return Verdict(out, n, bool(why), "; ".join(why))
