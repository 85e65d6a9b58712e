"""CPU restatement (numpy, exact integer arithmetic) of the device token sampler, pcv_sample (perceiver_io_b200/csrc/
pcv_sample.cu).

TEST INFRASTRUCTURE ONLY — nothing under perceiver_io_b200/ imports this file.

    bits(seed, b, pos)  two evaluations (multipliers (ca, cb), keys (k0, k1, k2) per half) of three multiply-hi/lo
                        rounds (pcv_hash.cuh's hash_round):
                          word = ((b * 0x9E3779B1 + pos) * 0x85EBCA6B) mod 2^32
                          x = round(word ^ seed_lo, ca, k0); x = round(x ^ seed_hi, cb, k1); x = round(x, ca, k2)
                          bits = half_1 << 32 | half_0
    x_i                 float32(logit_i) / float32(temperature), IEEE fp32 division (temperature 0: greedy argmax;
                        a row whose max x is +-inf has no finite mass and is greedy too: the first index of the max)
    top-k               keep x_i >= the k-th largest x (ties with it stay); 0 or >= V: off
    w_i                 round_half_even(2^40 exp(float64(x_i) - float64(max x))), 0 where x_i - max x < -29
    top-p               cut = floor((1 - float64(float32(top_p))) * float64(Z)); drop i iff W<=(x_i) <= cut, the top
                        tie group always stays
    draw                t = (bits * Z_kept) >> 64; the first index whose kept prefix mass exceeds t

Ambiguity.  x is reproduced bit for bit (both sides divide in IEEE fp32) and d = x - max x is exact in fp64 wherever
w can be non-zero, so the only difference between this file and the device is exp: the device's fp64 exp is within
1 ulp (CUDA C Programming Guide, table of double-precision functions), numpy's within 1 ulp, so 2^40 exp(d) differs by
at most 2^-11 and w_i by at most 1, and only where 2^40 exp(d) lies within 2^-11 of a half-integer.  ``slack``
counts such tokens with a margin (2^-9); when it is 0 every mass, sum, cut and draw is exact.  Otherwise Z, every W<=
and every prefix move by at most U = that count, the fp64 cut by at most U + 8 (its product rounds at 2^55), t by at
most U + 1; a draw is flagged when the cut or t lies within 2U + 16 of a boundary.

With ``logit_err`` = e > 0 (the logits known to within e each, e.g. a bf16 model against fp64) a draw is also flagged
when an e-perturbation could change it: greedy with a runner-up within 2e of the maximum; a top-k cut with the k-th
and (k+1)-th values within 2e/T; a top-p group boundary or the draw within eps = exp(4e/T) - 1 of the cut or of the
drawn token's CDF edges (every normalised mass moves by a factor within exp(+-2e/T)).
"""
import math
from typing import NamedTuple

import numpy as np

MASS_SCALE = 2.0 ** 40
MAX_VOCAB = 32768
_HALVES = ((0xD2511F53, 0xCD9E8D57, 0x3C6EF372, 0xA54FF53A, 0x510E527F),
           (0xCD9E8D57, 0xD2511F53, 0x9B05688C, 0x1F83D9AB, 0x5BE0CD19))
_M32 = 0xFFFFFFFF


def _round(x: np.ndarray, c: int, k: int) -> np.ndarray:
    prod = x.astype(np.uint64) * np.uint64(c)
    return ((prod >> np.uint64(32)) ^ (prod & np.uint64(_M32)) ^ np.uint64(k)).astype(np.uint64)


def uniform_bits(seed, b, pos) -> np.ndarray:
    """uint64 bits of the draws (seed, b, pos), broadcast over arrays; seed a uint64 bit pattern (int64 is taken
    modulo 2^64), b and pos taken modulo 2^32 (pos as the device's int32 -> uint32)."""
    seed = np.asarray(seed)
    seed = seed if seed.dtype == np.uint64 else seed.astype(np.int64).astype(np.uint64)
    b = np.asarray(b).astype(np.int64).astype(np.uint64) & np.uint64(_M32)
    pos = np.asarray(pos).astype(np.int64).astype(np.uint64) & np.uint64(_M32)
    with np.errstate(over="ignore"):
        word = ((b * np.uint64(0x9E3779B1) + pos) & np.uint64(_M32)) * np.uint64(0x85EBCA6B) & np.uint64(_M32)
        lo, hi = seed & np.uint64(_M32), seed >> np.uint64(32)
        halves = []
        for ca, cb, k0, k1, k2 in _HALVES:
            x = _round(word ^ lo, ca, k0)
            x = _round(x ^ hi, cb, k1)
            halves.append(_round(x, ca, k2))
    return (halves[1] << np.uint64(32)) | halves[0]


def scaled(logits, temperature: float) -> np.ndarray:
    """x = float32(logit) / float32(temperature) in IEEE fp32."""
    x = np.asarray(logits, dtype=np.float32)
    with np.errstate(over="ignore"):
        return x / np.float32(temperature)


def greedy_token(logits, temperature: float):
    """The token of a row drawn greedily, or None: temperature 0, or a max scaled value of +-inf (no finite mass).
    The first index of the max x (of the max logit when greedy), as torch.argmax."""
    x = np.asarray(logits, dtype=np.float32)
    if temperature != 0:
        x = scaled(x, temperature)
        if np.isfinite(x.max()):
            return None
    return int(np.argmax(x))


class Filtered(NamedTuple):
    x: np.ndarray        # float32 scaled logits
    kept: np.ndarray     # bool: the token survives top-k and top-p
    w: np.ndarray        # uint64 masses of every top-k survivor (0 elsewhere)
    z_kept: int          # Σ w over kept
    cut: int             # top-p cut (-1: top-p off)
    vals: np.ndarray     # the top-k survivors' distinct values, ascending
    W: np.ndarray        # uint64 W<=(vals[g])
    slack: int           # tokens whose mass could round the other way on the device


def filter_row(logits, temperature: float, top_k: int, top_p: float) -> Filtered:
    """The kept set and masses of one row; a greedy row (``greedy_token``) keeps its one token at mass 2^40."""
    tok = greedy_token(logits, temperature)
    if tok is not None:
        x = np.asarray(logits, dtype=np.float32) if temperature == 0 else scaled(logits, temperature)
        kept = np.zeros(x.shape[0], dtype=bool)
        kept[tok] = True
        w = np.where(kept, np.uint64(2 ** 40), np.uint64(0))
        return Filtered(x, kept, w, 2 ** 40, -1, x[tok:tok + 1], np.array([2 ** 40], np.uint64), 0)
    x = scaled(logits, temperature)
    V = x.shape[0]
    m = x.max()
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        kth = np.sort(x)[::-1][top_k - 1]
        keep = x >= kth
    d = x.astype(np.float64) - np.float64(m)
    e = np.exp(d) * MASS_SCALE
    e[d < -29.0] = 0.0
    w = np.where(keep, np.rint(e), 0.0).astype(np.uint64)
    frac = e - np.floor(e)
    slack = int(np.count_nonzero(keep & (d >= -29.0) & (np.abs(frac - 0.5) < 2.0 ** -9)))
    order = np.argsort(x[keep], kind="stable")
    sx, cs = x[keep][order], np.cumsum(w[keep][order], dtype=np.uint64)
    last = np.append(sx[1:] != sx[:-1], True)   # the last token of every tie group (-0 == +0), ascending
    vals, W = sx[last], cs[last]                 # W[g] = W<=(vals[g])
    Z = int(W[-1])
    cut = -1
    if top_p < 1.0:
        cut = math.floor((1.0 - float(np.float32(top_p))) * float(Z))
        over = np.nonzero(W > np.uint64(cut))[0] if cut < Z else []
        keep = keep & (x >= (vals[over[0]] if len(over) else vals[-1]))
    kept_w = np.where(keep, w, np.uint64(0))
    return Filtered(x, keep, w, int(kept_w.sum(dtype=np.uint64)), cut, vals, W, slack)


def probs(logits, temperature: float, top_k: int, top_p: float) -> np.ndarray:
    """fp64 probabilities of the filtered distribution (w / Z_kept; one-hot of the argmax when greedy)."""
    f = filter_row(logits, temperature, top_k, top_p)
    return np.where(f.kept, f.w.astype(np.float64), 0.0) / float(f.z_kept)


class Draw(NamedTuple):
    token: int
    logprob: float
    ambiguous: bool
    why: str


def sample_row(logits, temperature: float, top_k: int, top_p: float, seed: int, b: int, pos: int,
               logit_err: float = 0.0) -> Draw:
    """The device's draw for one row, and whether it is ambiguous (see the module docstring)."""
    logits = np.asarray(logits, dtype=np.float32)
    tok = greedy_token(logits, temperature)
    if tok is not None:
        amb = False
        if temperature == 0 and logit_err > 0 and len(logits) > 1:
            rest = np.delete(logits, tok).astype(np.float64)
            amb = bool(rest.max() >= float(logits[tok]) - 2 * logit_err)
        return Draw(tok, 0.0, amb, "greedy runner-up" if amb else "")
    f = filter_row(logits, temperature, top_k, top_p)
    bits = int(uniform_bits(np.uint64(seed & (2 ** 64 - 1)), b, pos))
    t = (bits * f.z_kept) >> 64
    pre = np.cumsum(np.where(f.kept, f.w, np.uint64(0)), dtype=np.uint64)
    tok = int(np.searchsorted(pre, np.uint64(t), side="right"))
    logprob = float(np.float32(math.log(int(f.w[tok])) - math.log(f.z_kept)))
    lo_edge = int(pre[tok - 1]) if tok > 0 else 0
    hi_edge = int(pre[tok])
    why = []
    if f.slack:
        s = 2 * f.slack + 16
        if f.cut >= 0 and np.any(np.abs(f.W.astype(np.float64) - f.cut) <= s):
            why.append("top-p cut within the mass slack")
        if t - lo_edge <= s or hi_edge - 1 - t <= s:
            why.append("draw within the mass slack")
    if logit_err > 0:
        dx = 2 * logit_err / temperature + 2.0 ** -22 * float(np.abs(f.x).max())
        V = len(logits)
        if 0 < top_k < V:
            srt = np.sort(f.x.astype(np.float64))[::-1]
            if srt[top_k - 1] - srt[top_k] <= dx:
                why.append("top-k cut within the logit error")
        eps = math.expm1(2 * dx)
        if f.cut >= 0 and np.any(np.abs(f.W / float(f.W[-1]) - (1.0 - float(np.float32(top_p)))) <= eps):
            why.append("top-p cut within the logit error")
        u = t / f.z_kept
        if u - lo_edge / f.z_kept <= eps or hi_edge / f.z_kept - u <= eps:
            why.append("draw within the logit error")
    return Draw(tok, logprob, bool(why), "; ".join(why))
