"""numpy restatement of the device beam step (pcv_beam_step) and of 🤗's ``GenerationMixin._beam_search`` with
``do_sample=False`` and no logits processors, which the step reproduces.

One step of an item (batch entry) with K beams, E EOS ids and ``beams_to_keep`` = max(2, E + 1) * K:
  1. logp = log_softmax(fp32 logits) per beam row, defined as d_i = (double)x_i - (double)max, S = sum exp(d_i) in fp64,
     logp_i = fp32(d_i - log S);
  2. acc = fp32(running_score[beam] + logp); the top beams_to_keep of the K*V values of acc, by score descending and
     flat index (beam * V + token) ascending on ties;
  3. a candidate hits the stopping criteria if its token is an EOS id or it is the n-th generated token;
  4. running beams: hitting candidates get -1e9 (fp32 add); the top K (ties by candidate position) give the next
     tokens, parents and running scores;
  5. finished set: of the first K candidates those that just hit are eligible; scores / fp32(g ** length_penalty)
     (g = the generated length) in fp32, then -1e9 if (early_stopping is True and the item's K finished slots are all
     taken), -1e9 if the early-stop heuristic is satisfied, -1e9 if not eligible; merged with the K finished entries and
     the top K kept, ties by position in [finished | candidates];
  6. the early-stop heuristic (sticky) and the item's "done" flag, as 🤗 computes them.

Flags: a decision is flagged (``Step.flagged[b]``) when the device's fp64 exp / log / pow, or a different fp64 summation
order, could move an fp32 value that enters it (a rounding boundary within reach), or, with ``tie_tol`` > 0 (comparing
against 🤗's fp32 log_softmax), when two scores that are compared lie within ``tie_tol`` of each other.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

MAX_VOCAB = 32768
MAX_BEAMS = 8
MAX_EOS = 4
EARLY_STOPPING = {False: 0, True: 1, "never": 2}
NEG = np.float32(-1e9)


def _moves(v: np.ndarray, r: np.ndarray) -> np.ndarray:
    """True where an fp32 rounding boundary lies within r of the fp64 value v."""
    with np.errstate(invalid="ignore"):
        return np.isfinite(v) & ((v - r).astype(np.float32) != (v + r).astype(np.float32))


def log_softmax(x: np.ndarray):
    """(logp fp32, ambiguous bool) of one row of logits (any float dtype, taken in fp32)."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    m = x.max()
    with np.errstate(invalid="ignore"):
        d = x - m
    S = np.exp(d).sum()
    v = d - np.log(S)
    # reach: the fp64 exp / log error and any summation order (V terms: at most 4V + 16 ulps of S), and the subtraction
    reach = (4.0 * x.shape[0] + 16.0) * 2.0 ** -53 + np.abs(v) * 2.0 ** -50
    return v.astype(np.float32), _moves(v, reach)


def divisor(g: int, length_penalty: float):
    """(fp32(g ** length_penalty), ambiguous): the length-penalty divisor as torch divides an fp32 tensor by it."""
    v = float(g) ** float(length_penalty)
    return np.float32(v), bool(_moves(np.float64(v), np.float64(abs(v) * 2.0 ** -48)))


def fill_value(eos, pad_token_id) -> int:
    """🤗's output_fill_value: ``pad_token_id or eos_token_id[0] if eos_token_id is not None else -1``."""
    eos = list(eos or [])
    return (pad_token_id or eos[0]) if eos else -1


def _top(scores: np.ndarray, k: int) -> np.ndarray:
    """positions of the top k of scores: descending, lowest position first on ties (-0 == +0)."""
    return np.lexsort((np.arange(scores.shape[0]), -scores.astype(np.float64)))[:k]


def _near(vals: np.ndarray, tol: float) -> bool:
    """two of the (sorted descending) real scores within tol of each other."""
    v = vals[vals > -5e8].astype(np.float64)
    return tol > 0 and v.shape[0] > 1 and bool(np.any(np.abs(np.diff(v)) <= tol * np.maximum(1.0, np.abs(v[1:]))))


@dataclass
class State:
    running: np.ndarray    # (B, K) fp32 running scores
    fin: np.ndarray        # (B, K) fp32 finished scores
    fin_flag: np.ndarray   # (B, K) bool
    run_hist: np.ndarray   # (B, K, H) int64
    fin_hist: np.ndarray   # (B, K, H) int64
    unsat: np.ndarray      # (B,) bool: the early-stop heuristic is not satisfied
    done: np.ndarray       # (B,) bool
    gen: int               # tokens generated so far
    n: int                 # max_new_tokens

    @property
    def all_done(self) -> bool:
        return bool(self.done.all())


def init_state(B: int, K: int, n: int, hist_len: int, fill: int) -> State:
    running = np.zeros((B, K), np.float32)
    running[:, 1:] = NEG
    return State(running, np.full((B, K), NEG, np.float32), np.zeros((B, K), bool),
                 np.full((B, K, hist_len), fill, np.int64), np.full((B, K, hist_len), fill, np.int64),
                 np.ones(B, bool), np.zeros(B, bool), 0, n)


def step(st: State, logits: np.ndarray, eos=(), length_penalty: float = 1.0, early_stopping=False,
         tie_tol: float = 0.0):
    """One beam step on logits (B*K, V), in place on st.  Returns (next tokens (B*K,) int64, parents (B*K,) int32 as
    global beam rows b*K + k, flagged (B,) bool)."""
    B, K = st.running.shape
    V = logits.shape[-1]
    E = len(eos)
    btk = max(2, E + 1) * K
    es = EARLY_STOPPING[early_stopping]
    eos_set = set(int(e) for e in eos)
    g = st.gen + 1
    div, amb_div = divisor(g, length_penalty)
    hg = st.n if (es == 2 and length_penalty > 0.0) else g
    hdiv, amb_hdiv = divisor(hg, length_penalty)
    tokens = np.zeros(B * K, np.int64)
    parents = np.zeros(B * K, np.int32)
    flagged = np.zeros(B, bool)
    for b in range(B):
        acc = np.empty(K * V, np.float32)
        amb = np.empty(K * V, bool)
        for k in range(K):
            lp, a = log_softmax(logits[b * K + k])
            acc[k * V:(k + 1) * V] = st.running[b, k] + lp
            amb[k * V:(k + 1) * V] = a
        order = _top(acc, btk + 1)
        cand = order[:btk]
        if amb[order].any() or _near(acc[order], tie_tol):
            flagged[b] = True
        score = acc[cand]
        parent, tok = cand // V, cand % V
        hit = np.array([(int(t) in eos_set) or g >= st.n for t in tok])
        # running beams
        trun = (score + hit.astype(np.float32) * NEG).astype(np.float32)
        sel = _top(trun, K)
        if _near(trun[_top(trun, K + 1)], tie_tol):
            flagged[b] = True
        # finished set (step 5), with the state before this step
        elig = hit & (np.arange(btk) < K)
        s = (score / div).astype(np.float32)
        full = bool(st.fin_flag[b].all()) and es == 1
        s = (s + np.float32(full) * NEG).astype(np.float32)
        s = (s + np.float32(not st.unsat[b]) * NEG).astype(np.float32)
        s = (s + (~elig).astype(np.float32) * NEG).astype(np.float32)
        if elig.any() and amb_div:
            flagged[b] = True
        merged = np.concatenate([st.fin[b], s])
        mflag = np.concatenate([st.fin_flag[b], elig])
        msel = _top(merged, K)
        if _near(merged[_top(merged, K + 1)], tie_tol):
            flagged[b] = True
        cand_hist = st.run_hist[b][parent].copy()
        cand_hist[:, st.gen] = tok
        mhist = np.concatenate([st.fin_hist[b], cand_hist])
        st.fin[b], st.fin_flag[b], st.fin_hist[b] = merged[msel], mflag[msel], mhist[msel]
        st.running[b] = trun[sel]
        st.run_hist[b] = cand_hist[sel]
        tokens[b * K:(b + 1) * K] = tok[sel]
        parents[b * K:(b + 1) * K] = b * K + parent[sel]
        # the early-stop heuristic after this step (step 6)
        best = np.float32(st.running[b, 0] / hdiv)
        worst = np.where(st.fin_flag[b], st.fin[b].min(), NEG).astype(np.float32)
        if amb_hdiv or (tie_tol > 0 and np.any(np.abs(best.astype(np.float64) - worst) <= tie_tol * max(1.0, abs(best)))):
            flagged[b] = True
        st.unsat[b] = st.unsat[b] and bool(np.any(best > worst))
        st.done[b] = (not st.unsat[b]) or (es == 1 and bool(st.fin_flag[b].all()))
    st.gen = g
    return tokens, parents, flagged


def beam_search(logits_fn, B: int, K: int, n: int, eos=(), length_penalty: float = 1.0, early_stopping=False,
                num_return_sequences: int = 1, pad_token_id=None, tie_tol: float = 0.0, stop_early: bool = True):
    """🤗's beam search driven by ``logits_fn(rows)``: rows a list of B*K generated-token lists (beam b*K + k), returns
    (B*K, V) logits.  Returns (sequences (B, R, n) int64, scores (B, R) fp32, flagged: any flagged step, steps run).
    ``stop_early`` stops when every item is done (🤗's loop); the result is the same either way."""
    fill = fill_value(eos, pad_token_id)
    st = init_state(B, K, n, n + 1, fill)
    rows = [[] for _ in range(B * K)]
    flagged = False
    steps = 0
    while st.gen < n:
        tok, par, fl = step(st, np.asarray(logits_fn(rows), np.float32), eos, length_penalty, early_stopping, tie_tol)
        flagged |= bool(fl.any())
        rows = [rows[p] + [int(t)] for p, t in zip(par, tok)]
        steps += 1
        if stop_early and st.all_done:
            break
    R = num_return_sequences
    return st.fin_hist[:, :R, :n].copy(), st.fin[:, :R].copy(), flagged, steps
