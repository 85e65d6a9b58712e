"""numpy restatement of the device logits processors (pcv_logits_process): 🤗's RepetitionPenaltyLogitsProcessor ->
NoRepeatNGramLogitsProcessor -> MinNewTokensLengthLogitsProcessor on one fp32 row and its history (🤗's input_ids row).

fp32 rounding, as torch rounds an fp32 tensor times / over a Python float (the float is taken in fp32 first):
``x * θ`` is fp32(x * fp32(θ)) and ``x / θ`` is fp32(x / fp32(θ)), one correctly rounded operation each;
test_process_cpu pins both against 🤗's class.  Ids outside [0, V) take part in the n-gram matching, but their own
score is never written (🤗 would index out of range there)."""
from __future__ import annotations

import numpy as np

MAX_NGRAM = 8
MAX_EOS = 4


def process(x, hist, repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, prompt_len=0, eos=()):
    """The processed fp32 row of ``x`` (V,) with history ``hist`` (L,) int64."""
    x = np.array(x, dtype=np.float32)
    hist = [int(t) for t in np.asarray(hist, dtype=np.int64).reshape(-1)]
    V, L = x.shape[0], len(hist)
    theta = np.float32(repetition_penalty)
    if theta != np.float32(1.0):
        ids = sorted({t for t in hist if 0 <= t < V})
        for t in ids:
            x[t] = x[t] * theta if x[t] < 0 else x[t] / theta
    N = int(no_repeat_ngram_size)
    if N > 0 and L + 1 >= N:
        suffix = hist[L - N + 1:] if N > 1 else []
        for s in range(L - N + 1):
            if hist[s:s + N - 1] == suffix and 0 <= hist[s + N - 1] < V:
                x[hist[s + N - 1]] = -np.inf
    if min_new_tokens > 0 and L - prompt_len < min_new_tokens:
        for e in eos:
            x[e] = -np.inf
    return x


def process_rows(rows, hists, **kw):
    """``process`` of every row of ``rows`` (R, V) with its history ``hists[r]``."""
    return np.stack([process(r, h, **kw) for r, h in zip(rows, hists)])
