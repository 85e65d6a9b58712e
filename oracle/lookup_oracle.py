"""CPU restatement (Python integers) of the device's prompt-lookup drafts, pcv_prompt_lookup
(perceiver_io_b200/csrc/pcv_lookup.cu), and of the round loop of ``GraphedDecoder.prompt_lookup_generate``.

TEST INFRASTRUCTURE ONLY — nothing under perceiver_io_b200/ imports this file.

    lookup        🤗 PromptLookupCandidateGenerator.get_candidates (no logits processor) on one history: for n =
                  min(N, len - 1) down to 1, the first window equal to the last n ids that ends at or before len - 2;
                  the up to G ids after it, cut before the first EOS id (empty: no draft, no other window), capped at
                  ``limit``
    lookup_rows   the kernel's batched form: row b's history is ids[b, start_b : L_b]; drafts padded to G with the
                  history's last id (0 for an empty history)
    settle        one row's round: the accepted drafts, the next t_0 and the row's new state
    greedy_rounds the round loop at batch 1 on a next-token function, with per-round (drafts offered, accepted)
"""
from typing import Callable, List, NamedTuple, Optional, Sequence, Tuple


def lookup(history: Sequence[int], G: int, N: int, eos: Sequence[int] = (), limit: Optional[int] = None) -> List[int]:
    """The drafts of one history."""
    h = [int(x) for x in history]
    n_ids = len(h)
    for n in range(min(N, n_ids - 1), 0, -1):
        suffix = h[n_ids - n:]
        for e in range(n - 1, n_ids - 1):          # window h[e-n+1 .. e], e <= len - 2
            if h[e - n + 1:e + 1] == suffix:
                draft = h[e + 1:min(e + 1 + G, n_ids)]
                for i, t in enumerate(draft):
                    if t in eos:
                        draft = draft[:i]
                        break
                return draft[:limit] if limit is not None else draft
    return []


def lookup_rows(ids, lengths, G: int, N: int, starts=None, limits=None, eos: Sequence[int] = ()):
    """(drafts (B, G) lists, counts (B,) list) of the kernel's search mode."""
    drafts, counts = [], []
    for b, row in enumerate(ids):
        L = max(0, min(int(lengths[b]), len(row)))
        s = max(0, min(int(starts[b]), L)) if starts is not None else 0
        lim = max(0, min(int(limits[b]), G)) if limits is not None else G
        h = [int(x) for x in row[s:L]]
        d = lookup(h, G, N, eos, lim)
        fill = h[-1] if h else 0
        drafts.append(d + [fill] * (G - len(d)))
        counts.append(len(d))
    return drafts, counts


class Settled(NamedTuple):
    accepted: int        # n_b
    t0: int              # the next t_0
    emitted: List[int]   # the tokens the round emits (empty for a row that is not live)
    unfinished: bool
    left: int


def settle(fed: Sequence[int], draws: Sequence[int], count: int, unfinished: bool, left: int,
           eos: Sequence[int] = ()) -> Settled:
    """One row of a round that fed ``fed`` (t_0, ``count`` drafts, filler) and drew ``draws``."""
    if not (unfinished and left > 0):
        return Settled(0, int(fed[0]), [], unfinished, left)
    n = 0
    while n < count and fed[n + 1] == draws[n]:
        n += 1
    t = int(draws[n])
    return Settled(n, t, [int(x) for x in draws[:n + 1]], unfinished and t not in eos, left - n - 1)


def greedy_rounds(next_tokens: Callable[[List[int]], List[int]], prompt: Sequence[int], n: int, G: int, N: int,
                  eos: Sequence[int] = ()) -> Tuple[List[int], List[Tuple[int, int]]]:
    """The round loop at batch 1: ``next_tokens(seq)`` returns the greedy token after each of seq's last k positions
    (k = len(drafts) + 1 of the round).  Returns (the up to n emitted tokens, per round (drafts offered, accepted))."""
    seq = [int(x) for x in prompt]
    out, rounds = [], []
    while len(out) < n:
        drafts = lookup(seq, G, N, eos, n - len(out) - 1)
        k = len(drafts) + 1
        picks = next_tokens(seq + drafts)[-k:]
        s = settle([seq[-1]] + drafts, picks, len(drafts), True, n - len(out), eos)
        rounds.append((len(drafts), s.accepted))
        out += s.emitted
        seq += s.emitted
        if not s.unfinished:
            break
    return out, rounds
