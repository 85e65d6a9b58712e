"""Graph-replayed cached generation of a Perceiver AR ``CausalSequenceModel``: one generated token is one CUDA-graph
replay.

An eager cached step spends most of its time on the host (module code, arena and rotated-shadow bookkeeping, a few
hundred ctypes / ATen launches).  Every length in it changes each token, so it cannot be recorded as it is.
``GraphedDecoder`` keeps the caches in static arenas and the lengths in a few device int32s: per batch row and layer
group the key window ``[begin, end)`` and the new token's row.  The append (``ops.kv_append_at``), the rotary embedding
(``ops.rotary_apply_at``) and the decode attention (``ops.attention_decode_window``) read their rows from there when they
run, and in-graph int32 ops advance them at the end of each step.

    dec = GraphedDecoder(model, batch=B, max_new_tokens=T, kv_cache="bf16")   # or "fp8": e4m3 arenas
    logits = dec.prefill(input_ids, prefix_len, pad_mask=None)                # (B, vocab): eager prompt pass
    logits = dec.step(token_ids)                                              # (B, 1) int64 -> (B, vocab), one replay
    logits = dec.extend(token_ids)                                            # (B, k) int64 -> (B, k, vocab)
    dec.rewind(n)                                                             # drop the last n fed tokens
    dec.rewind(counts)                                                        # drop the last counts[b] of row b
    dec.reorder(beam_idx)                                                     # beam search (eager)
    dec.set_seed(seed); dec.set_sampling(temperature=1.0, top_k=10, top_p=1.0)  # sampling on the device
    first = dec.draw(logits)                                                  # (B, 1): prefill's logits, eager
    tokens = dec.generate(first, n)                                           # (B, n): n replays, no host sync
    tokens, logits = dec.sample(token_ids)                                    # (B, k) drafts -> (B, k) draws
    tokens, q = dec.generate(first, n, logits=True)                           # and the (B, n, vocab) logits drawn from
    out, accepted = dec.verify(token_ids, draft_logits, draft_sampling)       # (B, G+1) -> one speculative round
    tokens, stats = speculative_generate(target, draft, first, n, draft_tokens=G)
    tokens, stats = dec.prompt_lookup_generate(first, n, num_output_tokens=G)   # n-gram drafts from the row's history
    out = dec.beam_search(input_ids, prefix_len, n, num_beams=K)              # batch = B*K: (B, R, n), (B, R)
    tokens = dec.contrastive_search(input_ids, prefix_len, n, penalty_alpha=0.6, top_k=K)   # batch = B*K: (B, n)

Rows: cross-attention arena row r holds token r of the sequence (prompt and generated tokens); self-attention arena
row r holds token ``prefix_len + r`` (prefix_len of the prompt).  The windows follow the 🤗 wrapper's truncation, as
:func:`decode_windows` states it.  ``step`` returns a view of the graph's static logits, valid until the next step.

``extend`` feeds 1 to 64 tokens in one replay of a graph recorded for that count on first use (``step``'s graph for
one token) and returns the logits after each of them: every token attends exactly the keys the one-token loop gives it
(``ops.attention_window`` with a causal band of the group's window width), so speculative decoding can verify k draft
tokens in one replay, keep the accepted prefix and ``rewind`` the rest.  ``rewind(n)`` moves the row counters back by
n tokens with eager int32 ops (no host read, no re-capture); the arena rows past the new end are overwritten later.
Every batch row has its own counters, so ``rewind`` also takes one count per batch row: a batched speculative loop
drops exactly each row's rejected drafts, and the next ``extend`` feeds every row at its own next row (the kernels
read each batch row's bounds; one graph per k serves every pattern of rows).

Budget: ``max_new_tokens`` counts per batch row.  The arenas hold room for the row that has fed the most tokens, so
``extend(k)`` is refused exactly when that row has fewer than k tokens left, and a per-row ``rewind`` gives back what
that row regains.  The counts are host integers; nothing is read back from the device.

Sampling: ``sample`` and ``generate`` replay graphs that also run the device sampler (``ops.sample_tokens``:
temperature, top-k and top-p with the 🤗 warpers' semantics) on the graph's own logits, so a generated token costs one
replay and nothing else.  The sampling values are host values recorded into the graphs (one set of graphs per
``set_sampling`` triple, recorded on first use); the seeds (``set_seed``, one per batch row) and the positions live on
the device.  Counter rule: the token that will be fed at cross-attention arena row p of batch row b is drawn with the
counter (seed_b, b, p).  A replay that feeds k tokens at rows r .. r+k-1 draws at positions r+1 .. r+k, computed in the
graph from the row counters, so after a ``rewind`` the same positions draw the same bits again: a rewound sequence that
is fed the same tokens resamples identically.  ``sample(drafts)`` returns the token drawn after each draft, so
speculative acceptance is ``drafts[:, i+1] == tokens[:, i]`` on the device: the accepted tokens are draws from the
model's own filtered distribution.  ``verify`` and :func:`speculative_generate` use a draft model's probabilities
instead: min(1, p/q) acceptance and a draw from max(0, p - q) on rejection (``ops.spec_verify``), so every emitted token
is distributed as the target's own draw and a draft is accepted with probability Σ min(p, q).

Beam search: ``beam_search`` runs 🤗's ``_beam_search`` (``do_sample=False``, the processors above: EOS ids, length
penalty, ``early_stopping`` and ``num_return_sequences`` as 🤗 takes them) with one replay per token: the replay feeds
the K beams' tokens, runs the device beam step (``ops.beam_step``) on the logits and gathers, by parent, only the arena
rows generated since the prefill (``ops.kv_gather_rows``): every beam of an item was prefilled with the same prompt, so
the prompt rows never move.

Contrastive search: ``contrastive_search`` runs 🤗 4.28's ``contrastive_search`` (``penalty_alpha``, ``top_k``, the
processors above run in fp32 where 4.28 runs them in the model dtype, no warpers) with one replay per token: the replay feeds each item's K candidates on K batch rows,
ranks them on the device by model confidence minus the degeneration penalty, the largest cosine between a candidate's
final hidden row and the item's context of hidden rows (``ops.contrastive_step``), and copies the selected row's newly
appended arena row into the item's other rows (``ops.kv_gather_rows(..., last_rows=1)``): the K rows of an item share
every earlier row, so a step moves one row, whatever its length.  The ranking is fp64 where 🤗 computes in the model
dtype, so on near-ties the two may choose differently.

Logits processors: ``set_sampling``, ``beam_search`` and ``contrastive_search`` take 🤗's ``repetition_penalty``,
``no_repeat_ngram_size`` and ``min_new_tokens``, run in the graph by ``ops.process_logits`` on an fp32 copy of the
logits (the log-softmax for beam search), in the order of 🤗's ``_get_logits_processor`` and before temperature /
top-k / top-p.  A row's history is 🤗's ``input_ids``: the prompt as passed to ``prefill`` and every token fed since,
which each step graph writes into a token arena at its cross-attention row (so ``rewind`` needs nothing and ``reorder``
permutes it).  With ``set_sampling`` EOS ids ``generate`` pads a finished row and stops early, as 🤗's ``_sample``.

Not covered: steps of more than 64 tokens, a different k per batch row, a ring buffer bounded at ``max_seq_len`` (the
arenas grow by ``max_new_tokens`` rows), beam sampling, contrastive search with sampling or a different top_k per item,
per-row sampling or processor values, ``min_length``, bad-words lists, forced tokens, min-p, logits processors under
speculative verification (``verify``, ``speculative_generate``, ``generate(logits=True)`` refuse them), and wiring
into 🤗 ``generate()``.
"""
from __future__ import annotations

import math
import operator
from collections.abc import Sequence
from typing import List, NamedTuple

import torch

from . import modules, ops
from .graphs import GraphedForward
from .utils import Residual

# bounds columns of one batch row and layer group: [window begin, window end, new row, 1, new row, 0]
#   [0:2] the decode window, [2:3] the append row, [2:4] rotary into the rotated-key arena, [4:6] rotary of q
_NCOL = 6


class Window(NamedTuple):
    ca_begin: int    # cross-attention key window [ca_begin, ca_end) in cross-attention arena rows (= token index)
    ca_end: int
    sa_begin: int    # self-attention key window in self-attention arena rows (token index - prompt prefix_len)
    sa_end: int
    prefix_len: int  # the prefix_len an eager cached call of this step passes


def decode_windows(prompt_len: int, prefix_len: int, steps: int, max_seq_len: int, max_latents: int) -> List[Window]:
    """The key windows of ``steps`` one-token cached steps after a prompt of ``prompt_len`` tokens whose first
    ``prefix_len`` are prefix — the truncation of the 🤗 wrapper (``prepare_inputs_for_generation`` and the
    ``_truncate_*_past_key_values`` helpers): before each step the cross-attention cache keeps at most
    ``max_seq_len - 1`` old rows and the self-attention caches at most ``max_latents - 1``, so the prefix grows by one
    token per step once the latents are full.  Each window includes the step's new token (its last row)."""
    out = []
    for s in range(steps):
        ca_end = prompt_len + s + 1
        sa_end = prompt_len - prefix_len + s + 1
        ca_begin, sa_begin = max(0, ca_end - max_seq_len), max(0, sa_end - max_latents)
        out.append(Window(ca_begin, ca_end, sa_begin, sa_end, (ca_end - ca_begin) - (sa_end - sa_begin)))
    return out


def window_positions(pad: torch.Tensor, window: torch.Tensor, cols: torch.Tensor) -> torch.Tensor:
    """(B, 1) int64 absolute position of the last token of the window ``[window[0], window[1])`` of left-padded rows:
    ``positions(b, n, shift)[:, -1:]`` of the eager call, with ``n`` the window length and ``shift`` its padding count,
    computed from tensors alone (no host read).  ``pad`` (B, rows) bytes, non-zero = padding; ``cols`` = arange(rows).
    ``window`` (B, 2): batch row b's own window ``window[b]``."""
    lo, hi = window[..., 0:1], window[..., 1:2]
    inside = (cols >= lo) & (cols < hi)
    shift = ((pad != 0) & inside).sum(dim=1, keepdim=True)
    return (hi - lo - 1 - shift).clamp_min(0).long()


def window_positions_rows(pad: torch.Tensor, bounds: torch.Tensor, cols: torch.Tensor, k: int,
                          width: int) -> torch.Tensor:
    """(B, k) int64 absolute positions of the k tokens of a step whose last token is row ``bounds[1] - 1``: token i at
    row ``r_i = bounds[1] - k + i`` takes :func:`window_positions` of its own one-token window
    ``[max(0, r_i + 1 - width), r_i + 1)``.  Tensors alone, no host read; ``pad`` and ``cols`` as there.  ``bounds``
    (B, >= 2): batch row b's own ``bounds[b]``."""
    r = bounds[..., 1:2] - k + torch.arange(k, device=cols.device, dtype=cols.dtype)
    begin = (r + 1 - width).clamp_min(0)
    inside = (cols >= begin[..., None]) & (cols <= r[..., None])
    shift = ((pad != 0)[:, None, :] & inside).sum(dim=2)
    return (r - begin - shift).clamp_min(0).long()


def extend_bounds(bounds: torch.Tensor, k: int) -> torch.Tensor:
    """The (groups, 6) int32 bounds of a k-token step from the one-token state ``bounds`` (``[begin, end, row, 1, row,
    0]`` per layer group, end = row + 1): the window's end moves to the last token's row + 1, everything else stays —
    the window starts at the first token's begin, appends and rotations start at its row.  (B, groups, 6) per-row
    states move every batch row the same way."""
    out = bounds.clone()
    out[..., 1] += k - 1
    return out


def advance_bounds_(bounds: torch.Tensor, inc: torch.Tensor, wmax: torch.Tensor, n) -> torch.Tensor:
    """Move the one-token state ``bounds`` by n tokens in place (n < 0 rewinds): row and end += n, begin = max(0,
    end - the group's window width ``wmax``).  ``inc`` is ``[0, 1, 1, 0, 1, 0]``.  ``n`` an integer moves every row;
    a (B,) int32 tensor on ``bounds``' device moves batch row b of a (B, groups, 6) state by ``n[b]``."""
    if isinstance(n, torch.Tensor):
        bounds.add_(inc * n[:, None, None])
    else:
        bounds.add_(inc, alpha=n)
    bounds[..., 0].copy_((bounds[..., 1] - wmax).clamp_min_(0))
    return bounds


def sample_positions(bounds: torch.Tensor, steps: torch.Tensor, k: int) -> torch.Tensor:
    """(B, k) int32 counters of the draws of a k-token replay from the one-token state ``bounds`` (B, groups, 6) before
    the replay: the tokens fed at cross-attention rows r .. r+k-1 (r = ``bounds[b, 0, 2]``) are followed by draws at
    positions r+1 .. r+k.  ``steps`` is ``arange(1, 65)`` int32 on ``bounds``' device.  Tensors alone, no host read."""
    return bounds[:, 0, 2:3] + steps[:k]


def _triple(vals):
    if not isinstance(vals, (tuple, list)) or len(vals) != 3:
        raise ValueError(f"GraphedDecoder.verify: draft_sampling must be a (temperature, top_k, top_p) triple, got "
                         f"{vals!r}")
    return vals


def _as_count(x):
    """x as an int when it is integer-like (operator.index) and not a bool, else None."""
    if isinstance(x, bool):
        return None
    try:
        return operator.index(x)
    except TypeError:
        return None


def _sampling_triple(what: str, temperature, top_k, top_p):
    """(temperature, top_k, top_p) checked as ``ops.sample_tokens`` takes them (top_k clamped to int32)."""
    t, p, k = float(temperature), float(top_p), _as_count(top_k)
    if not t >= 0.0 or math.isinf(t):
        raise ValueError(f"{what}: temperature must be finite and >= 0 (0: greedy), got {temperature!r}")
    if k is None or k < 0:
        raise ValueError(f"{what}: top_k must be an integer >= 0 (0: off), got {top_k!r}")
    if not 0.0 < p <= 1.0:
        raise ValueError(f"{what}: top_p must be in (0, 1] (1: off), got {top_p!r}")
    return t, min(k, 2 ** 31 - 1), p


_NO_PROCESS = (1.0, 0, 0)   # (repetition_penalty, no_repeat_ngram_size, min_new_tokens) with every processor off


def _process_values(what: str, repetition_penalty, no_repeat_ngram_size, min_new_tokens, eos):
    """(θ, N, M) checked as ``ops.process_logits`` takes them; M > 0 needs EOS ids (🤗 drops the processor silently
    there; this refuses)."""
    t, n, m = repetition_penalty, _as_count(no_repeat_ngram_size), _as_count(min_new_tokens)
    # the kernel takes θ in fp32: it must stay finite and > 0 there
    t32 = float(torch.tensor(float(t), dtype=torch.float32)) if isinstance(t, (int, float)) else math.nan
    if isinstance(t, bool) or not isinstance(t, (int, float)) or not math.isfinite(t32) or not t32 > 0:
        raise ValueError(f"{what}: repetition_penalty must be a number > 0 that is finite and > 0 in fp32 (1: off), got "
                         f"{repetition_penalty!r}")
    if n is None or not 0 <= n <= ops.PROCESS_MAX_NGRAM:
        raise ValueError(f"{what}: no_repeat_ngram_size must be an integer in [0, {ops.PROCESS_MAX_NGRAM}] (0: off), got "
                         f"{no_repeat_ngram_size!r}")
    if m is None or not 0 <= m < 2 ** 31:
        raise ValueError(f"{what}: min_new_tokens must be an integer >= 0 (0: off), got {min_new_tokens!r}")
    if m > 0 and not eos:
        raise ValueError(f"{what}: min_new_tokens={m} needs eos_token_id (it bans the EOS ids until {m} tokens are new)")
    if len(eos) > ops.PROCESS_MAX_EOS:
        raise ValueError(f"{what}: at most {ops.PROCESS_MAX_EOS} EOS ids, got {len(eos)}")
    return float(t), n, m


class BeamSearchOutput(NamedTuple):
    sequences: torch.Tensor   # (B, R, n) int64 generated tokens, the output fill value after a hypothesis's end
    scores: torch.Tensor      # (B, R) fp32, 🤗's sequences_scores


def _eos_ids(eos_token_id, what: str = "GraphedDecoder.beam_search") -> List[int]:
    if eos_token_id is None:
        return []
    ids = [eos_token_id] if _as_count(eos_token_id) is not None else eos_token_id
    if isinstance(ids, torch.Tensor):
        ids = ids.flatten().tolist()
    if not isinstance(ids, Sequence) or isinstance(ids, (str, bytes)) or any(_as_count(e) is None for e in ids):
        raise ValueError(f"{what}: eos_token_id must be None, an integer or a list of integers, got "
                         f"{eos_token_id!r}")
    return [_as_count(e) for e in ids]


class _Attn:
    """Static state of one attention layer: arenas, rotated-key arena, scales."""

    def __init__(self, owner, group: int, rotary: bool, norms, key: str):
        self.owner, self.mha, self.group, self.rotary, self.norms, self.key = owner, owner.attention, group, rotary, norms, key
        self.K = self.V = self.S = None
        self.kv8 = self.k_inv_h = None


class GraphedDecoder:
    # per-row counts: None while every batch row has fed the same tokens, else _lag[b] = the tokens row b has fed fewer
    # than the furthest row (whose count is _fed)
    _lag = None
    _seeds = None   # (B,) int64 sampler seeds, set in __init__
    _draft_sampling = (1.0, 0, 1.0)   # the draft's values of the verify graph being recorded or replayed
    _beam_state = None                # ops.BeamState of the last beam_search
    _beam_table = None                # ops.KvGatherTable of the last beam_search (its scratch is reused)
    _cs_state = None                  # ops.ContrastiveState of the last contrastive_search
    _cs_table = None                  # ops.KvGatherTable of the last contrastive_search (its scratch is reused)
    _hidden = None                    # the final hidden rows (B, k, D) of the last _step_fn call
    _tokens = None                    # (B, n0 + max_new_tokens) int64: the prompt and every fed token, by arena row
    _process = _NO_PROCESS            # the sampling graphs' (repetition_penalty, no_repeat_ngram_size, min_new_tokens)
    _eos = ()                         # the sampling EOS ids, and the token fed after one
    _pad_token = None
    _lookup_state = ()                # prompt lookup: (next t_0 and drafts (B, 64), state (4, B), start (B,)) buffers
    _lookup_args = (0, 0)             # the (G, N) of the lookup graph being recorded or replayed

    def __init__(self, model, batch: int, max_new_tokens: int, kv_cache: str = "bf16"):
        if max_new_tokens < 1:
            raise ValueError(f"GraphedDecoder: max_new_tokens must be >= 1, got {max_new_tokens}")
        if batch < 1:
            raise ValueError(f"GraphedDecoder: batch must be >= 1, got {batch}")
        if kv_cache not in ("bf16", "fp8"):
            raise ValueError(f"GraphedDecoder: kv_cache must be 'bf16' or 'fp8', got {kv_cache!r}")
        if not isinstance(model, modules.CausalSequenceModel):
            raise TypeError("GraphedDecoder covers this package's CausalSequenceModel")
        if model.training:
            raise RuntimeError("GraphedDecoder is inference-only: put the model in eval mode")
        w = model.input_adapter.txt_embedding.weight
        if not w.is_cuda:
            raise RuntimeError(f"GraphedDecoder runs on CUDA (sm_90a); the model is on {w.device}")
        if w.dtype not in (torch.bfloat16, torch.float16):
            raise RuntimeError(f"GraphedDecoder needs a bf16 / fp16 model, got {w.dtype}")
        inv_freq = getattr(getattr(model.input_adapter, "frq_pos_encoding", None), "inv_freq", None)
        if inv_freq is None:
            raise RuntimeError("GraphedDecoder needs the rotary frequency table (inv_freq) of this package's adapter")
        H = model.cross_attention[0].module.attention.num_heads
        mult = 16 if kv_cache == "fp8" else 8
        for m in model.modules():
            if isinstance(m, modules.MultiHeadAttention):
                dqk, dv = m.num_qk_channels // m.num_heads, m.num_v_channels // m.num_heads
                if dqk % mult or dv % mult or dqk > 256 or dv > 256:
                    raise RuntimeError(f"GraphedDecoder: head dims ({dqk}, {dv}) must be multiples of {mult} and <= 256 "
                                       f"for the {kv_cache} cache")
        self.model, self.batch, self.max_new_tokens, self.kv_cache = model, batch, max_new_tokens, kv_cache
        self.fp8 = kv_cache == "fp8"
        self.num_heads = H
        self.inv_freq = inv_freq
        self.device = w.device
        self.dtype = w.dtype
        self.captures = 0
        self._graphs = {}      # tokens per step, or ("sample", tokens per step, sampling values) -> GraphedForward
        self._seeds = torch.zeros(batch, dtype=torch.int64, device=w.device)
        self._seeded = False
        self._sampling = (1.0, 0, 1.0)
        self._steps = torch.arange(1, ops.WINDOW_MAX_ROWS + 1, dtype=torch.int32, device=w.device)
        self._bounds = None
        self._remaining = 0
        self._fed = 0          # tokens fed since prefill (what rewind may drop)
        sa = model.self_attention
        nrot = sa.num_rotary_layers
        ca = model.cross_attention[0].module
        self._layers = [_Attn(ca, 0, True, (ca.kv_norm, ca.q_norm), "min_rows")]
        for idx, layer in enumerate(sa):
            self._layers.append(_Attn(layer[0].module, 1, nrot == -1 or idx < nrot, (layer[0].module.norm,),
                                      "min_rows_latent"))

    # ---- prompt ------------------------------------------------------------------------------------------------------
    def prefill(self, input_ids: torch.Tensor, prefix_len: int, pad_mask=None) -> torch.Tensor:
        """Run the prompt through the eager model (``kv_cache=[]``), load its caches and rotated keys into the arenas
        and return the last position's logits (B, vocab).  Resets the step budget to ``max_new_tokens``."""
        return self._prefill(input_ids, prefix_len, pad_mask).logits[:, -1]

    def _prefill(self, input_ids: torch.Tensor, prefix_len: int, pad_mask=None):
        """``prefill``, returning the prompt pass's whole output (its ``last_hidden_state`` included)."""
        m, T = self.model, self.max_new_tokens
        B, n0 = input_ids.shape
        if B != self.batch:
            raise ValueError(f"GraphedDecoder: batch {B} != {self.batch}")
        old = modules.fp8_config["kv_cache"]
        modules.fp8_config["kv_cache"] = self.fp8
        try:
            with torch.no_grad():
                out = m(input_ids, prefix_len=prefix_len, pad_mask=pad_mask, kv_cache=[])
        finally:
            modules.fp8_config["kv_cache"] = old
        caches = out.kv_cache
        caps = (n0 + T, n0 - prefix_len + T)
        dev = self.device
        self._table = ops.rotary_angle_table(self.inv_freq, caps[0])
        rotate_dim = self._table.shape[1]
        for a, (k, v) in zip(self._layers, caches):
            if self.fp8 and (k.dtype != ops.F8 or v.dtype != ops.F8):
                raise RuntimeError("GraphedDecoder: the prompt pass did not produce an e4m3 cache (call not covered)")
            cap, L = caps[a.group], k.shape[1]
            a.K = torch.zeros(B, cap, k.shape[2], dtype=k.dtype, device=dev)
            a.V = torch.zeros(B, cap, v.shape[2], dtype=v.dtype, device=dev)
            a.K[:, :L].copy_(k)
            a.V[:, :L].copy_(v)
            a.table = self._table[:cap]
            if a.rotary:
                hit = ops.rotated_cache_shadow(k)
                if hit is None or hit[1] != 0:
                    raise RuntimeError("GraphedDecoder: the prompt pass left no rotated-key shadow at position 0")
                a.S = torch.zeros_like(a.K)
                a.S[:, :L].copy_(hit[0])
            if self.fp8:
                a.kv8 = modules._kv8_scales(a.owner, a.norms, rotate_dim if a.rotary else 0)
                a.k_inv_h = 1.0 / a.kv8.k_descale.float().contiguous()
        self._tokens = torch.zeros(B, caps[0], dtype=torch.int64, device=dev)
        self._tokens[:, :n0].copy_(input_ids)
        self._n0 = n0
        self._unfinished = torch.ones(B, 1, dtype=torch.bool, device=dev)
        self._pad = torch.zeros(B, caps[0], dtype=torch.uint8, device=dev)
        if pad_mask is not None:
            self._pad[:, :n0].copy_(pad_mask != 0)
        self._cols = torch.arange(caps[0], device=dev, dtype=torch.int32)
        w = decode_windows(n0, prefix_len, 1, m.max_seq_len, m.max_latents)[0]
        rows = (n0, n0 - prefix_len)
        self._bounds = torch.tensor([[w.ca_begin, w.ca_end, rows[0], 1, rows[0], 0],
                                     [w.sa_begin, w.sa_end, rows[1], 1, rows[1], 0]],
                                    dtype=torch.int32, device=dev).repeat(B, 1, 1)   # (B, groups, 6): per batch row
        self._inc = torch.tensor([0, 1, 1, 0, 1, 0], dtype=torch.int32, device=dev)
        self._wmax = torch.tensor([m.max_seq_len, m.max_latents], dtype=torch.int32, device=dev)
        self._width = (m.max_seq_len, m.max_latents)
        self._graphs = {}
        self._remaining = T
        self._fed = 0
        self._lag = None
        return out

    # ---- one step of 1 to 64 tokens ----------------------------------------------------------------------------------
    def _attend(self, a: _Attn, bounds, q, k, v):
        H, g = a.mha.num_heads, bounds[:, a.group]   # (B, 6): every batch row's own rows
        fp8 = self.fp8
        ops.kv_append_at(a.K, a.V, k, v, g[:, 2:3], *((a.kv8.k_inv, a.kv8.v_inv) if fp8 else ()))
        keys = a.K
        if a.rotary:   # the new key into the rotated-key arena, q at the new token's row
            ops.rotary_apply_at(k, H, a.table, g[:, 2:4], a.S, a.k_inv_h)
            q = ops.rotary_apply_at(q, H, a.table, g[:, 4:6], torch.empty(q.shape, dtype=q.dtype, device=q.device))
            keys = a.S
        kw = dict(pad_mask=self._pad if a.group == 0 else None, causal=a.mha.causal_attention,
                  k_descale=a.kv8.k_descale if fp8 else None, v_descale=a.kv8.v_descale if fp8 else None)
        if q.shape[1] == 1:
            o = ops.attention_decode_window(q, keys, a.V, g[:, 0:2], H, a.mha.dp_scale, **kw)
        else:   # every token sees its own one-token window: a causal band of the group's window width
            o = ops.attention_window(q, keys, a.V, g[:, 0:2], H, a.mha.dp_scale, band=self._width[a.group], **kw)
        return modules.fused_linear(a.mha, "_pcv_o_fold", None, a.mha.o_proj, o, a.key)

    @staticmethod
    def _residual(block, y, x):
        return block.dropout(y) + x if isinstance(block, Residual) else y

    def _step_fn(self, token: torch.Tensor) -> torch.Tensor:
        m = self.model
        adapter = m.input_adapter
        k = token.shape[1]
        b = self._bounds if k == 1 else extend_bounds(self._bounds, k)
        # the token history: each fed token at its cross-attention row (clamped: warm-up calls may run past the arena,
        # and every row at or past the current one is written again before it is read)
        rows = b[:, 0, 2:3] if k == 1 else b[:, 0, 2:3] + (self._steps[:k] - 1)
        self._tokens.scatter_(1, rows.clamp_max(self._tokens.shape[1] - 1).long(), token)
        x = adapter.txt_embedding(token)
        if getattr(adapter, "_abs_pos_emb", False):
            pos = (window_positions(self._pad, b[:, 0, 0:2], self._cols) if k == 1
                   else window_positions_rows(self._pad, b[:, 0], self._cols, k, self._width[0]))
            x = x + adapter.pos_embedding(pos)
        # cross-attention (cached: the keys of this token are its own q_norm'd row, reference modules.py:222-224)
        ca_layer, ca = m.cross_attention, self._layers[0].owner
        xq = ca.q_norm(x)
        a = ca.attention
        h = self._residual(ca_layer[0], self._attend(self._layers[0], b, a.q_proj(xq), a.k_proj(xq), a.v_proj(xq)), x)
        h = ca_layer[1](h).last_hidden_state
        for layer, st in zip(m.self_attention, self._layers[1:]):
            sa = st.owner
            qkv = modules.project_qkv(sa, h)
            if qkv is None:
                xn = sa.norm(h)
                qkv = sa.attention.q_proj(xn), sa.attention.k_proj(xn), sa.attention.v_proj(xn)
            h = self._residual(layer[0], self._attend(st, b, *qkv), h)
            h = layer[1](h).last_hidden_state
        if m.config.output_norm:
            h = m.out_norm(h)
        self._hidden = h   # the final hidden rows, for contrastive search (no work of its own)
        logits = m.output_adapter(h, txt_embedding=adapter.txt_embedding)
        # the next step's rows and windows: row += k, end += k, begin = max(0, end - window limit)
        advance_bounds_(self._bounds, self._inc, self._wmax, k)
        return logits[:, -1] if k == 1 else logits

    def _sample_fn(self, token: torch.Tensor):
        """_step_fn followed by the sampler on its logits: (tokens (B, k), logits (B, k, vocab))."""
        k = token.shape[1]
        pos = sample_positions(self._bounds, self._steps, k)   # before _step_fn advances the rows
        logits = self._step_fn(token)
        if k == 1:
            logits = logits[:, None]
        logits = self._processed(logits, pos)
        t, top_k, top_p = self._sampling
        return ops.sample_tokens(logits, self._seeds, pos, t, top_k, top_p), logits

    def _processed(self, logits: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        """``logits`` (B, k, V) through the ``set_sampling`` processors (fp32), or as they are when every one is off.
        The draw at position p sees the history's first p tokens (🤗's input_ids at that draw)."""
        if self._process == _NO_PROCESS:
            return logits
        B, k, V = logits.shape
        theta, N, M = self._process
        return ops.process_logits(logits.reshape(B * k, V), self._tokens, pos.reshape(-1), rows_per_hist=k,
                                  repetition_penalty=theta, no_repeat_ngram_size=N, min_new_tokens=M,
                                  prompt_len=self._n0, eos=self._eos).view(B, k, V)

    def _generate_fn(self, token: torch.Tensor):
        """_sample_fn with 🤗 ``_sample``'s EOS rule: a finished row's draw is replaced by the pad token."""
        tokens, logits = self._sample_fn(token)
        tokens = torch.where(self._unfinished, tokens, self._pad_token)
        self._unfinished &= ~self._is_eos(tokens)
        return tokens, logits

    def _is_eos(self, tokens: torch.Tensor) -> torch.Tensor:
        hit = tokens == self._eos[0]
        for e in self._eos[1:]:
            hit |= tokens == e
        return hit

    def _verify_fn(self, token: torch.Tensor, draft_logits: torch.Tensor):
        """_step_fn followed by ``ops.spec_verify`` on its logits: (tokens (B, k), accepted (B,))."""
        pos = sample_positions(self._bounds, self._steps, token.shape[1])   # before _step_fn advances the rows
        logits = self._step_fn(token)
        self._verify_logits = logits   # the static target logits of the verify graph recorded last (for tests)
        return ops.spec_verify(logits, draft_logits, token, self._seeds, pos, self._sampling, self._draft_sampling)

    def _lookup_fn(self, token: torch.Tensor) -> torch.Tensor:
        """_sample_fn followed by the round mode of ``ops.prompt_lookup``: settle the round, write the next t_0 and
        search the next drafts (into ``_lookup_state``).  Returns the draws (B, k)."""
        k = token.shape[1]
        tokens, _ = self._sample_fn(token)
        tokens = tokens.contiguous()
        nxt, state, start = self._lookup_state
        G, N = self._lookup_args
        # after _step_fn, bounds[:, 0, 2] is t_0's row + k; t_0's successor goes to row + n_b + 1 = L_b - 1
        ops.prompt_lookup_round(self._tokens, self._bounds[:, 0, 2], 2 - k, token, tokens, nxt, state, G, N,
                                start=start, eos=self._eos)
        return tokens

    def _replay(self, token_ids: torch.Tensor, fn: str, *extra: torch.Tensor) -> torch.Tensor:
        """One replay of the graph of ``token_ids.shape[1]`` tokens per step, recorded on first use (``fn`` "sample":
        the graph that also samples, one per sampling triple; "verify": the graph that also verifies drafts, one per
        pair of sampling triples, with ``extra`` its draft logits)."""
        k = token_ids.shape[1] if token_ids.dim() == 2 else 0
        kmax = 1 if fn in ("step", "generate") else ops.WINDOW_MAX_ROWS
        if self._bounds is None:
            raise RuntimeError("GraphedDecoder: call prefill() first")
        if tuple(token_ids.shape) != (self.batch, k) or token_ids.dtype != torch.long or not 1 <= k <= kmax:
            want = "1)" if kmax == 1 else f"k) with 1 <= k <= {ops.WINDOW_MAX_ROWS}"
            raise ValueError(f"GraphedDecoder.{fn} takes ({self.batch}, {want} int64 tokens, got "
                             f"{tuple(token_ids.shape)} {token_ids.dtype}")
        if self._remaining < k:
            raise RuntimeError(f"GraphedDecoder: {self._remaining} of max_new_tokens={self.max_new_tokens} tokens remain "
                               f"to the furthest batch row (the arenas hold no room for {k} more); rewind, or call "
                               f"prefill() again")
        if torch.is_autocast_enabled():
            raise RuntimeError("GraphedDecoder does not run under autocast")
        sample = fn in ("sample", "generate")
        key = ("sample", k, self._sampling) if sample else k
        if sample and self._process != _NO_PROCESS:
            key += (self._process, self._eos)
        fwd = self._sample_fn if sample else self._step_fn
        if fn == "generate" and self._eos:
            key, fwd = ("generate", self._sampling, self._process, self._eos, self._pad_token), self._generate_fn
        if fn == "verify":
            key, fwd = ("verify", k, self._sampling, self._draft_sampling), self._verify_fn
        if fn == "lookup":
            key, fwd = ("lookup", k, self._sampling, self._process, self._eos, self._lookup_args), self._lookup_fn
        graph = self._graphs.get(key)
        if graph is None:
            snapshot = self._bounds.clone()   # the warm-up calls advance the rows; their arena writes are rewritten later
            unfinished = self._unfinished.clone()   # and may finish rows of the generate graph
            lookup = [t.clone() for t in self._lookup_state] if fn == "lookup" else []   # and settle lookup rounds
            old = torch.cuda.get_sync_debug_mode()
            torch.cuda.set_sync_debug_mode(0)  # recording a graph synchronises the device once
            try:
                graph = GraphedForward(fwd, token_ids, *extra)
            finally:
                torch.cuda.set_sync_debug_mode(old)
            self._bounds.copy_(snapshot)
            self._unfinished.copy_(unfinished)
            for t, saved in zip(self._lookup_state, lookup):
                t.copy_(saved)
            self._graphs[key] = graph
            self.captures += 1
        out = graph(token_ids, *extra)
        self._remaining -= k
        self._fed += k
        return out

    def step(self, token_ids: torch.Tensor) -> torch.Tensor:
        """Append the tokens ``token_ids`` (B, 1) int64 and return the next logits (B, vocab) — one graph replay (the
        first call records the graph).  A view of the graph's static output, valid until the next step."""
        return self._replay(token_ids, "step")

    def extend(self, token_ids: torch.Tensor) -> torch.Tensor:
        """Append the k tokens ``token_ids`` (B, k) int64, 1 <= k <= 64, and return the logits after each of them (B, k,
        vocab) — one replay of the graph recorded for k on first use (k = 1 shares ``step``'s graph).  Token i sees
        exactly the keys it would see had the k tokens been fed by k ``step`` calls.  Consumes k tokens of the
        budget.  A view of the graph's static output, valid until the next step."""
        if token_ids.dim() == 2 and token_ids.shape[1] == 1:
            return self._replay(token_ids, "extend")[:, None]
        return self._replay(token_ids, "extend")

    # ---- sampling ------------------------------------------------------------------------------------------------
    def set_seed(self, seed) -> None:
        """Load the per-batch-row seeds of the sampler: one integer for every row, or B integers (each in [0, 2^64)).
        An eager copy into the graphs' seed buffer: no re-capture.  Without a call, the first sampling call draws one
        seed from torch's CPU generator (``ops.new_dropout_seed``)."""
        seeds = [seed] * self.batch if _as_count(seed) is not None else seed
        if isinstance(seeds, torch.Tensor):
            seeds = seeds.tolist() if not seeds.is_cuda and seeds.dim() == 1 else None
        if not isinstance(seeds, Sequence) or isinstance(seeds, (str, bytes)) or len(seeds) != self.batch:
            raise ValueError(f"GraphedDecoder.set_seed: one integer or {self.batch} integers (one per batch row), got "
                             f"{seed!r}")
        vals = []
        for b, s in enumerate(seeds):
            v = _as_count(s)
            if v is None or not 0 <= v < 2 ** 64:
                raise ValueError(f"GraphedDecoder.set_seed: the seed of batch row {b} must be an integer in [0, 2^64), "
                                 f"got {s!r}")
            vals.append(v - 2 ** 64 if v >= 2 ** 63 else v)   # the uint64 bit pattern in an int64
        host = torch.tensor(vals, dtype=torch.int64)
        if self._seeds.is_cuda:   # pinned and asynchronous: no synchronisation
            host = host.pin_memory()
        self._seeds.copy_(host, non_blocking=True)
        self._seeded = True

    def set_sampling(self, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0, *,
                     repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0, min_new_tokens: int = 0,
                     eos_token_id=None, pad_token_id=None) -> None:
        """The sampler's values for ``draw``, ``sample`` and ``generate``: ``temperature`` >= 0 (0: greedy), ``top_k`` >= 0
        (0: off), ``top_p`` in (0, 1] (1: off), as ``ops.sample_tokens`` takes them.

        Before them, 🤗's logits processors run on an fp32 copy of the logits (``ops.process_logits``), in the order of
        🤗's ``_get_logits_processor``: ``repetition_penalty`` θ > 0 (1: off), ``no_repeat_ngram_size`` N in [0, 8] (0:
        off) and ``min_new_tokens`` M >= 0 (0: off; needs ``eos_token_id``), counted from the prompt's padded width.  A
        row's history is the prompt as passed to ``prefill`` and every token fed to that row since (the draw at the row
        a token will take sees every earlier row).  ``eos_token_id`` (an id or a list) also makes ``generate`` stop:
        see there; ``pad_token_id`` is what a finished row is fed (None: the first EOS id).  The first replay under
        new values records their graphs; with every processor off and no EOS ids the graphs are the plain sampling
        ones.  Invalid values are refused with the reason, leaving the old values in place."""
        what = "GraphedDecoder.set_sampling"
        sampling = _sampling_triple(what, temperature, top_k, top_p)
        eos = tuple(_eos_ids(eos_token_id, what))
        process = _process_values(what, repetition_penalty, no_repeat_ngram_size, min_new_tokens, eos)
        vocab = self.model.config.vocab_size
        if any(not 0 <= e < vocab for e in eos):
            raise ValueError(f"{what}: every EOS id must be in [0, {vocab}), got {list(eos)}")
        pad = None
        if eos:
            pad = eos[0] if pad_token_id is None else _as_count(pad_token_id)
            if pad is None or not 0 <= pad < vocab:
                raise ValueError(f"{what}: pad_token_id must be None or an id in [0, {vocab}) (it is fed after an EOS), "
                                 f"got {pad_token_id!r}")
        self._sampling, self._process, self._eos, self._pad_token = sampling, process, eos, pad

    def _ready_to_sample(self, what: str) -> None:
        if self._bounds is None:
            raise RuntimeError("GraphedDecoder: call prefill() first")
        vocab = self.model.config.vocab_size
        if vocab > ops.SAMPLE_MAX_VOCAB:
            raise RuntimeError(f"GraphedDecoder.{what}: the device sampler takes vocabularies up to "
                               f"{ops.SAMPLE_MAX_VOCAB}, this model has {vocab}")
        if not self._seeded:
            self.set_seed(ops.new_dropout_seed())

    def draw(self, logits: torch.Tensor) -> torch.Tensor:
        """(B, 1) int64 tokens drawn, eagerly, from ``logits`` (B, vocab) — typically ``prefill``'s — at each batch row's
        next position (the row its next fed token takes)."""
        self._ready_to_sample("draw")
        if logits.dim() != 2 or logits.shape[0] != self.batch:
            raise ValueError(f"GraphedDecoder.draw takes ({self.batch}, vocab) logits, got {tuple(logits.shape)}")
        t, top_k, top_p = self._sampling
        pos = sample_positions(self._bounds, self._steps, 1) - 1
        return ops.sample_tokens(self._processed(logits[:, None], pos), self._seeds, pos, t, top_k, top_p)

    def sample(self, token_ids: torch.Tensor):
        """Feed the k tokens ``token_ids`` (B, k) int64, 1 <= k <= 64, in one replay and return ``(tokens, logits)``:
        ``tokens[:, i]`` (B, k) int64 is drawn on the device from ``logits[:, i]`` (B, k, vocab), the logits after token
        i, at the position of the row it would be fed at.  Consumes k tokens of the budget.  Views of the graph's static
        outputs, valid until the next replay."""
        self._ready_to_sample("sample")
        return self._replay(token_ids, "sample")

    def generate(self, first_tokens: torch.Tensor, n: int, logits: bool = False, check_every: int = 16):
        """Feed ``first_tokens`` (B, 1) int64 and then every drawn token, for n replays of the one-token sampling graph;
        return the n drawn tokens (B, n) int64.  Each replay's input is copied on the device from the previous one's
        output: no host read and no synchronisation.  Consumes n tokens of the budget; asking for more than remain is
        refused before any replay, leaving the state untouched.  With ``logits=True`` also return the logits each token
        was drawn from, (B, n, vocab), copied on the device after each replay (a draft model's probabilities for
        :meth:`verify`; refused while a ``set_sampling`` processor is on).

        With ``set_sampling`` EOS ids, 🤗 ``_sample``'s rule: a row that has emitted an EOS id (``first_tokens``
        included) is fed, and returns, the pad token from then on; the device's "every row finished" flag is read
        every ``check_every`` replays and the loop stops once it is set.  The output stays (B, n), padded; replays not
        run stay in the budget."""
        self._ready_to_sample("generate")
        count, every = _as_count(n), _as_count(check_every)
        if count is None or count < 1:
            raise ValueError(f"GraphedDecoder.generate: n must be an integer >= 1, got {n!r}")
        if every is None or every < 1:
            raise ValueError(f"GraphedDecoder.generate: check_every must be an integer >= 1, got {check_every!r}")
        if logits and self._process != _NO_PROCESS:
            raise ValueError("GraphedDecoder.generate: logits=True (a draft's distribution for verify) is not covered "
                             "with logits processors on")
        if self._remaining < count:
            raise RuntimeError(f"GraphedDecoder.generate: {self._remaining} of max_new_tokens={self.max_new_tokens} "
                               f"tokens remain to the furthest batch row, {count} asked for")
        if tuple(first_tokens.shape) != (self.batch, 1) or first_tokens.dtype != torch.long:
            raise ValueError(f"GraphedDecoder.generate takes ({self.batch}, 1) int64 first tokens, got "
                             f"{tuple(first_tokens.shape)} {first_tokens.dtype}")
        if self._eos:
            out = torch.full((self.batch, count), self._pad_token, dtype=torch.long, device=self.device)
            torch.logical_not(self._is_eos(first_tokens), out=self._unfinished)
        else:
            out = torch.empty(self.batch, count, dtype=torch.long, device=self.device)
        kept = None
        tokens = first_tokens
        for i in range(count):
            tokens, lg = self._replay(tokens, "generate")
            out[:, i:i + 1].copy_(tokens)
            if logits:
                if kept is None:
                    kept = torch.empty(self.batch, count, lg.shape[-1], dtype=lg.dtype, device=self.device)
                kept[:, i:i + 1].copy_(lg)
            if self._eos and (i + 1) % every == 0 and i + 1 < count:
                old = torch.cuda.get_sync_debug_mode()
                torch.cuda.set_sync_debug_mode(0)
                try:
                    stop = not bool(self._unfinished.any().item())   # the one host read: every row finished
                finally:
                    torch.cuda.set_sync_debug_mode(old)
                if stop:
                    break
        return (out, kept) if logits else out

    def verify(self, token_ids: torch.Tensor, draft_logits: torch.Tensor, draft_sampling=(1.0, 0, 1.0)):
        """One round of speculative sampling with a draft model's probabilities, in one replay.

        ``token_ids`` (B, G+1) int64, 1 <= G <= 63: t_0 (the newest emitted token not fed yet) and the draft's G draws;
        ``draft_logits`` (B, G, vocab), of this model's logits dtype: the logits the draft drew t_1 .. t_G from, under
        ``draft_sampling`` = (temperature, top_k, top_p).  The replay feeds the G+1 tokens (as :meth:`extend`) and runs
        ``ops.spec_verify`` on the logits after each of them, under this decoder's ``set_sampling`` values, at the
        positions :meth:`sample` would draw at.  Returns ``(tokens, accepted)``: (B, G+1) int64, the n_b accepted
        drafts, the correction or bonus token, then -1; and (B,) int32 n_b.  Views of the graph's static outputs, valid
        until the next replay; nothing is read back to the host.  Consumes G+1 tokens of the budget: the caller then
        rewinds row b by G - n_b.  The graph is recorded on first use, one per (G, target values, draft values)."""
        self._ready_to_sample("verify")
        if self._process != _NO_PROCESS:
            raise ValueError("GraphedDecoder.verify: speculative verification is not covered with logits processors on "
                             "(the draft's processed distribution)")
        draft = _sampling_triple("GraphedDecoder.verify: draft_sampling", *_triple(draft_sampling))
        k = token_ids.shape[1] if token_ids.dim() == 2 else 0
        if not 2 <= k <= ops.SPEC_MAX_DRAFTS + 1:
            raise ValueError(f"GraphedDecoder.verify takes ({self.batch}, G+1) int64 tokens with 1 <= G <= "
                             f"{ops.SPEC_MAX_DRAFTS}, got {tuple(token_ids.shape)}")
        vocab = self.model.config.vocab_size
        if tuple(draft_logits.shape) != (self.batch, k - 1, vocab) or draft_logits.dtype != self.dtype:
            raise ValueError(f"GraphedDecoder.verify takes ({self.batch}, {k - 1}, {vocab}) {self.dtype} draft logits, "
                             f"got {tuple(draft_logits.shape)} {draft_logits.dtype}")
        self._draft_sampling = draft
        return self._replay(token_ids, "verify", draft_logits)

    # ---- prompt lookup ----------------------------------------------------------------------------------------------
    def prompt_lookup_generate(self, first: torch.Tensor, n: int, num_output_tokens: int = 10,
                               max_matching_ngram_size: int = 2):
        """Prompt-lookup decoding (🤗 ``generate(prompt_lookup_num_tokens=G, max_matching_ngram_size=N)``): n tokens
        per batch row, each the model's own draw at its position under the ``set_sampling`` values, with drafts
        copied from the row's own history.  Returns ``(tokens, stats)``: (B, n) int64, and a dict with ``rounds``,
        ``k`` (the tokens each round fed) and per batch row ``proposed`` (drafts offered while the row was live) and
        ``accepted`` (of those, accepted).

        ``first`` (B, 1) int64 is the token after the prompt (``draw``).  A row's history is what ``prefill`` was given
        after its left padding, then every token it was fed, then t_0 (its newest token, fed by the next round).  Its
        drafts are ``ops.prompt_lookup``'s: the up to G = ``num_output_tokens`` ids after the first earlier occurrence
        of its last n ids (n = N = ``max_matching_ngram_size`` down to 1), cut before an EOS id and capped so that the
        row never drafts past its n tokens; the processors play no part in them (🤗 crops candidates on fake logits).
        A round is one replay of k = max(draft count) + 1 tokens per row, t_0 then the drafts (filler after a row's
        own, never accepted): the sampler draws after each, the device accepts the leading drafts equal to the draws
        (``drafts[:, i+1] == tokens[:, i]``, so every emitted token is the draw at its position), takes the draw after
        the last accepted draft as the next t_0, finishes a row that emitted an EOS id, and searches the next drafts
        (``ops.prompt_lookup_round``), all in the graph.  Then one device-to-host read of the accept counts, the next
        draft counts and the finished flags; row b is rewound by k - 1 - n_b, or by k once it is finished or has n
        tokens (it stops advancing).  Before the first round the drafts of ``first`` are searched eagerly and their
        counts read once.  The graph is recorded on first use, one per (k, sampling values, processors, EOS ids, G, N).

        With ``set_sampling`` EOS ids, 🤗 ``_sample``'s rule: a row that has emitted an EOS id (``first`` included)
        emits the pad token from then on; the loop stops once every row is finished or has n tokens.  Needs
        :func:`prompt_lookup_budget` (n, G, B) tokens of budget left, refused before any replay."""
        what = "GraphedDecoder.prompt_lookup_generate"
        G, N, count = _as_count(num_output_tokens), _as_count(max_matching_ngram_size), _as_count(n)
        if G is None or not 1 <= G <= ops.LOOKUP_MAX_DRAFTS:
            raise ValueError(f"{what}: num_output_tokens must be an integer in [1, {ops.LOOKUP_MAX_DRAFTS}], got "
                             f"{num_output_tokens!r}")
        if N is None or not 1 <= N <= ops.LOOKUP_MAX_NGRAM:
            raise ValueError(f"{what}: max_matching_ngram_size must be an integer in [1, {ops.LOOKUP_MAX_NGRAM}], got "
                             f"{max_matching_ngram_size!r}")
        if count is None or count < 1:
            raise ValueError(f"{what}: n must be an integer >= 1, got {n!r}")
        self._ready_to_sample("prompt_lookup_generate")
        B, dev = self.batch, self.device
        if tuple(first.shape) != (B, 1) or first.dtype != torch.long:
            raise ValueError(f"{what} takes ({B}, 1) int64 first tokens, got {tuple(first.shape)} {first.dtype}")
        need = prompt_lookup_budget(count, G, B)
        if self._remaining < need:
            raise RuntimeError(f"{what}: {self._remaining} tokens of budget left, n={count} with up to {G} drafts per "
                               f"round needs {need} (prompt_lookup_budget)")
        if torch.is_autocast_enabled():
            raise RuntimeError("GraphedDecoder does not run under autocast")
        if not self._lookup_state:   # one set per decoder: the recorded graphs keep their addresses
            self._lookup_state = (torch.zeros(B, ops.LOOKUP_MAX_DRAFTS + 1, dtype=torch.long, device=dev),
                                  torch.zeros(4, B, dtype=torch.int32, device=dev),
                                  torch.zeros(B, dtype=torch.int32, device=dev))
        nxt, state, start = self._lookup_state
        self._lookup_args = (G, N)
        # the first round's drafts: first at the row it will be fed at, searched eagerly
        rows = self._bounds[:, 0, 2]
        self._tokens.scatter_(1, rows[:, None].long(), first)
        start.copy_(self._pad[:, :self._n0].sum(dim=1))
        if self._eos:
            state[2].copy_(~self._is_eos(first[:, 0]))
        else:
            state[2].fill_(1)
        state[3].fill_(count)
        state[0].copy_(state[2] * min(count - 1, G))   # the first search's per-row limit
        drafts, counts = ops.prompt_lookup(self._tokens, rows, G, N, start=start, limit=state[0], eos=self._eos,
                                           length_offset=1)
        nxt[:, :1].copy_(first)
        nxt[:, 1:G + 1].copy_(drafts)
        state[1].copy_(counts)
        cnt, unf = state[1:3].to("cpu").tolist()   # the drafts of the first round
        width = count + G + 2                      # column width - 1 takes the tokens a round does not keep
        fill = self._pad_token if self._eos else 0
        buf = torch.full((B, width), fill, dtype=torch.long, device=dev)
        done, proposed, accepted = [0] * B, [0] * B, [0] * B
        ks = []
        while True:
            live = [bool(u) and d < count for u, d in zip(unf, done)]
            if not any(live):
                break
            k = max(c for c, l in zip(cnt, live) if l) + 1
            tokens = self._replay(nxt[:, :k], "lookup")
            acc, nxt_cnt, unf = state[:3].to("cpu").tolist()   # the round's one synchronisation
            ks.append(k)
            idx, back = _settle_round(acc, live, [c if l else 0 for c, l in zip(cnt, live)], done, proposed, accepted,
                                      k, width, dev)
            buf.scatter_(1, idx[:, :k], tokens)
            self.rewind(back)
            cnt = nxt_cnt
        return buf[:, :count], {"rounds": len(ks), "k": ks, "proposed": proposed, "accepted": accepted}

    # ---- beam search ----------------------------------------------------------------------------------------------
    def _beam_args(self, B: int, n, num_beams, eos_token_id, length_penalty, early_stopping, num_return_sequences,
                   check_every):
        """The checked arguments of ``beam_search``: (K, n, eos ids, length_penalty, early_stopping, R, check_every)."""
        what = "GraphedDecoder.beam_search"
        K, count, R, every = _as_count(num_beams), _as_count(n), _as_count(num_return_sequences), _as_count(check_every)
        if K is None or not 1 <= K <= ops.BEAM_MAX_BEAMS:
            raise ValueError(f"{what}: num_beams must be an integer in [1, {ops.BEAM_MAX_BEAMS}], got {num_beams!r}")
        if self.batch != B * K:
            raise ValueError(f"{what}: the decoder's batch {self.batch} must be batch * num_beams = {B} * {K}")
        if count is None or count < 1 or count - 1 > self.max_new_tokens:
            raise ValueError(f"{what}: n must be an integer in [1, max_new_tokens + 1 = {self.max_new_tokens + 1}] "
                             f"(token 1 comes from the prefill), got {n!r}")
        if R is None or not 1 <= R <= K:
            raise ValueError(f"{what}: num_return_sequences must be an integer in [1, num_beams={K}], got "
                             f"{num_return_sequences!r}")
        if every is None or every < 1:
            raise ValueError(f"{what}: check_every must be an integer >= 1, got {check_every!r}")
        vocab = self.model.config.vocab_size
        if vocab > ops.SAMPLE_MAX_VOCAB:
            raise RuntimeError(f"{what}: the device beam step takes vocabularies up to {ops.SAMPLE_MAX_VOCAB}, this "
                               f"model has {vocab}")
        eos = _eos_ids(eos_token_id)
        if len(eos) > ops.BEAM_MAX_EOS or any(not 0 <= e < vocab for e in eos):
            raise ValueError(f"{what}: at most {ops.BEAM_MAX_EOS} EOS ids, each in [0, {vocab}), got {eos}")
        if K * vocab < ops.beams_to_keep(K, len(eos)):
            raise ValueError(f"{what}: num_beams * vocab = {K * vocab} is below the {ops.beams_to_keep(K, len(eos))} "
                             f"candidates a step keeps")
        lp = float(length_penalty)
        if not math.isfinite(lp):
            raise ValueError(f"{what}: length_penalty must be finite, got {length_penalty!r}")
        ops.early_stopping_code(early_stopping)
        return K, count, eos, lp, early_stopping, R, every

    def beam_search(self, input_ids: torch.Tensor, prefix_len: int, n: int, num_beams: int, pad_mask=None,
                    eos_token_id=None, pad_token_id=None, length_penalty: float = 1.0, early_stopping=False,
                    num_return_sequences: int = 1, check_every: int = 16, repetition_penalty: float = 1.0,
                    no_repeat_ngram_size: int = 0, min_new_tokens: int = 0) -> BeamSearchOutput:
        """🤗's beam search (``GenerationMixin._beam_search`` with ``do_sample=False``) of n
        generated tokens for the B prompts ``input_ids`` (B, n0), with K = ``num_beams`` beams each; the decoder's batch
        must be B * K.  Returns ``BeamSearchOutput(sequences, scores)``: 🤗's ``sequences[:, :num_return_sequences]``
        (generated part, (B, R, n) int64, the output fill value — ``pad_token_id or eos_token_id[0]`` with EOS ids, else
        -1 — after each hypothesis's end) and its ``sequences_scores`` (B, R) fp32.

        Prefills ``input_ids.repeat_interleave(K, 0)`` (beam k of item b is batch row b*K + k), runs the device beam
        step (``ops.beam_step``) eagerly on the prefill's logits, then n - 1 replays of one graph: feed the K beams'
        tokens, the beam step on their logits, and the gather of the rows generated since the prefill by parent
        (``ops.kv_gather_rows``).  Each replay's input is copied on the device from the previous replay's output.  With
        EOS ids, the device's "every item done" flag is read every ``check_every`` replays and the loop stops once it
        is set (🤗's stop condition; a stopped item's finished set no longer changes, so the output is the same);
        without, nothing is read until the end.  The graph is recorded on first use after each prefill, keyed by (K, EOS
        ids, length_penalty, early_stopping).  Refusals come before any replay.

        ``repetition_penalty``, ``no_repeat_ngram_size`` and ``min_new_tokens`` are 🤗's logits processors, as
        ``set_sampling`` takes them (``min_new_tokens`` needs EOS ids): 🤗 runs them on the fp32 log-softmax of every
        beam's logits, with the prompt and the beam's own generated tokens as its history, so the step and every replay
        then run ``ops.process_logits(..., log_softmax=True)`` and ``ops.beam_step(..., logprobs=True)``.  With every
        processor off the graph is the plain one."""
        B = input_ids.shape[0] if input_ids.dim() == 2 else 0
        K, count, eos, lp, es, R, every = self._beam_args(B, n, num_beams, eos_token_id, length_penalty,
                                                          early_stopping, num_return_sequences, check_every)
        process = _process_values("GraphedDecoder.beam_search", repetition_penalty, no_repeat_ngram_size,
                                  min_new_tokens, eos)
        if torch.is_autocast_enabled():
            raise RuntimeError("GraphedDecoder does not run under autocast")
        fill = (pad_token_id or eos[0]) if eos else -1

        def beams(t):   # (B, ...) -> (B*K, ...), beam k of item b at row b*K + k (repeat_interleave without a sync)
            return t[:, None].expand(t.shape[0], K, *t.shape[1:]).reshape(-1, *t.shape[1:])

        logits = self.prefill(beams(input_ids), prefix_len, beams(pad_mask) if pad_mask is not None else None)
        state = self._beam_state
        if state is None or (state.B, state.K, state.n_eos) != (B, K, len(eos)):
            state = self._beam_state = ops.BeamState(B, K, len(eos), self.max_new_tokens + 1, fill, self.device)
        state.fill = fill   # reset() fills the histories with it
        n0 = input_ids.shape[1]
        first = (n0, n0 - prefix_len)
        # prefill allocated new arenas: a new table, but the scratch of the last one when the shapes match
        table = self._beam_table = ops.KvGatherTable(
            [(t, first[a.group], a.group * _NCOL + 2) for a in self._layers for t in (a.K, a.V, a.S) if t is not None],
            reuse=self._beam_table)
        rows = self._bounds.view(self.batch, -1)
        on = process != _NO_PROCESS
        if on:
            logp = torch.empty(self.batch, self.model.config.vocab_size, dtype=torch.float32, device=self.device)
            hist = state.running_hist.view(self.batch, -1)

        def step(logits):   # the beam step, after the processors on the log-softmax when one is on
            if not on:
                return ops.beam_step(logits, state, eos, lp, es)
            ops.process_logits(logits, self._tokens, n0, tail=hist, tail_len=state.counters[0:1], out=logp,
                               log_softmax=True, repetition_penalty=process[0], no_repeat_ngram_size=process[1],
                               min_new_tokens=process[2], prompt_len=n0, eos=eos)
            return ops.beam_step(logp, state, eos, lp, es, logprobs=True)

        def beam_fn(token):
            tokens, parents = step(self._step_fn(token))
            ops.kv_gather_rows(table, parents, rows)
            return tokens

        gkey = ("beam", K, tuple(eos), lp, str(es)) + ((process,) if on else ())
        state.reset(count)
        if count > 1 and gkey not in self._graphs:
            # recorded before the first step: the warm-up calls append, and gather, only rows that are rewritten later
            snapshot = self._bounds.clone()
            old = torch.cuda.get_sync_debug_mode()
            torch.cuda.set_sync_debug_mode(0)
            try:
                self._graphs[gkey] = GraphedForward(beam_fn, state.tokens)
            finally:
                torch.cuda.set_sync_debug_mode(old)
            self._bounds.copy_(snapshot)
            self.captures += 1
            state.reset(count)
        step(logits)
        graph = self._graphs.get(gkey)
        for i in range(count - 1):
            graph(state.tokens)
            self._remaining -= 1
            self._fed += 1
            if eos and (i + 1) % every == 0 and i + 1 < count - 1:
                old = torch.cuda.get_sync_debug_mode()
                torch.cuda.set_sync_debug_mode(0)
                try:
                    stop = bool(state.counters[2].item())   # the one host read: every item done
                finally:
                    torch.cuda.set_sync_debug_mode(old)
                if stop:
                    break
        return BeamSearchOutput(state.finished_hist[:, :R, :count].clone(), state.finished[:, :R].clone())

    # ---- contrastive search -------------------------------------------------------------------------------------------
    def _contrastive_args(self, B: int, n, penalty_alpha, top_k, eos_token_id, pad_token_id, check_every):
        """The checked arguments of ``contrastive_search``: (K, n, alpha, eos ids, pad token, check_every)."""
        what = "GraphedDecoder.contrastive_search"
        K, count, every = _as_count(top_k), _as_count(n), _as_count(check_every)
        if K is None or not 1 <= K <= ops.CONTRASTIVE_MAX_K:
            raise ValueError(f"{what}: top_k must be an integer in [1, {ops.CONTRASTIVE_MAX_K}], got {top_k!r}")
        if self.batch != B * K:
            raise ValueError(f"{what}: the decoder's batch {self.batch} must be batch * top_k = {B} * {K}")
        if count is None or not 1 <= count <= self.max_new_tokens:
            raise ValueError(f"{what}: n must be an integer in [1, max_new_tokens = {self.max_new_tokens}], got {n!r}")
        if isinstance(penalty_alpha, bool) or not isinstance(penalty_alpha, (int, float)) or not 0.0 <= penalty_alpha <= 1.0:
            raise ValueError(f"{what}: penalty_alpha must be a number in [0, 1], got {penalty_alpha!r}")
        if every is None or every < 1:
            raise ValueError(f"{what}: check_every must be an integer >= 1, got {check_every!r}")
        vocab = self.model.config.vocab_size
        if vocab > ops.SAMPLE_MAX_VOCAB:
            raise RuntimeError(f"{what}: the device candidate step takes vocabularies up to {ops.SAMPLE_MAX_VOCAB}, this "
                               f"model has {vocab}")
        if K > vocab:
            raise ValueError(f"{what}: top_k={K} is above the vocabulary size {vocab}")
        D = self.model.config.num_channels
        if D % 8 or D > ops.CONTRASTIVE_MAX_HIDDEN:
            raise RuntimeError(f"{what}: the device ranking takes hidden widths that are multiples of 8 up to "
                               f"{ops.CONTRASTIVE_MAX_HIDDEN}, this model has {D}")
        eos = _eos_ids(eos_token_id, what)
        if len(eos) > ops.CONTRASTIVE_MAX_EOS or any(not 0 <= e < vocab for e in eos):
            raise ValueError(f"{what}: at most {ops.CONTRASTIVE_MAX_EOS} EOS ids, each in [0, {vocab}), got {eos}")
        if pad_token_id is None:
            pad = eos[0] if eos else -1   # 🤗 generate(): the first EOS id; without EOS ids nothing is ever padded
        else:
            pad = _as_count(pad_token_id)
            if pad is None or not -2 ** 63 <= pad < 2 ** 63:
                raise ValueError(f"{what}: pad_token_id must be None or an integer, got {pad_token_id!r}")
        return K, count, float(penalty_alpha), eos, pad, every

    def contrastive_search(self, input_ids: torch.Tensor, prefix_len: int, n: int, penalty_alpha: float, top_k: int,
                           pad_mask=None, eos_token_id=None, pad_token_id=None, check_every: int = 16,
                           repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0,
                           min_new_tokens: int = 0) -> torch.Tensor:
        """🤗 4.28's contrastive search (``GenerationMixin.contrastive_search`` without warpers) of
        n generated tokens for the B prompts ``input_ids`` (B, n0), with K = ``top_k`` candidates and α =
        ``penalty_alpha``; the decoder's batch must be B * K and n <= ``max_new_tokens``.  Returns the generated tokens
        (B, n) int64: ``pad_token_id`` after an item has emitted an EOS id (``pad_token_id=None`` with EOS ids means the
        first EOS id, as in 🤗 ``generate()``; an explicit 0 stays 0).

        Each step takes the K most likely tokens of the selected row's logits (p_j their softmax probabilities), runs
        the model on all K, and selects the lowest j maximising ``(1 - α) p_j - α max_s cos(c_s, h_j)``, where h_j is
        candidate j's final hidden row and c_s the item's context: the prompt's final hidden rows at its latent
        positions, then every selected candidate's.  Unlike 4.28, padded prompt positions are left out of the max (they
        carry no token; later 🤗 releases mask them too); on unpadded prompts the two agree.  The ranking is computed
        in fp64, not in the model dtype as 🤗 does, so on near-ties 🤗 may choose differently.

        Prefills ``input_ids.repeat_interleave(K, 0)`` (candidate j of item b is batch row b*K + j), loads the context,
        takes the first candidates eagerly (``ops.contrastive_candidates``), then n replays of one graph: feed the
        candidates, rank them (``ops.contrastive_step``), and copy the selected row's newest arena row into the item's
        other rows (``ops.kv_gather_rows(..., last_rows=1)``).  Each replay's input is its predecessor's output.  With
        EOS ids the device's "every item finished" flag is read every ``check_every`` replays and the loop stops once
        it is set; nothing else is read.  The graph is recorded once after each prefill, keyed by (K, α, EOS ids, pad).
        Refusals come before any replay.

        ``repetition_penalty``, ``no_repeat_ngram_size`` and ``min_new_tokens`` are 🤗's logits processors, as
        ``set_sampling`` takes them (``min_new_tokens`` needs EOS ids): they run on the selected row's logits, with the
        prompt and the tokens emitted so far as its history, before the softmax and top-k that pick the candidates
        (the first candidates included), through ``ops.process_logits``.  4.28 runs them in the model dtype; here they
        run in fp32, like the ranking's fp64, so on near-ties the two may choose differently."""
        B = input_ids.shape[0] if input_ids.dim() == 2 else 0
        K, count, alpha, eos, pad, every = self._contrastive_args(B, n, penalty_alpha, top_k, eos_token_id, pad_token_id,
                                                                  check_every)
        process = _process_values("GraphedDecoder.contrastive_search", repetition_penalty, no_repeat_ngram_size,
                                  min_new_tokens, eos)
        if torch.is_autocast_enabled():
            raise RuntimeError("GraphedDecoder does not run under autocast")

        def rows_of(t):   # (B, ...) -> (B*K, ...), row b*K + j (repeat_interleave without a sync)
            return t[:, None].expand(t.shape[0], K, *t.shape[1:]).reshape(-1, *t.shape[1:])

        out = self._prefill(rows_of(input_ids), prefix_len, rows_of(pad_mask) if pad_mask is not None else None)
        logits, hidden = out.logits[:, -1], out.last_hidden_state[::K]   # the K rows of an item are equal
        del out
        L, D = hidden.shape[1], hidden.shape[2]
        cap = L + self.max_new_tokens
        state = self._cs_state
        if state is None or (state.B, state.K, state.D, state.cap, state.dtype) != (B, K, D, cap, hidden.dtype):
            state = self._cs_state = ops.ContrastiveState(B, K, D, cap, self.max_new_tokens, pad, hidden.dtype,
                                                          self.device)
        state.fill = pad
        ctx_pad = pad_mask[:, prefix_len:] if pad_mask is not None else None
        n0 = input_ids.shape[1]
        first = (n0, n0 - prefix_len)
        table = self._cs_table = ops.KvGatherTable(
            [(t, first[a.group], a.group * _NCOL + 2) for a in self._layers for t in (a.K, a.V, a.S) if t is not None],
            reuse=self._cs_table)
        rows = self._bounds.view(self.batch, -1)
        proc = None
        if process != _NO_PROCESS:
            # the selected row of every item, with the item's prompt (its row b*K) and emitted tokens as its history
            proc = dict(prefix=self._tokens[::K], prefix_len=n0, tail=state.history, tail_len=state.counters[1:2],
                        out=torch.empty(self.batch, logits.shape[-1], dtype=torch.float32, device=self.device),
                        repetition_penalty=process[0], no_repeat_ngram_size=process[1], min_new_tokens=process[2],
                        prompt_len=n0, eos=eos)

        def cs_fn(token):
            logits = self._step_fn(token)
            tokens, parents = ops.contrastive_step(logits, self._hidden, state, alpha, eos, process=proc)
            ops.kv_gather_rows(table, parents, rows, last_rows=1)
            return tokens

        def start():
            state.reset(hidden, ctx_pad)
            first = logits if proc is None else ops.process_logits(logits, row_map=state.sel, **proc)
            ops.contrastive_candidates(first, state)

        gkey = ("contrastive", K, alpha, tuple(eos), pad) + ((process,) if proc is not None else ())
        start()
        if gkey not in self._graphs:
            # the warm-up calls append, and select, only rows that the replays rewrite; the state is reloaded after
            snapshot = self._bounds.clone()
            old = torch.cuda.get_sync_debug_mode()
            torch.cuda.set_sync_debug_mode(0)
            try:
                self._graphs[gkey] = GraphedForward(cs_fn, state.tokens)
            finally:
                torch.cuda.set_sync_debug_mode(old)
            self._bounds.copy_(snapshot)
            self.captures += 1
            start()
        graph = self._graphs[gkey]
        for i in range(count):
            graph(state.tokens)
            self._remaining -= 1
            self._fed += 1
            if eos and (i + 1) % every == 0 and i + 1 < count:
                old = torch.cuda.get_sync_debug_mode()
                torch.cuda.set_sync_debug_mode(0)
                try:
                    stop = bool(state.counters[2].item())   # the one host read: every item finished
                finally:
                    torch.cuda.set_sync_debug_mode(old)
                if stop:
                    break
        return state.history[:, :count].clone()

    def rewind(self, n) -> None:
        """Drop fed tokens: the next token of a batch row is fed at the row of its first dropped one, as if the dropped
        tokens had never been fed.  ``n`` an integer drops the last n tokens of every batch row; a sequence of B
        integers, or a CPU integer tensor of shape (B,), drops the last ``n[b]`` of row b (per-row accept counts of
        batched speculative decoding).  Each count is at most the tokens its row has fed since prefill.  Eager int32 ops
        on the row counters (no host read of the device, no re-capture).  Gives back to the budget what the furthest
        row regains.  A refused ``n`` leaves the state untouched."""
        if self._bounds is None:
            raise RuntimeError("GraphedDecoder: call prefill() first")
        lag = self._lag or [0] * self.batch
        if isinstance(n, (Sequence, torch.Tensor)) and not isinstance(n, (str, bytes)) and (
                not isinstance(n, torch.Tensor) or n.dim() > 0):
            counts = self._row_counts(n, lag)
        else:
            count = _as_count(n)
            top = self._fed - max(lag)
            if count is None or count < 0 or count > top:
                raise ValueError(f"GraphedDecoder.rewind: n must be an integer in [0, {top}] (the tokens every batch "
                                 f"row has fed since prefill), got {n!r}")
            counts = [count] * self.batch
        if len(set(counts)) == 1:   # one count: every row moves alike, the lags stay
            if counts[0]:
                advance_bounds_(self._bounds, self._inc, self._wmax, -counts[0])
                self._remaining += counts[0]
                self._fed -= counts[0]
            return
        per_row = torch.tensor(counts, dtype=torch.int32)
        if self._bounds.is_cuda:   # pinned and asynchronous: no synchronisation
            per_row = per_row.pin_memory().to(self._bounds.device, non_blocking=True)
        advance_bounds_(self._bounds, self._inc, self._wmax, -per_row)
        self._set_fed([self._fed - lg - c for lg, c in zip(lag, counts)])

    def _row_counts(self, n, lag) -> List[int]:
        """The per-row counts of ``rewind``, checked against every row's fed tokens."""
        if isinstance(n, torch.Tensor):
            if n.is_cuda:
                raise ValueError("GraphedDecoder.rewind: per-row counts must be a CPU tensor (a CUDA tensor would need a "
                                 "host read of the device)")
            if n.dim() != 1 or n.dtype == torch.bool or n.dtype.is_floating_point or n.dtype.is_complex:
                raise ValueError(f"GraphedDecoder.rewind: per-row counts must be a ({self.batch},) integer tensor, got "
                                 f"{tuple(n.shape)} {n.dtype}")
            n = n.tolist()
        if len(n) != self.batch:
            raise ValueError(f"GraphedDecoder.rewind: {self.batch} per-row counts (one per batch row), got {len(n)}")
        counts = []
        for b, c in enumerate(n):
            count = _as_count(c)
            fed = self._fed - lag[b]
            if count is None or count < 0 or count > fed:
                raise ValueError(f"GraphedDecoder.rewind: the count of batch row {b} must be an integer in [0, {fed}] "
                                 f"(the tokens it has fed since prefill), got {c!r}")
            counts.append(count)
        return counts

    def _set_fed(self, fed: List[int]) -> None:
        """Host bookkeeping from the tokens every batch row has fed: the budget follows the furthest row."""
        top = max(fed)
        self._remaining += self._fed - top
        self._fed = top
        self._lag = [top - f for f in fed] if min(fed) != top else None

    def reorder(self, beam_idx: torch.Tensor) -> None:
        """Permute the batch rows of every arena, rotated-key arena, the pad rows and the row counters (beam search),
        eagerly.  Sync-free while every row has fed the same tokens; once per-row rewinds left them at different
        counts, ``beam_idx`` is read to the host once to permute the host bookkeeping."""
        idx = beam_idx.to(device=self.device, dtype=torch.long)
        for a in self._layers:
            for t in (a.K, a.V, a.S):
                if t is not None:
                    t.copy_(t.index_select(0, idx))
        self._pad.copy_(self._pad.index_select(0, idx))
        if self._tokens is not None:
            self._tokens.copy_(self._tokens.index_select(0, idx))
        self._bounds.copy_(self._bounds.index_select(0, idx))
        if self._seeds is not None:
            self._seeds.copy_(self._seeds.index_select(0, idx))
        if self._lag is not None:
            self._set_fed([self._fed - self._lag[i] for i in beam_idx.tolist()])


def _settle_round(acc: List[int], live: List[bool], offered: List[int], done: List[int], proposed: List[int],
                  accepted: List[int], k: int, width: int, device):
    """Host bookkeeping of one verified round that fed k tokens (t_0 and up to k - 1 drafts) to every batch row, from
    the n_b read back: live row b emitted its n_b accepted drafts and one more token, which go to columns done[b] ..
    done[b] + n_b of the output (``done``, ``proposed`` and ``accepted`` are updated in place; ``offered[b]`` drafts
    were proposed); a row that is not live emits nothing.  Returns ``(idx, back)``: (B, k+1) int64 on ``device``,
    whose first k columns place the round's k emitted-token columns in a (B, ``width``) output (column width - 1
    takes what is not kept) and whose last column is the column of ``[t_0 | tokens]`` that holds the row's next t_0;
    and the per-row rewind counts, k - 1 - n_b for a live row and k for the others (they stop advancing)."""
    B = len(acc)
    idx = torch.full((B, k + 1), width - 1, dtype=torch.long)
    back = []
    for b in range(B):
        if not live[b]:
            idx[b, k] = 0
            back.append(k)
            continue
        nb = acc[b]
        idx[b, :nb + 1] = done[b] + torch.arange(nb + 1)
        idx[b, k] = nb + 1
        back.append(k - 1 - nb)
        done[b] += nb + 1
        proposed[b] += offered[b]
        accepted[b] += nb
    if device.type == "cuda":                  # pinned and asynchronous: no synchronisation
        idx = idx.pin_memory().to(device, non_blocking=True)
    return idx, back


def prompt_lookup_budget(n: int, num_output_tokens: int, batch: int) -> int:
    """The ``max_new_tokens`` (budget left after ``prefill``) :meth:`GraphedDecoder.prompt_lookup_generate` needs for n
    tokens with G = ``num_output_tokens``: n for one batch row, n + min(G, n - 1) + 1 for more.

    A live row that has emitted e < n tokens has fed e of them (its newest, t_0, is fed by the next round) and drafts
    at most min(G, n - e - 1), so a round feeds k <= min(G, n - 1) + 1 tokens.  Alone, the row is fed k <= n - e:
    e + k <= n.  With more rows, k follows the row with the most drafts: a live row reaches at most e + k <= n - 1 +
    min(G, n - 1) + 1, and a row that is done has fed at most n and is still fed, then rewound, k tokens per round
    while another row is live: n + min(G, n - 1) + 1."""
    return n if batch == 1 else n + min(num_output_tokens, n - 1) + 1


def speculative_budget(n: int, draft_tokens: int, batch: int) -> int:
    """The ``max_new_tokens`` (budget left after ``prefill``) both decoders of :func:`speculative_generate` need for n
    tokens with G = ``draft_tokens`` drafts per round: n + G for one batch row, n + 2G + 1 for more.

    A row that has emitted e < n tokens has fed e of them, and a round feeds G+1 more before the rewind: at most
    n - 1 + G + 1 = n + G.  With more than one row a finished row can stand at n + G (it accepted every draft of its
    last round) and still be fed, and rewound, G+1 tokens per round while another row finishes: n + 2G + 1."""
    return n + draft_tokens if batch == 1 else n + 2 * draft_tokens + 1


def speculative_generate(target: "GraphedDecoder", draft: "GraphedDecoder", first: torch.Tensor, n: int,
                         draft_tokens: int = 4):
    """Speculative sampling with a draft model (Leviathan et al. 2023; Chen et al. 2023): n tokens per batch row, each
    distributed exactly as ``target.generate`` would draw it under the target's ``set_sampling`` values.

    Both decoders must have been prefilled with the same prompt (same batch and vocabulary); ``first`` (B, 1) int64 is
    drawn from the target (``target.draw``).  Each round of G = ``draft_tokens`` drafts:
      1. ``draft.generate(t_0, G+1, logits=True)``: the first G draws are the drafts, the last is discarded (it makes the
         draft feed t_0 .. t_G, as the target does);
      2. ``target.verify``: min(1, p/q) acceptance, the residual or bonus token, on the device;
      3. one device-to-host read of ``accepted`` — the round's only synchronisation;
      4. both decoders rewind row b by G - n_b (a row that already has n tokens by G+1: it stops advancing);
      5. the next t_0 of row b is its correction or bonus token, gathered on the device.
    Needs :func:`speculative_budget` (n, G, B) tokens of budget left in both decoders, refused before any replay.

    Returns ``(tokens, stats)``: (B, n) int64, and a dict with ``rounds``, and per batch row ``proposed`` (drafts
    offered while the row was unfinished) and ``accepted`` (of those, accepted)."""
    G, count = _as_count(draft_tokens), _as_count(n)
    if G is None or not 1 <= G <= ops.SPEC_MAX_DRAFTS:
        raise ValueError(f"speculative_generate: draft_tokens must be an integer in [1, {ops.SPEC_MAX_DRAFTS}], got "
                         f"{draft_tokens!r}")
    if count is None or count < 1:
        raise ValueError(f"speculative_generate: n must be an integer >= 1, got {n!r}")
    B = target.batch
    if draft.batch != B:
        raise ValueError(f"speculative_generate: the draft's batch {draft.batch} != the target's {B}")
    if draft.model.config.vocab_size != target.model.config.vocab_size:
        raise ValueError(f"speculative_generate: the draft's vocabulary {draft.model.config.vocab_size} != the "
                         f"target's {target.model.config.vocab_size}")
    if target._bounds is None or draft._bounds is None:
        raise RuntimeError("speculative_generate: prefill() both decoders first")
    if target._process != _NO_PROCESS or draft._process != _NO_PROCESS:
        raise ValueError("speculative_generate: not covered with logits processors on (the draft's processed "
                         "distribution)")
    if tuple(first.shape) != (B, 1) or first.dtype != torch.long:
        raise ValueError(f"speculative_generate takes ({B}, 1) int64 first tokens, got {tuple(first.shape)} "
                         f"{first.dtype}")
    need = speculative_budget(count, G, B)
    for name, dec in (("target", target), ("draft", draft)):
        if dec._remaining < need:
            raise RuntimeError(f"speculative_generate: the {name} has {dec._remaining} tokens of budget left, n={count} "
                               f"with {G} drafts per round needs {need} (speculative_budget)")
    dev = target.device
    width = count + G + 2                       # column width - 1 takes the tokens a round does not keep
    buf = torch.empty(B, width, dtype=torch.long, device=dev)
    done, proposed, accepted_total = [0] * B, [0] * B, [0] * B
    t0, rounds = first, 0
    while min(done) < count:
        drafts, q_logits = draft.generate(t0, G + 1, logits=True)
        fed = torch.cat([t0, drafts[:, :G]], dim=1)
        tokens, accepted = target.verify(fed, q_logits[:, :G], draft_sampling=draft._sampling)
        acc = accepted.to("cpu").tolist()       # the round's one synchronisation
        rounds += 1
        idx, back = _settle_round(acc, [d < count for d in done], [G] * B, done, proposed, accepted_total, G + 1,
                                  width, dev)
        buf.scatter_(1, idx[:, :G + 1], tokens)
        t0 = torch.cat([t0, tokens], dim=1).gather(1, idx[:, G + 1:])
        target.rewind(back)
        draft.rewind(back)
    return buf[:, :count], {"rounds": rounds, "proposed": proposed, "accepted": accepted_total}
