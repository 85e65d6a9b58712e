"""CPU checks of per-batch-row device rows: every device-row entry point refuses a negative bounds_stride_b before any
CUDA call, and GraphedDecoder's per-row rewind keeps every batch row on its own one-token loop: through seeded
schedules of extend and per-row / scalar rewinds, each fed token's band window and append / rotary row are those the
one-token truncation loop gives that row, and the per-row positions are those of ``positions()``."""
import ctypes
import random

import pytest
import torch

import window_variants as WV
from perceiver_io_b200 import _lib
from test_decode_step_entries_cpu import APP, APP8, DEC, DEC8, ROT, ROT8, _inputs, _launch, _supported
from test_graph_decode_cpu import _truncation_loop
from test_window_cpu import ENTRIES as WIN_ENTRIES
from test_window_cpu import _call as _win_call
from test_window_cpu import _params as _win_params
from test_window_cpu import _state

STRIDE_REASON = b"rows->bounds_stride_b must be >= 0"


@pytest.mark.parametrize("entry", [DEC, DEC8, APP, APP8, ROT, ROT8])
def test_decode_append_rotary_refuse_a_negative_bounds_stride(entry):
    lib = _lib.lib()
    p, f, rows = _inputs(None, entry)
    rows.bounds_stride_b = -1
    if entry in (DEC, DEC8):
        assert _supported(entry, p, f, rows) == 0
        assert STRIDE_REASON in lib.pcv_last_error(), lib.pcv_last_error()
    assert _launch(entry, p, f, rows) != 0
    assert STRIDE_REASON in lib.pcv_last_error(), lib.pcv_last_error()
    if entry in (DEC, DEC8):   # a per-row stride is accepted
        rows.bounds_stride_b = 12
        assert _supported(entry, p, f, rows) == 1, lib.pcv_last_error()


@pytest.mark.parametrize("entry", WIN_ENTRIES)
def test_window_refuses_a_negative_bounds_stride(entry):
    lib = _lib.lib()
    p, f, rows = _win_params()
    rows.bounds_stride_b = -6
    assert _win_call(entry, p, f, rows, 4, True) == 0
    assert STRIDE_REASON in lib.pcv_last_error(), lib.pcv_last_error()
    assert _win_call(entry, p, f, rows, 4, False) != 0
    assert STRIDE_REASON in lib.pcv_last_error(), lib.pcv_last_error()
    rows.bounds_stride_b = 12
    assert _win_call(entry, p, f, rows, 4, True) == 1, lib.pcv_last_error()


def test_dev_rows_struct_layout_is_unchanged():
    assert ctypes.sizeof(_lib.DevRows) == 16
    assert _lib.DevRows.bounds_stride_b.offset == 12 and _lib.DevRows.capacity.offset == 8


# ---- GraphedDecoder: per-row bookkeeping ------------------------------------------------------------------------------
class _Steps:
    """Stands in for the recorded graphs: a k-token replay moves the bounds exactly as _step_fn does, and records the
    bounds the kernels of that replay read."""

    def __init__(self, dec):
        self.dec, self.seen = dec, []

    def get(self, k):
        from perceiver_io_b200.generation import advance_bounds_, extend_bounds

        def replay(tokens):
            d = self.dec
            self.seen.append(extend_bounds(d._bounds, k))
            advance_bounds_(d._bounds, d._inc, d._wmax, k)
            return torch.zeros(d.batch, k, 1)

        return replay


def _decoder(B, n0, prefix, max_seq_len, max_latents, T):
    from perceiver_io_b200 import GraphedDecoder

    dec = object.__new__(GraphedDecoder)
    b, inc, wmax = _state(n0, prefix, max_seq_len, max_latents)
    dec.batch, dec.max_new_tokens = B, T
    dec._bounds, dec._inc, dec._wmax = b.repeat(B, 1, 1), inc, wmax   # (B, groups, 6) as prefill builds it
    dec._remaining, dec._fed = T, 0
    dec._graphs = _Steps(dec)
    dec._layers, dec.device = [], torch.device("cpu")
    dec._pad = torch.zeros(B, n0 + T, dtype=torch.uint8)
    return dec


def _check_rows(dec, fed, n0, prefix, max_seq_len, max_latents, T):
    """The decoder's state against the one-token loop of every row, which has fed fed[b] tokens."""
    top = max(fed)
    assert dec._fed == top and dec._remaining == T - top
    assert dec._lag == (None if min(fed) == top else [top - f for f in fed])
    for b, f in enumerate(fed):
        nxt = _truncation_loop(n0, prefix, f + 1, max_seq_len, max_latents)[f]
        assert dec._bounds[b, 0, :2].tolist() == list(nxt[:2]) and dec._bounds[b, 1, :2].tolist() == list(nxt[2:4]), b
        assert dec._bounds[b, :, 2].tolist() == [n0 + f, n0 - prefix + f], b
        assert dec._bounds[b, :, 4].tolist() == [n0 + f, n0 - prefix + f] and dec._bounds[b, :, 3].tolist() == [1, 1]


GEOMETRIES = [
    # (batch, prompt_len, prefix_len, max_seq_len, max_latents, max_new_tokens, ks)
    (3, 20, 0, 64, 48, 120, (3, 5, 16, 1)),        # the latents fill mid-step
    (4, 120, 90, 160, 48, 200, (64, 5, 16, 3)),    # k > max_latents, both windows slide
    (3, 160, 112, 160, 48, 150, (2, 64, 7)),       # a full context from the start
    (5, 5, 4, 8, 2, 60, (7, 3, 1, 9)),             # windows narrower than k
]


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("B,n0,prefix,max_seq_len,max_latents,T,ks", GEOMETRIES)
def test_per_row_rewind_keeps_every_row_on_its_one_token_loop(seed, B, n0, prefix, max_seq_len, max_latents, T, ks):
    """Seeded schedules of extend(k) and rewinds (per-row counts from 0 to everything the row fed, and scalar counts):
    every fed token's band window and append / rotary row equal the one-token loop's for that row, and the state after
    every call is that loop's state for the row's next token."""
    rng = random.Random(seed * 1000 + B * 100 + n0)
    dec = _decoder(B, n0, prefix, max_seq_len, max_latents, T)
    fed = [0] * B
    for step in range(14):
        k = ks[step % len(ks)]
        if dec._remaining < k:
            with pytest.raises(RuntimeError, match=f"{dec._remaining} of max_new_tokens={T} tokens remain"):
                dec.extend(torch.zeros(B, k, dtype=torch.long))
            k = dec._remaining
            if k == 0:
                break
        dec.extend(torch.zeros(B, k, dtype=torch.long))
        kb = dec._graphs.seen[-1]
        for b in range(B):
            loop = _truncation_loop(n0, prefix, fed[b] + k, max_seq_len, max_latents)[fed[b]:]
            for i in range(k):
                ca = WV.row_keys(i, k, int(kb[b, 0, 0]), int(kb[b, 0, 1]), 10_000, max_seq_len, True)[:2]
                sa = WV.row_keys(i, k, int(kb[b, 1, 0]), int(kb[b, 1, 1]), 10_000, max_latents, True)[:2]
                assert ca + sa == loop[i][:4], (step, b, i)
            assert kb[b, :, 2].tolist() == [n0 + fed[b], n0 - prefix + fed[b]] and torch.equal(kb[b, :, 2], kb[b, :, 4])
        fed = [f + k for f in fed]
        _check_rows(dec, fed, n0, prefix, max_seq_len, max_latents, T)
        # accept counts: a row keeps a prefix of this step's tokens; sometimes a row drops everything it has fed, and
        # sometimes every row takes one scalar count
        if rng.random() < 0.25:
            n = rng.randint(0, min(fed))
            dec.rewind(n)
            fed = [f - n for f in fed]
        else:
            counts = [rng.randint(0, k) for _ in range(B)]
            counts[rng.randrange(B)] = 0
            if rng.random() < 0.3:
                b = rng.randrange(B)
                counts[b] = fed[b]
            dec.rewind(counts if rng.random() < 0.5 else torch.tensor(counts))
            fed = [f - c for f, c in zip(fed, counts)]
        _check_rows(dec, fed, n0, prefix, max_seq_len, max_latents, T)


def test_budget_follows_the_furthest_row():
    B, T = 3, 10
    dec = _decoder(B, 30, 10, 40, 16, T)
    dec.extend(torch.zeros(B, 6, dtype=torch.long))
    dec.rewind([0, 4, 6])                       # the furthest row keeps 6: 4 tokens left
    assert dec._remaining == 4 and dec._fed == 6 and dec._lag == [0, 4, 6]
    with pytest.raises(RuntimeError, match="4 of max_new_tokens=10 tokens remain"):
        dec.extend(torch.zeros(B, 5, dtype=torch.long))
    dec.extend(torch.zeros(B, 4, dtype=torch.long))
    assert dec._remaining == 0
    dec.rewind([1, 0, 0])                       # the furthest row regains 1, the others are not the furthest
    assert dec._remaining == 1 and dec._fed == 9 and dec._lag == [0, 3, 5]
    dec.rewind([3, 0, 0])                       # row 0 falls back to row 1's count: the budget follows it
    assert dec._remaining == 4 and dec._fed == 6 and dec._lag == [0, 0, 2]
    with pytest.raises(ValueError, match=r"n must be an integer in \[0, 4\]"):
        dec.rewind(5)                           # a scalar count is bounded by the row that fed the least
    dec.rewind(4)
    assert dec._fed == 2 and dec._lag == [0, 0, 2] and dec._remaining == 8


def test_equal_counts_take_the_scalar_path():
    B = 3
    a, b = (_decoder(B, 120, 90, 160, 48, 64) for _ in range(2))
    for d in (a, b):
        d.extend(torch.zeros(B, 9, dtype=torch.long))
        d.rewind([1, 4, 2])
    a.rewind([2, 2, 2])
    b.rewind(2)
    assert torch.equal(a._bounds, b._bounds) and (a._fed, a._remaining, a._lag) == (b._fed, b._remaining, b._lag)
    a.rewind(torch.tensor([0, 0, 0]))
    assert torch.equal(a._bounds, b._bounds) and a._lag == [0, 3, 1]


BAD = [
    ([1, 1], "3 per-row counts"),
    ([1, 1, 1, 1], "3 per-row counts"),
    ("abc", "n must be an integer"),
    ([0, "1", 0], "batch row 1"),
    ([0, 1.0, 0], "batch row 1"),
    ([True, 0, 0], "batch row 0"),
    ([0, 0, -1], "batch row 2"),
    ([0, 0, 3], r"batch row 2 must be an integer in \[0, 2\]"),
    ([0, 6, 0], r"batch row 1 must be an integer in \[0, 5\]"),
    (torch.tensor([0.0, 1.0, 0.0]), "integer tensor"),
    (torch.tensor([True, False, False]), "integer tensor"),
    (torch.zeros(3, 1, dtype=torch.long), "integer tensor"),
    (torch.tensor([0, 0]), "3 per-row counts"),
    (1.5, "n must be an integer"),
    (3, r"n must be an integer in \[0, 2\]"),
]


@pytest.mark.parametrize("n,match", BAD, ids=[f"bad{i}" for i in range(len(BAD))])
def test_rewind_refusals_leave_the_state_untouched(n, match):
    B = 3
    dec = _decoder(B, 30, 10, 40, 16, 20)
    dec.extend(torch.zeros(B, 5, dtype=torch.long))
    dec.rewind([0, 0, 3])
    before = (dec._bounds.clone(), dec._fed, dec._remaining, list(dec._lag))
    with pytest.raises(ValueError, match=match):
        dec.rewind(n)
    assert torch.equal(dec._bounds, before[0]) and (dec._fed, dec._remaining, dec._lag) == before[1:]


def test_reorder_permutes_the_per_row_state():
    B, n0, prefix = 3, 30, 10
    dec = _decoder(B, n0, prefix, 40, 16, 20)
    dec.extend(torch.zeros(B, 6, dtype=torch.long))
    dec.rewind([0, 2, 5])
    rows = dec._bounds.clone()
    dec.reorder(torch.tensor([2, 1, 1]))        # the furthest row is dropped
    assert torch.equal(dec._bounds, rows[[2, 1, 1]])
    assert dec._fed == 4 and dec._lag == [3, 0, 0] and dec._remaining == 16
    dec.reorder(torch.tensor([1, 2, 1]))
    assert dec._fed == 4 and dec._lag is None and dec._remaining == 16
    dec.reorder(torch.tensor([0, 0, 2]))        # equal rows: nothing on the host changes
    assert dec._fed == 4 and dec._lag is None


def test_per_row_positions_match_positions_with_left_padding():
    """window_positions / window_positions_rows with per-row bounds: every row's positions are those of its own
    one-token window, with different left padding per row."""
    from perceiver_io_b200 import positions
    from perceiver_io_b200.generation import extend_bounds, window_positions, window_positions_rows

    B, n0, prefix, cap, W = 4, 30, 12, 140, 40
    pad = torch.zeros(B, cap, dtype=torch.uint8)
    pad[1, :4] = 1
    pad[2, :n0] = 1                      # a fully padded prompt row
    pad[3, :17] = 1
    cols = torch.arange(cap, dtype=torch.int32)
    b, inc, wmax = _state(n0, prefix, W, 16)
    from perceiver_io_b200.generation import advance_bounds_

    state = b.repeat(B, 1, 1)
    lead = torch.tensor([0, 3, 11, 40], dtype=torch.int32)
    advance_bounds_(state, inc, wmax, lead)   # every row at its own next row
    for k in (1, 2, 7, 64):
        kb = extend_bounds(state, k)
        got = window_positions_rows(pad, kb[:, 0], cols, k, W)
        assert got.shape == (B, k) and got.dtype == torch.int64
        for row in range(B):
            for i in range(k):
                r = n0 + int(lead[row]) + i
                lo = max(0, r + 1 - W)
                shift = pad[row:row + 1, lo:r + 1].bool().sum(dim=1, keepdim=True)
                assert torch.equal(got[row:row + 1, i:i + 1], positions(1, r + 1 - lo, shift=shift)[:, -1:]), (k, row, i)
            # one row of the per-row form is the shared form of that row's bounds
            assert torch.equal(got[row], window_positions_rows(pad, kb[row, 0], cols, k, W)[row])
        if k == 1:
            assert torch.equal(got, window_positions(pad, kb[:, 0, 0:2], cols))
