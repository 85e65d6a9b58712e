"""CPU checks of the banded-window tensor-core attention (pcv_attn_cached_window / _fp8, the window instantiations of
attn_cached_kernel in csrc/pcv_attn_cached.cu) and of the k-token steps of GraphedDecoder: the entry points refuse what
they do not cover before any CUDA call, the workspace and the split plan are the restated ones of window_variants.py,
the variant matrix reaches every instantiation, the build has no spills and no serialised wgmma, the CPU emulation of
the kernel's arithmetic stays within half of the element-wise gate of test_gpu_window.py, and the decoder's k-step bounds
and positions give every fed token the window of the one-token loop through any sequence of extend and rewind."""
import ctypes
import random

import numpy as np
import pytest
import torch

import window_variants as WV
from cached_fp8_variants import device_sms, left_pad
from perceiver_io_b200 import _lib
from test_cached_fp8_cpu import cached_kernel_entries
from test_graph_decode_cpu import _truncation_loop

ENTRIES = ("pcv_attn_cached_window", "pcv_attn_cached_window_fp8")


def _params(N=8, M=300, dqk=64, dv=64, B=2, H=2, causal=1):
    p = _lib.AttnParams()
    p.q, p.k, p.v, p.out = 1 << 20, 2 << 20, 3 << 20, 4 << 20  # never dereferenced: the checks run first
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.q_stride_b, p.q_stride_n, p.q_stride_h = N * H * dqk, H * dqk, dqk
    p.k_stride_b, p.k_stride_m, p.k_stride_h = M * H * dqk, H * dqk, dqk
    p.v_stride_b, p.v_stride_m, p.v_stride_h = M * H * dv, H * dv, dv
    p.o_stride_b, p.o_stride_n, p.o_stride_h = N * H * dv, H * dv, dv
    p.scale, p.dtype, p.m_total, p.impl, p.causal = 0.125, _lib.PCV_BF16, M, _lib.PCV_IMPL_AUTO, causal
    f = _lib.DecodeFp8()
    f.k_descale, f.v_descale = 5 << 20, 6 << 20
    rows = _lib.DevRows()
    rows.bounds, rows.capacity = 7 << 20, M
    return p, f, rows


def _call(entry, p, f, rows, band, supported):
    lib = _lib.lib()
    args = (ctypes.byref(p),) + ((ctypes.byref(f),) if entry.endswith("fp8") else ()) + (
        ctypes.byref(rows) if rows is not None else None, band)
    if supported:
        return getattr(lib, entry + "_supported")(*args)
    return getattr(lib, entry)(*args, None)


def _refine(p, f, rows, what):
    if what == "partial":
        p.write_partial = 1
        p.part_o = p.part_m = p.part_l = 8 << 20
    elif what == "shard":
        p.m_total, p.m_offset = p.M + 100, 100
    elif what == "k_stride":
        p.k_stride_m = p.H * p.dqk + 4
    elif what == "q_stride":
        p.q_stride_n = p.H * p.dqk + 4
    elif what == "q_align":
        p.q = (1 << 20) + 8
    elif what == "v_align":
        p.v = (3 << 20) + 4
    elif what == "dtype":
        p.dtype = _lib.PCV_E4M3
    elif what == "impl":
        p.impl = _lib.PCV_IMPL_DECODE
    elif what == "bounds":
        rows.bounds = None
    elif what == "capacity":
        rows.capacity = 0
    elif what == "capacity_m":
        rows.capacity = p.M - 1
    elif what == "noncausal":
        p.causal = 0
    return p, f, rows


# (entries, params, refinement, band, reason): entries 0 = 16-bit, 1 = e4m3, 2 = both
REFUSALS = [
    (2, {"N": 65}, None, 0, b"more than 64 query rows"),
    (2, {}, "noncausal", 4, b"a band needs the causal mask"),
    (2, {}, None, -1, b"band must be >= 0"),
    (0, {"dqk": 36}, None, 0, b"multiples of 8"),
    (1, {"dqk": 40}, None, 0, b"multiples of 16"),
    (1, {"dv": 24}, None, 0, b"multiples of 16"),
    (2, {"dqk": 272}, None, 0, b"head dim > 256"),
    (2, {"dv": 272}, None, 0, b"head dim > 256"),
    (0, {}, "k_stride", 0, b"multiples of 8 elements"),
    (1, {}, "k_stride", 0, b"multiples of 16 elements"),
    (2, {}, "q_stride", 0, b"multiples of 8 elements"),
    (2, {}, "q_align", 0, b"16-byte aligned"),
    (2, {}, "v_align", 0, b"16-byte aligned"),
    (2, {}, "dtype", 0, b"e4m3 operands"),
    (2, {}, "impl", 0, b"impl must be AUTO"),
    (2, {}, "bounds", 0, b"bounds is NULL"),
    (2, {}, "capacity", 0, b"capacity must be >= 1"),
    (2, {}, "capacity_m", 0, b"M must equal rows->capacity"),
    (2, {}, "partial", 0, b"no write_partial"),
    (2, {}, "shard", 0, b"no key shard"),
]


@pytest.mark.parametrize("which,kw,what,band,reason", REFUSALS)
def test_window_refusals_without_gpu(which, kw, what, band, reason):
    lib = _lib.lib()
    for e, entry in enumerate(ENTRIES):
        if which not in (e, 2):
            continue
        p, f, rows = _refine(*_params(**kw), what)
        assert _call(entry, p, f, rows, band, True) == 0, entry
        assert reason in lib.pcv_last_error(), (entry, lib.pcv_last_error())
        assert _call(entry, p, f, rows, band, False) != 0, entry
        assert reason in lib.pcv_last_error(), (entry, lib.pcv_last_error())


def test_window_null_arguments():
    lib = _lib.lib()
    p, f, rows = _params()
    for entry in ENTRIES:
        assert _call(entry, p, f, None, 0, True) == 0 and b"rows is NULL" in lib.pcv_last_error()
        assert _call(entry, p, f, None, 0, False) != 0 and b"rows is NULL" in lib.pcv_last_error()
        need = ctypes.c_size_t(0)
        assert getattr(lib, entry + "_workspace_bytes")(None, ctypes.byref(need)) != 0
        assert b"params is NULL" in lib.pcv_last_error()
        assert getattr(lib, entry + "_workspace_bytes")(ctypes.byref(p), None) != 0
        assert b"bytes is NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_cached_window_fp8_supported(ctypes.byref(p), None, ctypes.byref(rows), 0) == 0
    assert b"fp8 params are NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_cached_window_fp8(ctypes.byref(p), None, ctypes.byref(rows), 0, None) != 0
    f.k_descale = None
    assert lib.pcv_attn_cached_window_fp8_supported(ctypes.byref(p), ctypes.byref(f), ctypes.byref(rows), 0) == 0
    assert b"k_descale / v_descale are NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_cached_window_supported(None, ctypes.byref(rows), 0) == 0
    assert b"params is NULL" in lib.pcv_last_error()


@pytest.mark.parametrize("N,M,dqk,dv,band", [(1, 1, 16, 16, 0), (2, 300, 96, 96, 1), (64, 16384, 128, 128, 6144),
                                             (64, 70, 256, 256, 64), (33, 100, 256, 16, 0)])
def test_window_accepts_its_range(N, M, dqk, dv, band):
    lib = _lib.lib()
    for entry in ENTRIES:
        p, f, rows = _params(N=N, M=M, dqk=dqk, dv=dv)
        assert _call(entry, p, f, rows, band, True) == 1, (entry, lib.pcv_last_error())
    p, f, rows = _params(N=N, M=M, dqk=dqk + 8 if dqk < 256 else dqk, dv=dv)
    assert _call(ENTRIES[0], p, f, rows, band, True) == 1, lib.pcv_last_error()   # odd multiples of 8: 16-bit rows


@pytest.mark.parametrize("B,H,N,M,dqk,dv", [(1, 1, 1, 1, 16, 16), (2, 2, 8, 300, 64, 64), (8, 8, 64, 16384, 128, 128),
                                            (16, 8, 16, 6208, 128, 128), (1, 1, 5, 65536, 256, 256),
                                            (4, 3, 17, 1000, 40, 24)])
def test_workspace_matches_the_restatement(B, H, N, M, dqk, dv):
    lib = _lib.lib()
    p, _, _ = _params(N=N, M=M, dqk=dqk, dv=dv, B=B, H=H)
    for entry in ENTRIES:
        need = ctypes.c_size_t(0)
        assert getattr(lib, entry + "_workspace_bytes")(ctypes.byref(p), ctypes.byref(need)) == 0
        assert need.value == WV.workspace_bytes(B, H, N, M, dqk, dv, device_sms())


@pytest.mark.parametrize("sms", [132, 78])
@pytest.mark.parametrize("B,H,cap", [(1, 1, 1), (1, 1, 200), (3, 2, 805), (8, 8, 16384), (16, 12, 6208)])
def test_split_plan_covers_every_window_once(sms, B, H, cap):
    """Every key of any window (clamped to the arena) is covered by exactly one split, in order; no split reaches past
    the window; at most nsplit splits are non-empty."""
    pl = WV.plan(B, H, cap, 128, 128, sms)
    rng = random.Random(cap * 31 + sms)
    wins = [(0, cap), (-5, 3), (cap - 1, cap + 9), (10, 10), (12, 4), (cap // 3, cap // 3 + 64),
            (cap // 3 + 1, cap // 3 + 66)]
    wins += [tuple(sorted(rng.randrange(-3, cap + 4) for _ in range(2))) for _ in range(40)]
    for b0, b1 in wins:
        w0, wend = WV.clamp_window(b0, b1, cap)
        covered = []
        for kb, ke in WV.split_tiles(b0, b1, cap, pl["nsplit"]):
            assert w0 <= kb <= ke <= max(w0, wend), (b0, b1, kb, ke)
            assert (kb - w0) % WV.KEYS == 0
            covered += range(kb, ke)
        assert covered == list(range(w0, max(w0, wend))), (b0, b1)
    # the full arena: the window kernel's split is pcv_attn_cached_fp8's
    from cached_fp8_variants import split_ranges
    assert [r for r in WV.split_tiles(0, cap, cap, pl["nsplit"])] == split_ranges(cap, pl)


def test_variant_matrix_reaches_every_instantiation():
    reach = WV.reachable_variants()
    assert len(reach) == 16
    cover = {WV.variant_of(dt, kind, dv) for dt, kind, _, dv in WV.VARIANT_CASES}
    assert cover == reach, reach - cover


def test_window_instantiations_have_no_spills_and_no_serialised_wgmma():
    kernels, text = cached_kernel_entries(win=True)
    if kernels is None:
        pytest.skip("the library was not built in this tree")
    assert len(kernels) == 16, len(kernels)
    for e in kernels:
        assert "0 bytes spill stores, 0 bytes spill loads" in e, e[:300]
    assert "C7515" not in text and "C7512" not in text


def test_row_keys_restate_the_one_token_windows():
    """A band W over a window ending at row `end` gives query i the keys of the one-token window of row r_i:
    [max(0, r_i + 1 - W), r_i + 1), when the window starts at the first row's begin."""
    for W in (1, 3, 48, 160):
        for row in (0, 5, 47, 48, 200):
            for k in (1, 2, 5, 64):
                b0, b1 = max(0, row + 1 - W), row + k
                for i in range(k):
                    r = row + i
                    lo, hi, cf = WV.row_keys(i, k, b0, b1, 10_000, W, True)
                    assert (lo, hi, cf) == (max(0, r + 1 - W), r + 1, r + 1)


EMU_CASES = [(case, N, win, band) for case in WV.VARIANT_CASES for N, win, band in
             ((5, (3, 68), 0), (64, (1, 300), 64), (2, (7, 205), 17), (9, (40, 45), 3), (63, (0, 320), 400))]


@pytest.mark.parametrize("case,N,win,band", EMU_CASES,
                         ids=[f"{WV.case_id(c)}-n{N}-w{w[0]}_{w[1]}-band{bd}" for c, N, w, bd in EMU_CASES])
def test_emulation_stays_within_half_the_gate(case, N, win, band):
    """The kernel's arithmetic (window_variants.emulate) against fp64 attention on each row's keys: at most half of the
    element-wise gate of the GPU tests, with left padding and a wholly padded batch row."""
    dt, kind, dqk, dv = case
    B, H, cap = 3, 2, 320
    q, k, v, kd, vd, k64, v64 = WV.random_operands(B, B, N, cap, H, dqk, dv, dt, kind, seed=N + win[0] + dqk)
    pad = left_pad(B, cap)
    got = WV.emulate(q, k, v, kd, vd, H, 0.3, win[0], win[1], band, pad, True, dt)
    pl = WV.plan(B, H, cap, dqk, dv)
    ref, bound = WV.reference_and_bound(q, k64, v64, H, 0.3, win[0], win[1], band, pad, True, dt, pl)
    assert torch.isfinite(got).all()
    ratio = ((got.double() - ref).abs() / torch.where(bound > 0, bound, 1.0)).max().item()
    print(f"[emulation] {WV.case_id(case)} N={N} window={win} band={band}: worst err / gate {ratio:.3f}")
    assert ratio <= 0.5, ratio


# ---- GraphedDecoder: k-token steps and rewind -----------------------------------------------------------------------
def _state(n0, prefix, max_seq_len, max_latents):
    """The decoder's one-token state after prefill, built as prefill builds it."""
    from perceiver_io_b200.generation import decode_windows

    w = decode_windows(n0, prefix, 1, max_seq_len, max_latents)[0]
    rows = (n0, n0 - prefix)
    b = torch.tensor([[w.ca_begin, w.ca_end, rows[0], 1, rows[0], 0],
                      [w.sa_begin, w.sa_end, rows[1], 1, rows[1], 0]], dtype=torch.int32)
    return b, torch.tensor([0, 1, 1, 0, 1, 0], dtype=torch.int32), torch.tensor([max_seq_len, max_latents],
                                                                                 dtype=torch.int32)


SCHEDULES = [
    # (prompt_len, prefix_len, max_seq_len, max_latents, ops): ("e", k) extend, ("r", n) rewind
    (20, 0, 64, 48, [("e", 3), ("e", 5), ("r", 2), ("e", 16), ("e", 1), ("e", 40)]),     # the latents fill mid-step
    (120, 90, 160, 48, [("e", 64), ("r", 10), ("e", 5), ("r", 5), ("e", 16), ("e", 3)]),  # k > max_latents, both slide
    (160, 112, 160, 48, [("e", 2), ("e", 64), ("r", 64), ("e", 64)]),                    # a full context from the start
    (5, 4, 8, 2, [("e", 7), ("r", 3), ("e", 3), ("e", 1), ("r", 1), ("e", 9)]),          # windows narrower than k
]


@pytest.mark.parametrize("n0,prefix,max_seq_len,max_latents,plan", SCHEDULES)
def test_extend_and_rewind_give_every_token_its_one_token_window(n0, prefix, max_seq_len, max_latents, plan):
    """Through extend(k) and rewind(n) as GraphedDecoder runs them (extend_bounds, then advance_bounds_ by k; rewind
    advance_bounds_ by -n), the band window of every fed token equals the window the one-token truncation loop gives
    the token at that row; the state after each call is the one-token loop's state for the next token."""
    from perceiver_io_b200.generation import advance_bounds_, extend_bounds

    b, inc, wmax = _state(n0, prefix, max_seq_len, max_latents)
    fed = 0
    for op, n in plan:
        if op == "r":
            advance_bounds_(b, inc, wmax, -n)
            fed -= n
            continue
        kb = extend_bounds(b, n)
        loop = _truncation_loop(n0, prefix, fed + n, max_seq_len, max_latents)[fed:]
        for i in range(n):
            ca_lo, ca_hi, _ = WV.row_keys(i, n, int(kb[0, 0]), int(kb[0, 1]), 10_000, max_seq_len, True)
            sa_lo, sa_hi, _ = WV.row_keys(i, n, int(kb[1, 0]), int(kb[1, 1]), 10_000, max_latents, True)
            assert (ca_lo, ca_hi, sa_lo, sa_hi) == loop[i][:4], (op, n, i)
        # appends and rotations start at the first token's row
        assert kb[:, 2].tolist() == [n0 + fed, n0 - prefix + fed] and torch.equal(kb[:, 2], kb[:, 4])
        advance_bounds_(b, inc, wmax, n)
        fed += n
        nxt = _truncation_loop(n0, prefix, fed + 1, max_seq_len, max_latents)[fed]
        assert b[0, :2].tolist() == list(nxt[:2]) and b[1, :2].tolist() == list(nxt[2:4])
        assert b[:, 2].tolist() == [n0 + fed, n0 - prefix + fed]


def test_k_row_positions_match_positions_with_left_padding():
    from perceiver_io_b200 import positions
    from perceiver_io_b200.generation import extend_bounds, window_positions, window_positions_rows

    B, n0, prefix, cap, W = 3, 30, 12, 120, 40
    pad = torch.zeros(B, cap, dtype=torch.uint8)
    pad[1, :4] = 1
    pad[2, :n0] = 1                      # a fully padded prompt row
    cols = torch.arange(cap, dtype=torch.int32)
    b, _, _ = _state(n0, prefix, W, 16)
    for k in (1, 2, 7, 64):
        kb = extend_bounds(b, k)
        got = window_positions_rows(pad, kb[0], cols, k, W)
        assert got.shape == (B, k) and got.dtype == torch.int64
        for i in range(k):
            r = n0 + i
            lo = max(0, r + 1 - W)
            shift = pad[:, lo:r + 1].bool().sum(dim=1, keepdim=True)
            assert torch.equal(got[:, i:i + 1], positions(B, r + 1 - lo, shift=shift)[:, -1:]), (k, i)
        if k == 1:
            assert torch.equal(got, window_positions(pad, kb[0, 0:2], cols))


def test_extend_and_rewind_refusals_without_a_gpu():
    from perceiver_io_b200 import GraphedDecoder

    dec = object.__new__(GraphedDecoder)   # the checks that run before any device work
    dec.batch, dec._bounds, dec._remaining, dec._fed, dec.max_new_tokens = 2, None, 0, 0, 8
    with pytest.raises(RuntimeError, match="prefill"):
        dec.extend(torch.zeros(2, 3, dtype=torch.long))
    with pytest.raises(RuntimeError, match="prefill"):
        dec.rewind(1)
    b, inc, wmax = _state(30, 10, 40, 16)
    dec._bounds, dec._inc, dec._wmax, dec._remaining = b, inc, wmax, 8
    for bad in (torch.zeros(2, 0, dtype=torch.long), torch.zeros(2, 65, dtype=torch.long),
                torch.zeros(3, 4, dtype=torch.long), torch.zeros(2, 4, dtype=torch.int32), torch.zeros(2, dtype=torch.long)):
        with pytest.raises(ValueError, match="extend takes"):
            dec.extend(bad)
    with pytest.raises(ValueError, match="step takes"):
        dec.step(torch.zeros(2, 2, dtype=torch.long))
    with pytest.raises(RuntimeError, match="8 of max_new_tokens=8 tokens remain"):
        dec.extend(torch.zeros(2, 9, dtype=torch.long))
    for n in (1, -1, 2.0, True, torch.tensor([1]), "1"):
        with pytest.raises(ValueError, match="rewind"):
            dec.rewind(n)
    dec._fed = 3
    dec.rewind(torch.tensor(1))          # integer-like values: operator.index
    dec.rewind(np.int64(1))
    assert dec._fed == 1 and dec._remaining == 10 and b[0, 1].item() == 29
