"""CPU checks of the M-sharded forward's fused merge (peer_tail_kernel, csrc/pcv_attn_tc.cu:171-269): the variant matrix
reaches every peer count, row slice and V-pass edge that test_gpu_tail_variants.py runs; the flag protocol of the
one-GPU simulation is sound; the merge restated in source order is the fp64 merge; the gates of the GPU test reject
mutants of the rules; and pcv_attn_fwd_sharded refuses buffers the tail cannot address, before any CUDA call."""
import ctypes

import pytest
import torch

import fwd_variants as FV
import merge_variants as MV
import tail_variants as TV
from perceiver_io_b200 import _lib
from tail_variants import TAIL_CASES, case_id


# ---- the matrix ----
def test_matrix_reaches_every_peer_count_and_dtype():
    assert {(c.dt, c.G) for c in TAIL_CASES} == {(dt, G) for dt in TV.DTYPES for G in range(1, 9)}


def test_matrix_reaches_the_row_slice_edges():
    assert any(c.R < c.G for c in TAIL_CASES), "no case where some ranks own no rows"
    empty = [c for c in TAIL_CASES if any(TV.rank_rows(c.R, c.G, r)[0] == TV.rank_rows(c.R, c.G, r)[1]
                                          for r in range(c.G))]
    assert {c.dt for c in empty} == set(TV.DTYPES)
    assert {c.G for c in TAIL_CASES if c.R % c.G} >= set(range(2, 9)), "every G > 1 needs a case with R % G != 0"
    for G in range(1, 5):   # RB > 1: a rank whose last warp iteration is partial (its guard `r < row_end` decides)
        assert any(c.G == G and any((hi - lo) % TV.rows_per_iter(G) for lo, hi in
                                    (TV.rank_rows(c.R, G, r) for r in range(G))) for c in TAIL_CASES), G
    for G in (1, 8):
        assert any(c.G == G and TV.warp_loop_wraps(c.R, G, TV.H100_SMS) for c in TAIL_CASES), G


def test_restated_liveness():
    """RB and the dead sources of every G: G = 3, 5, 6 and 7 leave sources without a row; the live sources of a full
    iteration are RB * G, each (row, rank) once; a partial iteration loads only rows below row_end."""
    assert {G: TV.rows_per_iter(G) for G in range(1, 9)} == {1: 8, 2: 4, 3: 2, 4: 2, 5: 1, 6: 1, 7: 1, 8: 1}
    assert {G for G in range(1, 9) if TV.dead_sources(G)} == {3, 5, 6, 7}
    for G in range(1, 9):
        RB = TV.rows_per_iter(G)
        live = [j for j in range(TV.MAX_PEERS) if TV.source_live(j, G, 100, 10 ** 6)]
        assert sorted(TV.source(j, G) for j in live) == [(rr, g) for rr in range(RB) for g in range(G)]
        assert len(live) + len(TV.dead_sources(G)) == TV.MAX_PEERS
        part = [j for j in range(TV.MAX_PEERS) if TV.source_live(j, G, 100, 101)]
        assert [TV.source(j, G) for j in part] == [(0, g) for g in range(G)]


def test_matrix_reaches_the_v_pass_and_layout_edges():
    dvs = {c.dv for c in TAIL_CASES}
    assert dvs >= {8, 64, 128, 200}
    assert TV.channel_iters(8) == [[0, 1]], "dv = 8: two live lanes"
    it = TV.channel_iters(200)
    assert len(it) == 2 and len(it[0]) == 32 and it[1] == list(range(18)), "dv = 200: a ragged second iteration"
    assert len(FV.nvb_passes(200)) == 2 and TV.cdiv(200, TV.MAX_DV_PASS) == 2, "dv = 200: two V passes"
    assert {c.o_pad for c in TAIL_CASES} >= {0, 8}
    for c in TAIL_CASES:
        assert c.dv % 8 == 0 and c.dqk % 8 == 0 and c.o_pad % 4 == 0 and all(s % 4 == 0 for s in c.strides)
        assert c.mask != "pad" or c.B >= 2, "batch row 1 is the all-padded row"
        assert c.mask != "causal" or c.m_total >= c.N
    for dt in TV.DTYPES:
        assert {(c.dv, c.o_pad > 0) for c in TAIL_CASES if c.dt == dt} >= {(200, True)}, dt


def test_matrix_reaches_the_special_rows():
    """Padding over every shard, padding over one shard, causal shards wholly in the future of row 0 (m = -inf)."""
    pads = [c for c in TAIL_CASES if c.mask == "pad"]
    assert {c.dt for c in pads} == set(TV.DTYPES) and any(c.G > 1 for c in pads)
    for c in pads:
        pad = TV.pad_mask(c)
        assert all(pad[1, a:b].all() for a, b in c.shards)
        if c.G > 1:
            assert pad[0, c.shards[-1][0]:].all() and not all(pad[0, a:b].all() for a, b in c.shards[:-1])
    fut = [c for c in TAIL_CASES if c.mask == "causal" and TV.future_shards(c)]
    assert {c.dt for c in fut} == set(TV.DTYPES) and max(c.G for c in fut) == 8


def test_matrix_reaches_the_split_plan():
    """Some cases' shards take the split plan on 132 SMs, so tc_combine_kernel writes the rank's state before the tail;
    others take the whole-unit plan.  (The GPU test asserts the plan again with the device's SM count.)"""
    split = {}
    for c in TAIL_CASES:
        counts, _ = FV.plan_segments(c.B, c.H, c.N, c.Ms, TV.H100_SMS, False)
        split[c] = counts["slots"] > 0 and counts["units"] > 0
    assert {c.dt for c in TAIL_CASES if split[c]} == set(TV.DTYPES)
    assert any(split[c] and c.dv > TV.MAX_DV_PASS for c in TAIL_CASES), "a split plan with two V passes"
    assert not all(split.values())


# ---- the flag protocol of the one-GPU simulation ----
@pytest.mark.parametrize("G", range(1, 9))
def test_sequential_ranks_satisfy_every_wait(G):
    """Epochs 1..3, ranks in the GPU test's order (G-1 first): before every launch preset_flags makes the wait set true,
    and a launch writes exactly written_words (the counter advancing by one grid).  Before the preset the wait set
    holds only for the epoch's last rank (the preset is what makes every other launch safe), and after epoch 1 a launch at a grid that differs
    from the last epoch's is refused by the predicate."""
    grid = TV.H100_SMS
    flags = torch.zeros(G, TV.FLAG_WORDS, dtype=torch.int64)
    for e in (1, 2, 3):
        ran = set()
        for r in [G - 1] + list(range(G - 1)):
            assert TV.wait_set_satisfied(flags, r, G, e, grid) == (ran == set(range(G)) - {r})
            TV.preset_flags(flags, r, G, e)
            assert TV.wait_set_satisfied(flags, r, G, e, grid)
            assert e == 1 or not TV.wait_set_satisfied(flags, r, G, e, grid + 1)
            assert not TV.wait_set_satisfied(flags, r, G, e + 1, grid)
            before = flags.clone()
            for blk, w in TV.written_words(r, G):    # the launch
                flags[blk, w] = before[r, w] + grid if w == TV.ARRIVE_WORD else (7 if w in TV.STAMP_WORDS else e)
            changed = {(int(a), int(b)) for a, b in (flags != before).nonzero()}
            assert changed <= TV.written_words(r, G)
            ran.add(r)
        assert (flags[:, :2 * G] == e).all() and (flags[:, TV.ARRIVE_WORD] == e * grid).all()
        assert not flags[:, 2 * G:TV.ARRIVE_WORD].any() and not flags[:, TV.STAMP_WORDS[-1] + 1:].any()


# ---- the merge restated, and the gates against mutants ----
EMU_SHAPES = [(G, R, dv) for G in range(1, 9) for R, dv in ((3, 8), (37, 200), (64, 64))]


@pytest.mark.parametrize("G, R, dv", EMU_SHAPES)
def test_restated_merge_is_the_fp64_merge(G, R, dv):
    """On dyadic states (every row kind: live, filled, -inf parts) the restatement in source order is RN16 of the fp64
    merge bit for bit, and passes both gates of the GPU test."""
    po, pm, pl = MV.dyadic_states(G, R, dv, seed=G * 100 + R + dv)
    for dt in TV.DTYPES:
        dtype = TV.TORCH_DTYPE[dt]
        want = TV.reference_rows(po, pm, pl, dtype)
        first, outs = TV.emulate_all(po, pm, pl, dtype)
        TV.gate_one_rank(first, *TV.rank_rows(R, G, G - 1), want, what=f"G={G} R={R}")
        TV.gate_complete(outs, want, what=f"G={G} R={R}")


def _caught(po, pm, pl, dtype, mut):
    G, R, _ = po.shape
    want = TV.reference_rows(po, pm, pl, dtype)
    try:
        first, outs = TV.emulate_all(po, pm, pl, dtype, mut)
        TV.gate_one_rank(first, *TV.rank_rows(R, G, G - 1), want)
        TV.gate_complete(outs, want)
    except (AssertionError, TV.AddressError) as ex:
        return type(ex).__name__
    return None


@pytest.mark.parametrize("mut", TV.TAIL_MUTANTS)
def test_gates_reject_mutant(mut):
    """Every mutant is rejected at every G where it changes anything:
    - the slice one row early by the value gates (a row outside the rank's slice written) or, where it starts a
      slice at row -1, by the restatement's address check;
    - RB = 8 / G + 1 by the value gates (a row merged from the wrong sources or never written) wherever a slice is
      longer than RB;
    - l without the weights by the comparison with the fp64 merge, on rows whose live parts have different maxima;
    - the dropped dead-source guard by the restatement's address check: the last rank's partial iteration loads rows
      past R, a read beyond the allocation on the device.  No value gate can see it, since no row uses a dead source."""
    caught = {}
    for G in range(1, 9):
        for R, dv in ((3, 8), (37, 200), (64, 64)):
            po, pm, pl = MV.dyadic_states(G, R, dv, seed=G + R)
            caught[(G, R)] = _caught(po, pm, pl, torch.bfloat16, mut)
    print(f"[tail mutant] {mut}: {caught}")
    if mut == "slice_off_by_one":
        assert all(caught[(G, R)] is not None for G, R in caught if G > 1)
        assert all(caught[(1, R)] is None for R in (3, 37, 64)), "G = 1 has no row_begin > 0"
    elif mut == "rb_plus_one":
        for (G, R), v in caught.items():
            longest = max(hi - lo for lo, hi in (TV.rank_rows(R, G, r) for r in range(G)))
            assert v == ("AssertionError" if longest > TV.rows_per_iter(G) else None), (G, R, v)
    elif mut == "unweighted_l":   # at G = 1 every weight is 1
        assert all((v == "AssertionError") == (G > 1) for (G, R), v in caught.items())
    else:
        for (G, R), v in caught.items():
            lo, hi = TV.rank_rows(R, G, G - 1)
            past = (hi - lo) % TV.rows_per_iter(G) != 0 or bool(TV.dead_sources(G))
            assert v == ("AddressError" if past else None), (G, R, v)


# ---- part 4: the fused entry refuses buffers the tail cannot address ----
def _fake_call(**change):
    """pcv_attn_fwd_sharded with plausible, never dereferenced addresses: 16-byte aligned part / out / flags of 3
    ranks, dense strides.  The attention parameters are invalid too (B = 0, which validate_attn refuses before any
    CUDA call), so no call of this test can reach the device, whichever check runs first."""
    G, H, N, dv = 3, 2, 5, 64
    p = _lib.AttnParams()
    p.q, p.k, p.v = 0x10000, 0x20000, 0x30000
    p.B, p.H, p.N, p.M, p.dqk, p.dv, p.scale = 0, H, N, 32, 64, dv, 0.125
    p.m_total, p.dtype = 96, _lib.PCV_BF16
    f = _lib.ShardFuse()
    for g in range(G):
        f.part[g], f.out[g], f.flags[g] = 0x100000 + 0x10000 * g, 0x200000 + 0x10000 * g, 0x300000 + 0x1000 * g
    f.o_stride_b, f.o_stride_n, f.o_stride_h = N * H * dv, H * dv, dv
    f.num_peers, f.rank, f.epoch = G, 1, 1
    for k, v in change.items():
        if isinstance(v, tuple):
            getattr(f, k)[v[0]] = v[1]
        else:
            setattr(f, k, v)
    lib = _lib.lib()
    before = _lib.launch_count()
    rc = lib.pcv_attn_fwd_sharded(ctypes.byref(p), ctypes.byref(f), None)
    assert _lib.launch_count() == before
    return rc, lib.pcv_last_error()


@pytest.mark.parametrize("change, reason", [
    (dict(part=(0, 0x100004)), b"part[0] must be 16-byte aligned"),
    (dict(part=(1, 0x110008)), b"part[1] must be 16-byte aligned"),   # the rank's own state
    (dict(part=(2, 0x120004)), b"part[2] must be 16-byte aligned"),
    (dict(out=(0, 0x200004)), b"out[0] must be 8-byte aligned"),
    (dict(out=(2, 0x220002)), b"out[2] must be 8-byte aligned"),
    (dict(flags=(2, 0x302002)), b"flags[2] must be 4-byte aligned"),
    (dict(o_stride_n=2 * 64 + 2), b"multiples of 4 elements"),
    (dict(o_stride_b=5 * 2 * 64 + 1), b"multiples of 4 elements"),
    (dict(o_stride_h=66), b"multiples of 4 elements"),
])
def test_fused_entry_refuses_unaddressable_buffers(change, reason):
    rc, msg = _fake_call(**change)
    assert rc == 1 and b"attn_fwd_sharded" in msg and reason in msg, (rc, msg)


def test_fused_entry_passes_addressable_buffers_to_the_shape_checks():
    """The aligned buffers pass the new checks: the call gets to validate_attn, which refuses B = 0."""
    rc, msg = _fake_call()
    assert rc == 1 and b"B=0" in msg, (rc, msg)
    rc, msg = _fake_call(o_stride_n=2 * 64 + 8, part=(0, 0x100010), out=(1, 0x210008), flags=(2, 0x302004))
    assert rc == 1 and b"B=0" in msg, (rc, msg)
