"""-m gpu: every instantiation of the streaming decode kernel (attn_decode_kernel<T, LPK, NQ, FP8, WIN>,
csrc/pcv_attn_decode.cu) at its split, window and mask edges.  The matrix, the restated schedule and the exact
expectations live in decode_variants.py; test_decode_variants_cpu.py checks that the matrix covers every instantiation,
that the shapes have their structure, that the restated split is the library's, and that the probes and the gate see the
bugs they are for.

Two exact probes, compared bit for bit:
  - count probe: q = 0, so every live score is exactly 0 and every masked one -FLT_MAX; V is 0 except at the keys under
    test (split, block and share edges, diagonals: 1, 2 or 4) and at padded keys (8).  The output is RN16(S / L) of the
    integer sum S and count L of the row's live keys (all its keys when none is live); the 16-bit partial state is
    (S, 0 or -FLT_MAX, L) exactly;
  - needle probe: query row n sees one channel c_n, and K is zero on it except at one needle key per (b, h, n), which
    scores ~185 (log2 units) above every other key.  Found, the output is RN16(v[needle]); masked or outside the
    window, the row is the count probe's.
Random operands then go through the derived gate row by row and the element-wise gate of the decode arithmetic
(gpu_util.decode_element_bound)."""
import pytest
import torch

import decode_variants as DV
from decode_variants import (CAPACITY, EDGE_SHAPES, NEEDLE_SCALE, SHORT_SHAPE, VARIANT_CASES, WIN_B, WIN_H, WIN_NSPLIT,
                             WINDOWS, case_id, check_schedule, check_window, choose_split, count_expect, count_operands,
                             count_state, edge_keys, key_sets, lanes_per_key, needle_candidates, needle_expect,
                             needle_operands, needle_rounds, needles, nq_of, serial_depth, split_ranges, v_descale,
                             variant_of, window_clamp, window_ranges)
from gpu_util import FLT_MAX, assert_decode_elements

pytestmark = pytest.mark.gpu

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
FULL_B, FULL_H, FULL_M = 3, 4, 1153     # EDGE_SHAPES["ragged_one"] at B*H = 12: 4 splits of 384 keys, the last of 1
CUDA = "cuda"


def _plan(B, H, M):
    """(nsplit, keys_per_split) as the library plans them on this device."""
    return choose_split(B, H, M, DV.device_sms())


def _ops():
    from perceiver_io_b200 import ops
    return ops


def _pad(B, M, marks, seed):
    """Batch row 0: ~15 % of the keys padded, every third key under test among them; row 1 unpadded; row 2 wholly
    padded (every key counts: the uniform average)."""
    g = torch.Generator(device=CUDA).manual_seed(seed)
    pad = torch.rand(B, M, generator=g, device=CUDA) < 0.15
    pad[0, list(marks)[1::3]] = True
    if B > 1:
        pad[1] = False
    if B > 2:
        pad[2] = True
    return pad


def _descales(case, H):
    """(k_descale, v_descale) of an e4m3 case, made before any graph capture; (None, None) otherwise."""
    if not case[1]:
        return None, None
    return torch.ones(H, device=CUDA), v_descale(H, case[4], CUDA)


def _run(case, q, k, v, H, scale, pad, causal, bounds=None, desc=(None, None)):
    ops = _ops()
    fp8, win = case[1], case[2]
    kd, vd = desc
    if win:
        return ops.attention_decode_window(q, k, v, bounds, H, scale, pad_mask=pad, causal=causal, k_descale=kd,
                                           v_descale=vd)
    if fp8:
        return ops.attention_decode_fp8(q, k, v, kd, vd, H, scale, pad_mask=pad, causal=causal)
    return ops.attention(q, k, v, H, scale, pad_mask=pad, causal=causal, impl="decode")


def _codes(v, case):
    """V as the expectation builders take it: e4m3 codes as floats (their v_descale passed apart)."""
    return v.float() if case[1] else v


def _record(fn):
    """(graph, static output) of fn() recorded once after one eager warm-up on a side stream."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    return graph, out


def _prefix_view(t, extra=64):
    """t as the first rows of a larger arena: the batch stride is not M * C."""
    B, M, C = t.shape
    arena = torch.zeros(B, M + extra, C, dtype=t.dtype, device="cuda")
    arena[:, :M] = t
    return arena[:, :M]


def _assert_bits(got, want, what):
    g, w = got, want.to(got.device)
    assert g.dtype == w.dtype and g.shape == w.shape, (what, g.dtype, w.dtype, g.shape, w.shape)
    eq = (g.view(torch.int16) == w.view(torch.int16)) | ((g == 0) & (w == 0))
    if not bool(eq.all()):
        g, w, eq = g.cpu(), w.cpu(), eq.cpu()
        bad = (~eq).nonzero()
        b, n, c = (int(x) for x in bad[0])
        raise AssertionError(f"{what}: {bad.shape[0]} of {eq.numel()} outputs differ; first at (b={b}, n={n}, "
                             f"channel {c}): got {g[b, n, c].item()!r} want {w[b, n, c].item()!r}")


def _v_scale(case, H):
    return v_descale(H, case[4], CUDA) if case[1] else None


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---- the exact probes of the non-window kernels ----
def _count_full(case, B, H, M, causal, seed, bcast=False, prefix=False):
    """The count probe of the non-window kernel (twice, bit-equal); the 16-bit partial state as well."""
    dt, fp8, _win, dqk, dv, N = case
    dtype = DTYPE[dt]
    lpk, nq = lanes_per_key(dqk, dv, fp8), nq_of(N)
    ranges = split_ranges(M, *_plan(B, H, M))
    marks = edge_keys(ranges, lpk, nq, fp8, extra=[M - N + i for i in range(N)], M=M)
    pad = _pad(B, M, marks, seed)
    q, k, v = count_operands(B, 1 if bcast else B, N, M, H, dqk, dv, marks, pad, fp8, dtype, seed, CUDA)
    if prefix:
        k, v = _prefix_view(k), _prefix_view(v)
    desc = _descales(case, H)
    what = f"count {case_id(case)} B={B} H={H} M={M} causal={causal} bcast={bcast} prefix={prefix}"
    out = _run(case, q, k, v, H, 1.0, pad, causal, desc=desc)
    in_range, live = key_sets(B, N, M, pad, causal, device=CUDA)
    _assert_bits(out, count_expect(_codes(v, case), H, in_range, live, dtype, _v_scale(case, H)), what)
    assert _bits_equal(out, _run(case, q, k, v, H, 1.0, pad, causal, desc=desc)), f"{what}: two calls differ"
    if not fp8:  # the partial state: (S, 0 or -FLT_MAX, L) exactly
        po, pm, pl = _ops().attention_partial(q, k, v, H, 1.0, pad_mask=pad, causal=causal, impl="decode")
        S, L, any_live = count_state(v, H, in_range, live)
        assert torch.equal(po.double(), S), f"{what}: partial o != the integer sum of V"
        assert torch.equal(pl.double(), L), f"{what}: partial l != the key count"
        assert torch.equal(pm, torch.where(any_live, 0.0, -FLT_MAX).float()), f"{what}: partial m"


def _needle_full(case, B, H, M, causal, seed, bcast=False, prefix=False):
    """The needle probe of the non-window kernel, in rounds until every candidate key of every batch row held a
    needle."""
    dt, fp8, _win, dqk, dv, N = case
    dtype = DTYPE[dt]
    lpk, nq = lanes_per_key(dqk, dv, fp8), nq_of(N)
    ranges = split_ranges(M, *_plan(B, H, M))
    pad = _pad(B, M, edge_keys(ranges, lpk, nq, fp8), seed)
    in_range, live = key_sets(B, N, M, pad, causal, device=CUDA)
    cands = [needle_candidates(N, 0, M, ranges, pad, b, causal, lpk, nq, fp8) for b in range(B)]
    desc = _descales(case, H)
    placed = [set() for _ in range(B)]
    for r in range(needle_rounds(cands, H, N)):
        nd = needles(B, H, N, cands, r)
        for b in range(B):
            placed[b] |= set(nd[b].flatten().tolist())
        q, k, v = needle_operands(B, 1 if bcast else B, N, M, H, dqk, dv, nd, fp8, dtype, seed + r, CUDA)
        if prefix:
            k, v = _prefix_view(k), _prefix_view(v)
        out = _run(case, q, k, v, H, NEEDLE_SCALE, pad, causal, desc=desc)
        want = needle_expect(_codes(v, case), H, in_range, live, nd, dtype, _v_scale(case, H))
        _assert_bits(out, want, f"needle {case_id(case)} B={B} H={H} M={M} causal={causal} bcast={bcast} round {r}")
    assert placed == [set(c) for c in cands], "a candidate key never held a needle"


# ---- the exact probes of the window kernels: one graph, replayed over every window ----
def _window_probe(case, causal, seed, needle=False, bcast=False, prefix=False):
    """The count (or needle) probe of a window variant on every window of WINDOWS, inside one recorded graph replayed
    with the window, q, K and V rewritten in device memory; the needle probe takes as many rounds per window as put a
    needle on every candidate key.  `bcast`: one q row set for every batch row (q_stride_b = 0); `prefix`: the arenas
    are the first CAPACITY rows of larger ones.  Two replays are bit-equal."""
    dt, fp8, _win, dqk, dv, N = case
    dtype = DTYPE[dt]
    B, H, M = WIN_B, WIN_H, CAPACITY
    lpk, nq = lanes_per_key(dqk, dv, fp8), nq_of(N)
    assert _plan(B, H, M)[0] == WIN_NSPLIT   # the arena's 11 * 256 keys cap its plan at 8 splits on any H100
    pad = _pad(B, M, [], seed)
    scale = NEEDLE_SCALE if needle else 1.0
    Bq = 1 if bcast else B
    bounds = torch.tensor([0, 1], dtype=torch.int32, device=CUDA)
    qs, ks, vs = count_operands(B, Bq, N, M, H, dqk, dv, [0], pad, fp8, dtype, seed, CUDA)
    if prefix:
        ks, vs = _prefix_view(ks), _prefix_view(vs)
    desc = _descales(case, H)
    graph, out = _record(lambda: _run(case, qs, ks, vs, H, scale, pad, causal, bounds, desc))
    for name, (w0, w1) in WINDOWS:
        check_window(name, (w0, w1), 4, lpk, nq, fp8)  # the windows are named for N = 4
        a, e = window_clamp(w0, w1, M)
        ranges = window_ranges(w0, w1, M, WIN_NSPLIT)
        in_range, live = key_sets(B, N, M, pad, causal, rng=(a, e), causal_end=e, device=CUDA)
        cands = [needle_candidates(N, a, e, ranges, pad, b, causal, lpk, nq, fp8) for b in range(B)] if e > a else []
        placed = [set() for _ in cands]
        for r in range(needle_rounds(cands, H, N) if needle and cands else 1):
            if needle and cands:
                nd = needles(B, H, N, cands, r)
                for b in range(B):
                    placed[b] |= set(nd[b].flatten().tolist())
                q, k, v = needle_operands(B, Bq, N, M, H, dqk, dv, nd, fp8, dtype, seed + r, CUDA)
                want = needle_expect(_codes(v, case), H, in_range, live, nd, dtype, _v_scale(case, H))
            else:  # the keys next to the window are marked too: a leak from outside moves S
                extra = [e - N + i for i in range(N + 1)] + [a - 1, a, e - 1, e]
                marks = edge_keys(ranges, lpk, nq, fp8, extra=extra, M=M)
                q, k, v = count_operands(B, Bq, N, M, H, dqk, dv, marks, pad, fp8, dtype, seed, CUDA)
                want = count_expect(_codes(v, case), H, in_range, live, dtype, _v_scale(case, H))
            qs.copy_(q)
            ks.copy_(k)
            vs.copy_(v)
            bounds.copy_(torch.tensor([w0, w1], dtype=torch.int32))
            graph.replay()
            _assert_bits(out, want, f"{'needle' if needle else 'count'} {case_id(case)} window {name} {(w0, w1)} "
                                    f"causal {causal} bcast {bcast} prefix {prefix} round {r}")
        if needle and cands:
            assert placed == [set(c) for c in cands], f"window {name}: a candidate key never held a needle"
    first = out.clone()
    graph.replay()
    assert _bits_equal(first, out), f"{case_id(case)}: two replays differ"


@pytest.mark.parametrize("case", VARIANT_CASES, ids=case_id)
def test_count_probe_is_exact(case):
    if case[2]:
        _window_probe(case, causal=True, seed=11)
        _window_probe(case, causal=False, seed=12, bcast=True, prefix=True)
        return
    for causal in (False, True):
        _count_full(case, FULL_B, FULL_H, FULL_M, causal, seed=11)
    _count_full(case, FULL_B, FULL_H, FULL_M, True, seed=12, bcast=True, prefix=True)


@pytest.mark.parametrize("case", VARIANT_CASES, ids=case_id)
def test_needle_probe_is_exact(case):
    if case[2]:
        _window_probe(case, causal=True, seed=21, needle=True)
        _window_probe(case, causal=False, seed=22, needle=True, bcast=True, prefix=True)
        return
    _needle_full(case, FULL_B, FULL_H, FULL_M, True, seed=21)
    _needle_full(case, FULL_B, FULL_H, FULL_M, False, seed=22, bcast=True, prefix=True)


# ---- random operands: the numerics ----
RANDOM_WINDOWS = [("mid_block", (517, 1518)), ("shorter_than_n", (2200, 2202)), ("past_capacity", (2500, 3500))]


@pytest.mark.parametrize("case", VARIANT_CASES, ids=case_id)
def test_random_operands_pass_the_element_gate(case):
    ops = _ops()
    dt, fp8, win, dqk, dv, N = case
    dtype = DTYPE[dt]
    lpk, nq = lanes_per_key(dqk, dv, fp8), nq_of(N)
    B, H, M = (WIN_B, WIN_H, CAPACITY) if win else (FULL_B, FULL_H, FULL_M)
    nsplit, kps = _plan(B, H, M)
    g = torch.Generator(device="cuda").manual_seed(31)
    k = torch.randn(B, M, H * dqk, device="cuda", generator=g)
    v = torch.randn(B, M, H * dv, device="cuda", generator=g)
    pad = torch.rand(B, M, device="cuda", generator=g) < 0.2
    pad[-1] = True
    kd = vd = None
    if fp8:
        kd = (k.reshape(B, M, H, dqk).abs().amax((0, 1, 3)) / 448).float()
        vd = (v.reshape(B, M, H, dv).abs().amax((0, 1)) / 448).float()
        k = ops.fp8_quantize(k.to(dtype), kd, H)
        v = ops.fp8_quantize(v.to(dtype), vd, H)
        kq, vq = ops.fp8_dequantize(k, kd, H, torch.float64), ops.fp8_dequantize(v, vd, H, torch.float64)
    else:
        k, v = k.to(dtype), v.to(dtype)
        kq, vq = k, v
    worst = 0.0
    for gain, causal in ((2.0, True), (6.0, False)):
        q = (gain * torch.randn(B, N, H * dqk, device="cuda", generator=g)).to(dtype)
        scale = dqk ** -0.5
        if win:
            for name, (w0, w1) in RANDOM_WINDOWS:
                a, e = window_clamp(w0, w1, M)
                bounds = torch.tensor([w0, w1], dtype=torch.int32, device="cuda")
                out = ops.attention_decode_window(q, k, v, bounds, H, scale, pad_mask=pad, causal=causal,
                                                  k_descale=kd, v_descale=vd)
                share = -(-(e - a) // nsplit)
                worst = max(worst, assert_decode_elements(
                    out, q, kq[:, a:e], vq[:, a:e], H, scale, pad[:, a:e], causal, dtype,
                    serial_depth(share, nsplit, lpk, nq, fp8), f"{case_id(case)} window {name} gain {gain}"))
        else:
            out = (ops.attention_decode_fp8(q, k, v, kd, vd, H, scale, pad_mask=pad, causal=causal) if fp8
                   else ops.attention(q, k, v, H, scale, pad_mask=pad, causal=causal, impl="decode"))
            worst = max(worst, assert_decode_elements(out, q, kq, vq, H, scale, pad, causal, dtype,
                                                      serial_depth(kps, nsplit, lpk, nq, fp8),
                                                      f"{case_id(case)} gain {gain} causal {causal}"))
    print(f"[decode variant] {variant_of(*case)} {case_id(case)}: worst element-wise err/bound {worst:.3f}")


# ---- named edge shapes ----
EDGE_CASES = {  # shape -> the variants it runs (the widest geometry spread that fits the shape's memory)
    "ragged_one": [("bf16", False, False, 64, 40, 3), ("fp16", True, False, 80, 128, 1)],
    "ragged_mid_step": [("bf16", False, False, 8, 8, 4), ("fp16", False, False, 72, 128, 1),
                        ("bf16", True, False, 64, 32, 2), ("fp16", True, False, 128, 80, 4),
                        ("bf16", False, False, 32, 160, 2)],
    "one_split": [("bf16", False, False, 8, 8, 1), ("fp16", False, False, 8, 8, 4)],
    "middle": [("fp16", False, False, 64, 40, 4), ("bf16", True, False, 160, 32, 1)],
    "cap_256": [("bf16", False, False, 64, 64, 1), ("fp16", True, False, 64, 32, 3)],
}


@pytest.mark.parametrize("shape", list(EDGE_SHAPES))
def test_edge_shapes_are_exact(shape):
    B, H, M = EDGE_SHAPES[shape]
    for case in EDGE_CASES[shape]:
        dt, fp8, _w, dqk, dv, N = case
        if DV.device_sms() == DV.SMS:
            print(check_schedule(shape, lanes_per_key(dqk, dv, fp8), nq_of(N), fp8))
        else:  # the expectations follow this device's plan; test_decode_variants_cpu.py asserts the structure
            print(f"{shape}: structure asserted at {DV.SMS} SMs only; {DV.device_sms()} SMs plan {_plan(B, H, M)}")
        for causal in (False, True):
            _count_full(case, B, H, M, causal, seed=41)
        if B * H <= 16:
            _needle_full(case, B, H, M, True, seed=42)


@pytest.mark.parametrize("fp8", [False, True], ids=["k16", "e4m3"])
def test_short_key_axis_is_one_split(fp8):
    """The e4m3 and window entry points take any M; below 512 keys they run one split."""
    B, H, M = SHORT_SHAPE
    assert _plan(B, H, M)[0] == 1
    for causal in (False, True):
        if fp8:
            _count_full(("bf16", True, False, 64, 64, 3), B, H, M, causal, seed=51)
        case = ("fp16", fp8, True, 64, 64, 3)
        dtype = DTYPE[case[0]]
        marks = edge_keys([(0, M)], lanes_per_key(64, 64, fp8), 4, fp8, extra=[M - 3, M - 2, M - 1])
        pad = _pad(B, M, marks, 53)
        q, k, v = count_operands(B, B, 3, M, H, 64, 64, marks, pad, fp8, dtype, 53, CUDA)
        bounds = torch.tensor([0, M], dtype=torch.int32, device=CUDA)
        out = _run(case, q, k, v, H, 1.0, pad, causal, bounds, _descales(case, H))
        in_range, live = key_sets(B, 3, M, pad, causal, device=CUDA)
        _assert_bits(out, count_expect(_codes(v, case), H, in_range, live, dtype, _v_scale(case, H)),
                     f"window decode on one split, e4m3 {fp8}, causal {causal}")
    if fp8:
        _needle_full(("bf16", True, False, 64, 64, 3), B, H, M, True, seed=52)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_key_shards_partial_state_is_exact(dt):
    """attention_partial(impl="decode") on two key shards [0, 1100) and [1100, 2200) of m_total = 2200, causal: each
    shard's (o, m, l) equals (S, 0 or -FLT_MAX, L) of its own keys under the global right-aligned diagonal."""
    ops = _ops()
    dtype = DTYPE[dt]
    B, H, M, N, d = 3, 2, 2200, 4, 40
    shard = edge_keys(split_ranges(1100, *_plan(B, H, 1100)), 8, 4, False)
    marks = sorted(set(shard) | {1100 + j for j in shard} | {M - N + i for i in range(N)})
    pad = _pad(B, M, marks, 61)
    q, k, v = count_operands(B, B, N, M, H, d, d, marks, pad, False, dtype, 61, CUDA)
    for m0 in (0, 1100):
        sl = slice(m0, m0 + 1100)
        po, pm, pl = ops.attention_partial(q, k[:, sl], v[:, sl], H, 1.0, pad_mask=pad[:, sl], causal=True, m_total=M,
                                           m_offset=m0, impl="decode")
        in_range, live = key_sets(B, N, 1100, pad[:, sl], True, m_total=M, m_offset=m0, device=CUDA)
        S, L, any_live = count_state(v[:, sl], H, in_range, live)
        assert torch.equal(po.double(), S) and torch.equal(pl.double(), L), f"shard {m0}"
        assert torch.equal(pm, torch.where(any_live, 0.0, -FLT_MAX).float()), f"shard {m0}"


# ---- the AUTO routing floor ----
@pytest.mark.parametrize("N", [1, 4])
@pytest.mark.parametrize("M", [1023, 1024])
def test_auto_routing_floor(M, N):
    """M = 1024 is the first key count pcv_attn_fwd runs the decode kernel for: AUTO is bit-equal to impl="decode".
    At M = 1023, impl="decode" is refused for the short key axis and AUTO is bit-equal to the tensor-core kernel."""
    ops = _ops()
    from perceiver_io_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(71)
    B, H, d = 2, 4, 64
    q = (2 * torch.randn(B, N, H * d, device="cuda", generator=g)).bfloat16()
    k = torch.randn(B, M, H * d, device="cuda", generator=g).bfloat16()
    v = torch.randn(B, M, H * d, device="cuda", generator=g).bfloat16()
    pad = torch.zeros(B, M, dtype=torch.bool, device="cuda")
    pad[0, :100] = True
    auto = ops.attention(q, k, v, H, d ** -0.5, pad_mask=pad, causal=True)
    if M >= DV.ROUTING_FLOOR:
        dec = ops.attention(q, k, v, H, d ** -0.5, pad_mask=pad, causal=True, impl="decode")
        assert torch.equal(auto.view(torch.int16), dec.view(torch.int16))
        return
    with pytest.raises(RuntimeError) as exc:
        ops.attention(q, k, v, H, d ** -0.5, pad_mask=pad, causal=True, impl="decode")
    assert "short key axis" in str(exc.value) or b"short key axis" in _lib.lib().pcv_last_error()
    assert ops.tcgen05_supported(q, k, v, H, pad_mask=pad, causal=True)
    tc = ops.attention(q, k, v, H, d ** -0.5, pad_mask=pad, causal=True, impl="tcgen05")
    assert torch.equal(auto.view(torch.int16), tc.view(torch.int16))


# ---- the binary: every restated instantiation is launched ----
def test_profiler_sees_every_instantiation():
    """One count probe per variant case under torch.profiler: the set of attn_decode_kernel<...> instantiations launched
    equals decode_variants.reachable_variants() (56)."""
    import re

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case in {variant_of(*c): c for c in VARIANT_CASES}.values():   # one case per instantiation
            dt, fp8, win, dqk, dv, N = case
            dtype = DTYPE[dt]
            B, H, M = (2, 1, 300) if win or fp8 else (2, 1, 1024)
            q, k, v = count_operands(B, B, N, M, H, dqk, dv, [0], torch.zeros(B, M, dtype=torch.bool), fp8, dtype, 1,
                                     CUDA)
            bounds = torch.tensor([3, 250], dtype=torch.int32, device=CUDA)
            _run(case, q, k, v, H, 1.0, None, False, bounds, _descales(case, H))
        torch.cuda.synchronize()
    pat = re.compile(r"attn_decode_kernel<(__nv_bfloat16|__half), (\d+), (\d+), (true|false), (true|false)>")
    seen, names = set(), set()
    for ev in prof.events():
        if "decode" in ev.name:
            names.add(ev.name)
        m = pat.search(ev.name)
        if m:
            seen.add(({"__nv_bfloat16": "bf16", "__half": "fp16"}[m[1]], int(m[2]), int(m[3]), m[4] == "true",
                      m[5] == "true"))
    want = DV.reachable_variants()
    print(f"[decode variants] profiler saw {len(seen)} of {len(want)} attn_decode_kernel instantiations")
    assert seen == want, (sorted(want - seen, key=str), sorted(seen - want, key=str), sorted(names)[:4])

