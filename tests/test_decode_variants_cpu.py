"""CPU companion of test_gpu_decode_variants.py: the decode variant matrix covers all 56 instantiations, the edge shapes
and windows have the structure they are named for, the restated split is the library's, every key of a split is read
exactly once, the element-wise gate (gpu_util.decode_element_bound) is calibrated on an fp32 emulation of the kernel's
arithmetic, and the exact probes and the gate reject the bugs they are meant to see."""
import ctypes
import itertools
import math

import pytest
import torch

import decode_variants as DV
from decode_variants import (CAPACITY, EDGE_SHAPES, HEAD_DIMS, VARIANT_CASES, WIN_B, WIN_H, WIN_NSPLIT, WINDOWS,
                             check_schedule, check_window, choose_split, count_expect, count_operands, edge_keys,
                             geometry, key_sets, lanes_per_key, needle_candidates, needle_expect, needle_operands,
                             needle_rounds, needles, partition, serial_depth, split_ranges, unroll, v_descale, variant_of,
                             window_clamp, window_ranges)
from gpu_util import FLT_MAX, decode_element_bound

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
LOG2E = 1.4426950408889634
GEOMETRIES = sorted({(lpk, nq, fp8) for (fp8, lpk) in HEAD_DIMS for nq in (1, 4)})


def test_matrix_reaches_all_56_instantiations():
    reach = DV.reachable_variants()
    covered = {variant_of(*c) for c in VARIANT_CASES}
    print(f"[decode matrix] {len(reach)} instantiations, {len(VARIANT_CASES)} cases cover {len(covered)}")
    assert len(reach) == 2 * 2 * 2 * (4 + 3) == 56  # dtype x NQ x WIN x (4 16-bit LPK + 3 e4m3 LPK)
    assert covered == reach, sorted(reach - covered, key=str)
    assert {nq for _, _, nq, _, _ in reach} == {1, 4} and {lpk for _, lpk, _, f, _ in reach if f} == {4, 8, 16}
    # idle lanes / dead chunks: dqk != dv both ways, and one chunk on a 4-lane group
    dims = {(fp8, dqk, dv) for _, fp8, _, dqk, dv, _ in VARIANT_CASES}
    assert (False, 32, 160) in dims and (False, 160, 32) in dims and (True, 32, 160) in dims and (True, 160, 32) in dims
    assert (False, 8, 8) in dims and (True, 16, 16) in dims and (False, 256, 256) in dims and (True, 256, 256) in dims
    assert {N for *_, N in VARIANT_CASES} == {1, 2, 3, 4}


def test_lanes_per_key_rule():
    assert [lanes_per_key(d, d, False) for d in (8, 32, 40, 64, 72, 128, 136, 256)] == [4, 4, 8, 8, 16, 16, 32, 32]
    assert [lanes_per_key(d, d, True) for d in (16, 64, 80, 128, 144, 256)] == [4, 4, 8, 8, 16, 16]
    assert unroll(True, 4) == 2 and unroll(True, 1) == unroll(False, 4) == unroll(False, 1) == 4


@pytest.mark.parametrize("shape", list(EDGE_SHAPES))
def test_edge_shapes_have_their_structure_at_132_sms(shape):
    for lpk, nq, fp8 in GEOMETRIES:
        print(check_schedule(shape, lpk, nq, fp8, 132))


def test_windows_have_their_structure():
    assert WIN_NSPLIT == choose_split(WIN_B, WIN_H, CAPACITY)[0] == 8
    for name, win in WINDOWS:
        for lpk, nq, fp8 in GEOMETRIES:
            desc = check_window(name, win, 4, lpk, nq, fp8)
        print(desc)


def _params(B, H, N, M, dv, dqk=64):
    from perceiver_io_b200 import _lib

    p = _lib.AttnParams()
    p.q, p.k, p.v, p.out = 1 << 20, 2 << 20, 3 << 20, 4 << 20   # never dereferenced: the queries touch no memory
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.q_stride_b, p.q_stride_n, p.q_stride_h = N * H * dqk, H * dqk, dqk
    p.k_stride_b, p.k_stride_m, p.k_stride_h = M * H * dqk, H * dqk, dqk
    p.v_stride_b, p.v_stride_m, p.v_stride_h = M * H * dv, H * dv, dv
    p.o_stride_b, p.o_stride_n, p.o_stride_h = N * H * dv, H * dv, dv
    p.scale, p.dtype, p.m_total, p.impl = 0.125, _lib.PCV_BF16, M, _lib.PCV_IMPL_AUTO
    return p


def test_restated_choose_split_matches_the_library():
    """The split count, recovered from the workspace bytes of the three decode queries.  dv = 64 makes the ws_o block
    B*H*nsplit*NQ*256 bytes, a multiple of 256, so the byte count grows strictly with nsplit and no alignment hides a
    wrong split count.  The library plans with the current device's SM count, 132 without a device."""
    from perceiver_io_b200 import _lib

    lib = _lib.lib()
    sms = DV.device_sms()
    seen = set()
    for B, H, N, M in [(4, 396, 1, 1024), (1, 1, 1, 5000), (1, 1, 3, 65536), (2, 2, 1, 1153), (3, 2, 4, 3000),
                       (1, 1, 1, 300), (2, 2, 2, 500), (1, 8, 1, 20000), (2, 2, 1, 1485), (1, 1, 1, 98000),
                       (5, 3, 2, 7000), (1, 1, 4, 1023)]:
        p = _params(B, H, N, M, 64)
        want = DV.workspace_bytes(B, H, N, M, 64, sms)
        nsplit = choose_split(B, H, M, sms)[0]
        queries = ["pcv_attn_decode_fp8_workspace_bytes", "pcv_attn_decode_window_workspace_bytes"]
        if M >= DV.ROUTING_FLOOR:
            queries.append("pcv_attn_workspace_bytes")
        for q in queries:
            need = ctypes.c_size_t(0)
            assert getattr(lib, q)(ctypes.byref(p), ctypes.byref(need)) == 0, lib.pcv_last_error()
            rows = B * H * DV.nq_of(N)
            a256 = lambda x: (x + 255) // 256 * 256  # noqa: E731
            cands = [n for n in range(1, 257)
                     if a256(rows * n * 64 * 4) + 2 * a256(rows * n * 4) + a256(B * H * 4) == need.value]
            assert len(cands) == 1, (q, B, H, N, M, need.value, cands)
            assert cands[0] == nsplit, (q, B, H, N, M, sms, cands[0], nsplit)
            assert need.value == want
        seen.add(nsplit)
    print(f"[choose_split] split counts walked at {sms} SMs: {sorted(seen)}")
    assert len(seen) >= 5 and 1 in seen and 256 in seen, seen


def _all_ranges():
    out = []
    for shape, (B, H, M) in EDGE_SHAPES.items():
        nsplit, kps = choose_split(B, H, M)
        out.append((shape, 0, M, split_ranges(M, nsplit, kps)))
    for name, win in WINDOWS:
        a, e = window_clamp(*win, CAPACITY)
        out.append((f"window {name}", a, max(a, e), window_ranges(*win, CAPACITY, WIN_NSPLIT)))
    return out


def test_partition_reads_every_key_exactly_once():
    """For every edge shape and window and every (LPK, NQ, FP8) geometry: the splits tile [kb, ke) of the call, and the
    warp loop of each split gives every key of it to exactly one (warp, lane group, block, step)."""
    for (name, k0, kend, ranges), (lpk, nq, fp8) in itertools.product(_all_ranges(), GEOMETRIES):
        keys = []
        for kb, ke in ranges:
            own = partition(kb, ke, lpk, nq, fp8)
            assert sorted(own) == list(range(kb, max(kb, ke))), (name, kb, ke, lpk, nq, fp8)
            keys += list(own)
        assert sorted(keys) == list(range(k0, kend)), (name, lpk, nq, fp8)
        # the (split, warp, group) owners: lane group g of a warp step reads key j0 + u KPW + g
        kpw = geometry(lpk, nq, fp8)[0]
        for kb, ke in ranges[:2]:
            for j, (w, g, r, u) in partition(kb, ke, lpk, nq, fp8).items():
                assert (j - kb) % kpw == g
    print(f"[partition] {len(_all_ranges())} shapes x {len(GEOMETRIES)} geometries: every key read once")


# ---- the fp32 emulation of the kernel's arithmetic ----
def _f32(x):
    return torch.tensor(x, dtype=torch.float32)


def emulate_decode(q, k, v, H, scale, pad, causal, ranges, lpk, nq, fp8, dtype, kd=None, vd=None, causal_end=None,
                   p16=False):
    """attn_decode_kernel's arithmetic in fp32, in its order: scores as per-chunk fp32 sums reduced by the lanes' xor
    tree; per lane group, blocks of kUnroll steps with one running-max rescale each (keys of the group: every KPW-th
    key of the warp's blocks, every 4th block); the v_descale of e4m3 rows on the accumulator; the xor merge of the lane
    groups, the warps in order, the splits in order; o / l rounded to 16 bits.  `p16` rounds each probability to 16
    bits before P V, as the tensor-core kernels do (reported, not gated).  q (Bq, N, H*dqk) and k, v (B, M, H*d) are
    the operands as the kernel reads them (e4m3 codes as floats, with kd (H,) and vd (H, dv))."""
    f32 = torch.float32
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    ch = 16 if fp8 else 8
    kpw, kpb, stride = geometry(lpk, nq, fp8)
    U = unroll(fp8, nq)
    qh = q.to(f32).expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)      # (B, H, N, dqk)
    kh = k.to(f32).reshape(B, M, H, -1).transpose(1, 2)
    vh = v.to(f32).reshape(B, M, H, -1).transpose(1, 2)
    dqk = qh.shape[-1]
    qs = _f32(scale * LOG2E)
    qs = qs * (kd.to(f32)[None, :, None, None] if kd is not None else 1.0)
    qsc = qh * qs
    nch = lpk
    pad_to = nch * ch
    qp = torch.nn.functional.pad(qsc, (0, pad_to - dqk)).reshape(B, H, N, nch, ch)
    kp = torch.nn.functional.pad(kh, (0, pad_to - dqk)).reshape(B, H, M, nch, ch)
    part = torch.zeros(B, H, N, M, nch, dtype=f32)
    for c in range(ch):  # the fma chain of one lane's chunk
        part = part + qp[:, :, :, None, :, c] * kp[:, :, None, :, :, c]
    o = nch // 2
    while o >= 1:        # the xor tree: lane 0 adds lane o at each step
        part = part[..., :o] + part[..., o:2 * o]
        o //= 2
    t = part[..., 0]                                                          # (B, H, N, M)
    end = (M if causal_end is None else causal_end)
    j = torch.arange(M)
    masked = torch.zeros(B, 1, N, M, dtype=torch.bool)
    if pad is not None:
        masked = masked | pad.bool()[:, None, None, :]
    if causal:
        masked = masked | (j[None, :] > torch.arange(N)[:, None] + end - N)[None, None]
    t = torch.where(masked, _f32(-FLT_MAX), t)
    ninf = _f32(-math.inf)
    splits = []
    for kb, ke in ranges:
        G = kpw
        m = torch.full((B, H, N, DV.WARPS, G), -math.inf)
        l = torch.zeros(B, H, N, DV.WARPS, G)
        acc = torch.zeros(B, H, N, DV.WARPS, G, vh.shape[-1])
        r = 0
        while True:
            j0 = kb + (torch.arange(DV.WARPS) + DV.WARPS * r) * kpb                # (W,)
            if not bool((j0 < ke).any()):
                break
            idx = j0[:, None, None] + torch.arange(U)[None, :, None] * kpw + torch.arange(G)[None, None, :]  # (W,U,G)
            valid = (idx < ke) & (j0 < ke)[:, None, None]
            idc = idx.clamp(max=M - 1)
            s = torch.where(valid, t[..., idc], ninf)                         # (B,H,N,W,U,G)
            mb = s.amax(-2)
            m_new = torch.maximum(m, mb)
            skip = m_new == -math.inf
            alpha = torch.where(skip, _f32(1.0), torch.exp2(torch.where(skip, _f32(0.0), m - m_new)))
            mnz = torch.where(skip, _f32(0.0), m_new)
            l = torch.where(skip, l, l * alpha)
            acc = torch.where(skip[..., None], acc, acc * alpha[..., None])
            for u in range(U):
                pe = torch.exp2(s[..., u, :] - mnz)
                pe = torch.where(skip | ~valid[:, u, :], _f32(0.0), pe)
                l = l + pe
                pv = pe.to(dtype).to(f32) if p16 else pe
                vv = vh[:, :, None, idc[:, u, :], :]                          # (B,H,1,W,G,dv)
                acc = acc + pv[..., None] * torch.where(valid[:, u, :, None], vv, _f32(0.0))
            m = torch.where(skip, m, m_new)
            r += 1
        if fp8:
            acc = acc * vd.to(f32)[None, :, None, None, None, :]
        o = 1
        while o < G:     # lane groups: xor shuffle merge (group g with g ^ o)
            perm = torch.arange(G) ^ o
            m_o, l_o, a_o = m[..., perm], l[..., perm], acc[..., perm, :]
            m_new = torch.maximum(m, m_o)
            wa = torch.where(m == -math.inf, _f32(0.0), torch.exp2(m - m_new))
            wb = torch.where(m_o == -math.inf, _f32(0.0), torch.exp2(m_o - m_new))
            l = l * wa + l_o * wb
            acc = acc * wa[..., None] + a_o * wb[..., None]
            m = m_new
            o <<= 1
        m, l, acc = m[..., 0], l[..., 0], acc[..., 0, :]                      # (B,H,N,W), (.., W, dv)
        splits.append(_merge(m, l, acc))
    sm = torch.stack([s_[0] for s_ in splits], -1)
    sl = torch.stack([s_[1] for s_ in splits], -1)
    so = torch.stack([s_[2] for s_ in splits], -2)
    mm, ll, oo = _merge(sm, sl, so)
    out = torch.where(ll[..., None] > 0, oo / ll[..., None], _f32(0.0))
    return out.to(dtype).transpose(1, 2).reshape(B, N, -1)



def _merge(m, l, acc):
    """The fixed-order merge of the warps (or the splits): weights 2^(m_w - max), fma in index order."""
    mm = m.amax(-1)
    o = torch.zeros(acc.shape[:-2] + acc.shape[-1:])
    ll = torch.zeros(mm.shape)
    for w in range(m.shape[-1]):
        wt = torch.where(m[..., w] == -math.inf, _f32(0.0), torch.exp2(m[..., w] - mm))
        o = o + acc[..., w, :] * wt[..., None]
        ll = ll + l[..., w] * wt
    return mm, ll, o


def _random_case(B, N, M, H, dqk, dv, dtype, gain, fp8, seed):
    g = torch.Generator().manual_seed(seed)
    q = (gain * torch.randn(B, N, H * dqk, generator=g)).to(dtype)
    k = torch.randn(B, M, H * dqk, generator=g)
    v = torch.randn(B, M, H * dv, generator=g)
    pad = torch.rand(B, M, generator=g) < 0.2
    pad[-1] = True
    if not fp8:
        return q, k.to(dtype), v.to(dtype), pad, None, None, k.to(dtype), v.to(dtype)
    kd = (k.reshape(B, M, H, dqk).abs().amax((0, 1, 3)) / 448).float()
    vd = (v.reshape(B, M, H, dv).abs().amax((0, 1)) / 448).float()
    k8 = (k.reshape(B, M, H, dqk) / kd[:, None]).to(torch.float8_e4m3fn).float()
    v8 = (v.reshape(B, M, H, dv) / vd).to(torch.float8_e4m3fn).float()
    kq = (k8 * kd[:, None].double()).reshape(B, M, -1)
    vq = (v8 * vd.double()).reshape(B, M, -1)
    return q, k8.reshape(B, M, -1), v8.reshape(B, M, -1), pad, kd, vd, kq, vq


CALIBRATION = [  # dtype, fp8, (dqk, dv), N, window (or None), gain, causal
    ("bf16", False, (64, 40), 4, None, 2.0, True),
    ("fp16", False, (8, 8), 1, None, 6.0, False),
    ("bf16", False, (32, 160), 3, (517, 1518), 6.0, True),
    ("fp16", False, (160, 32), 1, (3, 2000), 2.0, True),
    ("bf16", True, (128, 80), 2, None, 6.0, True),
    ("fp16", True, (256, 256), 1, (2500, 3500), 2.0, False),
    ("bf16", True, (16, 16), 4, (1001, 1066), 6.0, True),
    ("fp16", False, (128, 72), 4, None, 2.0, False),
]


def _calibration(case, seed, p16=False):
    dt, fp8, (dqk, dv), N, win, gain, causal = case
    dtype = DTYPE[dt]
    B, H = 3, 2
    M = CAPACITY if win else 1153
    q, k, v, pad, kd, vd, kq, vq = _random_case(B, N, M, H, dqk, dv, dtype, gain, fp8, seed)
    lpk, nq = lanes_per_key(dqk, dv, fp8), DV.nq_of(N)
    scale = dqk ** -0.5
    nsplit, kps = choose_split(B, H, M)
    if win:
        a, e = window_clamp(*win, M)
        ranges = window_ranges(*win, M, nsplit)
        share = -(-(e - a) // nsplit)
        got = emulate_decode(q, k, v, H, scale, pad, causal, ranges, lpk, nq, fp8, dtype, kd, vd, causal_end=e, p16=p16)
        bound, ref = decode_element_bound(q, kq[:, a:e], vq[:, a:e], H, scale, pad[:, a:e], causal, dtype,
                                          serial_depth(share, nsplit, lpk, nq, fp8))
    else:
        ranges = split_ranges(M, nsplit, kps)
        got = emulate_decode(q, k, v, H, scale, pad, causal, ranges, lpk, nq, fp8, dtype, kd, vd, p16=p16)
        bound, ref = decode_element_bound(q, kq, vq, H, scale, pad, causal, dtype, serial_depth(kps, nsplit, lpk, nq, fp8))
    return got, bound, ref, (q, kq, vq, pad, H, scale, causal, dtype, win)


@pytest.mark.parametrize("i", range(len(CALIBRATION)))
def test_gate_passes_the_emulated_kernel_arithmetic_with_margin(i):
    got, bound, ref, _ = _calibration(CALIBRATION[i], seed=i)
    ratio = ((got.double() - ref).abs() / bound).max().item()
    got16, _, _, _ = _calibration(CALIBRATION[i], seed=i, p16=True)
    r16 = ((got16.double() - ref).abs() / bound).max().item()
    print(f"[decode gate calibration] case {i} {CALIBRATION[i]}: emulated worst err/bound {ratio:.3f}; "
          f"with 16-bit P (the tensor-core kernels' rounding) {r16:.3f}")
    assert ratio <= 0.5, ratio


def test_gate_rejects_a_dropped_key_of_one_percent():
    """The fp64 output with one key left out of a row, that key carrying >= 1 % of the row's probability: the
    element-wise gate rejects it."""
    got, bound, ref, (q, kq, vq, pad, H, scale, causal, dtype, _w) = _calibration(CALIBRATION[0], seed=0)
    B, M, N = kq.shape[0], kq.shape[1], q.shape[1]
    qh = q.double().expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = kq.double().reshape(B, M, H, -1).transpose(1, 2)
    s = (qh * scale) @ kh.transpose(-1, -2)
    s = s.masked_fill(pad[:, None, None, :], -torch.finfo(torch.float64).max)
    s = s.masked_fill(torch.ones(N, M, dtype=torch.bool).triu(M - N + 1), -torch.finfo(torch.float64).max)
    P = s.softmax(-1)
    P[1:] = 0  # batch row 0 only (row 2 is wholly padded)
    b, h, n, j = (int(x) for x in ((P >= 0.01) & (P < 0.05)).nonzero()[0])
    pj = P[b, h, n, j].item()
    assert pj >= 0.01
    vh = vq.double().reshape(B, M, H, -1).transpose(1, 2)
    Pm = s.softmax(-1)
    Pm[b, h, n, j] = 0
    Pm[b, h, n] /= Pm[b, h, n].sum()
    mut = (Pm @ vh).transpose(1, 2).reshape(B, N, -1)
    bad = ((mut - ref).abs() > bound).any().item()
    print(f"[decode gate power] key {j} of row (b={b}, h={h}, n={n}) carries p = {pj:.4f}: rejected {bad}")
    assert bad


# ---- the exact probes: power against the bugs they are meant to see ----
def _bits_differ(a, b):
    return bool((a.view(torch.int16) != b.view(torch.int16)).any())


def _full_probe(dt="bf16", fp8=False, N=4, causal=True):
    B, H, M, dqk, dv = 3, 2, 1153, 64, 64
    dtype = DTYPE[dt]
    lpk, nq = lanes_per_key(dqk, dv, fp8), DV.nq_of(N)
    ranges = split_ranges(M, *choose_split(B, H, M))
    marks = edge_keys(ranges, lpk, nq, fp8, extra=[M - N + i for i in range(N)], M=M)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, marks[1::3]] = True
    pad[0, 500:520] = True
    pad[2] = True
    q, k, v = count_operands(B, B, N, M, H, dqk, dv, marks, pad, fp8, dtype, 5)
    vs = v_descale(H, dv) if fp8 else None
    return dict(B=B, H=H, M=M, N=N, dtype=dtype, ranges=ranges, marks=marks, pad=pad, v=v.float() if fp8 else v,
                vs=vs, causal=causal, dqk=dqk, dv=dv, fp8=fp8, lpk=lpk, nq=nq)


def _expect(P, drop=(), leak=(), causal_end=None, rng=None, vs=None, guard=True):
    in_range, live = key_sets(P["B"], P["N"], P["M"], P["pad"], P["causal"], rng=rng,
                              causal_end=causal_end if causal_end is not None else (rng[1] if rng else None))
    in_range, live = in_range.clone(), live.clone()
    for j in drop:
        in_range[:, :, j] = False
        live[:, :, j] = False
    for b, j in leak:
        live[b, :, j] = True
    out = count_expect(P["v"], P["H"], in_range, live, P["dtype"], P["vs"] if vs is None else vs)
    if not guard:  # o / l of a row that read no key: 0 / 0
        dead = ~in_range.any(-1)
        out = torch.where(dead[:, :, None], torch.full_like(out, float("nan")), out)
    return out


MUTANTS = ["split_boundary_key_dropped", "ragged_last_key_dropped", "padded_key_leaked", "causal_minus_1",
           "causal_plus_1", "window_causal_minus_1", "window_causal_plus_1", "window_begin_minus_1",
           "window_begin_plus_1", "window_end_minus_1", "window_end_plus_1", "empty_split_guard_lost",
           "v_descale_one_channel_over"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_count_probe_rejects_each_mutant(mutant):
    """Each mutant is one of the bugs the kernel could have, applied to the exact expectation; its output differs from
    the true expectation in at least one bit."""
    if mutant.startswith("window") or mutant == "empty_split_guard_lost":
        P = _full_probe()
        P.update(M=CAPACITY, B=WIN_B, H=WIN_H)
        name, win = ("empty", (40, 40)) if mutant == "empty_split_guard_lost" else ("mid_block", (517, 1518))
        a, e = window_clamp(*win, CAPACITY)
        ranges = window_ranges(*win, CAPACITY, WIN_NSPLIT)
        marks = edge_keys(ranges, P["lpk"], P["nq"], False, extra=[e - 4 + i for i in range(5)] + [a - 1, a, e - 1, e],
                          M=CAPACITY)
        pad = torch.zeros(WIN_B, CAPACITY, dtype=torch.bool)
        pad[2] = True
        _q, _k, v = count_operands(WIN_B, WIN_B, 4, CAPACITY, WIN_H, 64, 64, marks, pad, False, torch.bfloat16, 7)
        P.update(pad=pad, v=v)
        want = _expect(P, rng=(a, e))
        mut = {"window_causal_minus_1": lambda: _expect(P, rng=(a, e), causal_end=e - 1),
               "window_causal_plus_1": lambda: _expect(P, rng=(a, e), causal_end=e + 1),
               "window_begin_minus_1": lambda: _expect(P, rng=(a - 1, e), causal_end=e),
               "window_begin_plus_1": lambda: _expect(P, rng=(a + 1, e), causal_end=e),
               "window_end_minus_1": lambda: _expect(P, rng=(a, e - 1)),  # wend also aligns the diagonal
               "window_end_plus_1": lambda: _expect(P, rng=(a, e + 1)),
               "empty_split_guard_lost": lambda: _expect(P, rng=(a, e), guard=False)}[mutant]()
        assert bool((want == 0).all()) if mutant == "empty_split_guard_lost" else True
    else:
        P = _full_probe(fp8=mutant == "v_descale_one_channel_over")
        want = _expect(P)
        M, kps = P["M"], P["ranges"][0][1]
        mut = {"split_boundary_key_dropped": lambda: _expect(P, drop=[kps]),
               "ragged_last_key_dropped": lambda: _expect(P, drop=[M - 1]),
               "padded_key_leaked": lambda: _expect(P, leak=[(0, P["marks"][1])]),
               "causal_minus_1": lambda: _expect(P, causal_end=M - 1),
               "causal_plus_1": lambda: _expect(P, causal_end=M + 1),
               "v_descale_one_channel_over": lambda: _expect(P, vs=P["vs"].roll(-1, 1))}[mutant]()
    assert _bits_differ(want, mut), f"{mutant}: the count probe does not see it"
    print(f"[probe power] count probe rejects {mutant}")


@pytest.mark.parametrize("mutant", ["causal_minus_1", "causal_plus_1", "padded_key_leaked"])
def test_needle_probe_rejects_each_mutant(mutant):
    """The needle probe on the K side: a diagonal shifted by one loses the diagonal needle or finds the one past it;
    a leaked padded key finds a needle placed on it."""
    P = _full_probe()
    B, H, N, M = P["B"], P["H"], P["N"], P["M"]
    cands = [needle_candidates(N, 0, M, P["ranges"], P["pad"], b, True, P["lpk"], P["nq"], False) for b in range(B)]
    rejected = 0
    for r in range(needle_rounds(cands, H, N)):
        nd = needles(B, H, N, cands, r)
        _q, _k, v = needle_operands(B, B, N, M, H, 64, 64, nd, False, P["dtype"], 9 + r)
        in_range, live = key_sets(B, N, M, P["pad"], True)
        want = needle_expect(v, H, in_range, live, nd, P["dtype"])
        if mutant == "padded_key_leaked":
            live2 = live | (P["pad"][:, None, :] & in_range)
            live2[2] = live[2]
        else:
            live2 = key_sets(B, N, M, P["pad"], True, causal_end=M + (1 if mutant == "causal_plus_1" else -1))[1]
        rejected += _bits_differ(want, needle_expect(v, H, in_range, live2, nd, P["dtype"]))
    print(f"[probe power] needle probe rejects {mutant} in {rejected} rounds")
    assert rejected


def test_needles_cover_every_candidate():
    """The needle rounds of the GPU probes put a needle on every candidate key of every batch row: for the non-window
    shape (B = 3, H = 2, M = 1153) at N = 1..4 with and without causal, and for every window of the arena.  The causal
    candidates include key 0, the last key, every diagonal and the key past it, and the first key of every split."""
    B, H, M = 3, 2, 1153
    g = torch.Generator().manual_seed(0)
    pad = torch.rand(B, M, generator=g) < 0.15
    pad[1] = False
    pad[2] = True
    jobs = []
    for N, causal in itertools.product((1, 2, 3, 4), (False, True)):
        ranges = split_ranges(M, *choose_split(B, H, M))
        jobs.append((N, causal, 0, M, ranges, B, H))
    for (name, win), N in itertools.product(WINDOWS, (1, 4)):
        a, e = window_clamp(*win, CAPACITY)
        if e > a:
            jobs.append((N, True, a, e, window_ranges(*win, CAPACITY, WIN_NSPLIT), WIN_B, WIN_H))
    for N, causal, k0, kend, ranges, B_, H_ in jobs:
        pd = torch.zeros(B_, max(kend, M), dtype=torch.bool)
        pd[:, :M] = pad[:B_] if B_ == B else False
        for lpk, nq, fp8 in GEOMETRIES:
            if nq != DV.nq_of(N):
                continue
            cands = [needle_candidates(N, k0, kend, ranges, pd, b, causal, lpk, nq, fp8) for b in range(B_)]
            placed = [set() for _ in range(B_)]
            for r in range(needle_rounds(cands, H_, N)):
                nd = needles(B_, H_, N, cands, r)
                for b in range(B_):
                    placed[b] |= set(nd[b].flatten().tolist())
            assert placed == [set(c) for c in cands], (N, causal, k0, kend, lpk, nq, fp8)
            want = {k0, kend - 1} | {kb for kb, ke in ranges if ke > kb}
            if causal:
                want |= {kend - N + n for n in range(N)} | {kend - N + n + 1 for n in range(N - 1)}
            want = {j for j in want if k0 <= j < kend}
            assert all(want <= c for c in map(set, cands)), (N, causal, k0, kend, sorted(want - set(cands[1])))
    print(f"[needles] {len(jobs)} shapes x geometries: every candidate key held a needle")
