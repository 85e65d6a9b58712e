"""CPU companion of test_gpu_bwd_variants.py: the backward variant matrix covers every instantiation, the schedule
shapes have the structure they are named for, the restated dQ split is the library's, and the gradient gate
(gpu_util.assert_grads) is calibrated on an emulation of the kernels' arithmetic and rejects the bugs it is meant to
see."""
import ctypes
import math

import pytest
import torch

from bwd_variants import (DTYPES, KWIDE_SPLIT_SMS, SCHEDULE_CASES, SCHEDULE_SHAPES, TILE, VARIANT_CASES, check_bwd_schedule,
                          dq_split, reachable_variants, variants_of)
from gpu_util import assert_grads, element_bound, grad_magnitudes
from test_bwd_bighead_cpu import _bwd_params
from test_gpu_bwd import _ref_grads
from test_gpu_dropout import _drop_ref

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
LOG2E = 1.4426950408889634


def test_matrix_reaches_every_instantiation():
    covered = set().union(*(variants_of(dqk, dv, dt) for dqk, dv, dt in VARIANT_CASES))
    reach = reachable_variants()
    assert len(reach) == 2 * (4 * 2 + 5 * 3)  # 4 small pairs x (dK/dV, dQ), 5 wide x 3 kernels
    assert covered == reach, sorted(reach - covered, key=str)
    # head dims that are not multiples of 64 everywhere: every box has a zero-filled tail
    assert all(dqk % 64 and dv % 64 for dqk, dv, _ in VARIANT_CASES)


@pytest.mark.parametrize("shape", list(SCHEDULE_SHAPES))
def test_schedule_shapes_have_their_structure_at_132_sms(shape):
    for case in SCHEDULE_CASES[shape]:
        print(check_bwd_schedule(shape, case, 132))
    assert {dt for *_, dt in SCHEDULE_CASES[shape]} == set(DTYPES)


def test_restated_dq_split_matches_the_library():
    """Wide head dims, no pad mask: workspace = stats blocks + dq_bytes * (Bq == 1 ? B : 1) * splits, the split planned
    at kWideSplitSms.  dq_bytes is a multiple of 256 (N * H * Bq a multiple of 8 at dqk = 136), so no alignment hides a
    wrong split count."""
    from perceiver_io_b200 import _lib

    handle = _lib.lib()
    seen = set()
    for B, H, N, M, bcast in [(1, 1, 64, 1000, False), (2, 8, 256, 1024, True), (1, 1, 8, 20000, False),
                              (4, 2, 128, 12000, True), (3, 8, 64, 2700, True), (2, 4, 1000, 65536, False),
                              (8, 8, 512, 65536, True), (1, 2, 64, 40000, False), (2, 1, 8, 129, True),
                              (6, 4, 200, 9000, False), (1, 1, 4096, 300, False)]:
        dqk = 136
        Bq = 1 if bcast else B
        p = _bwd_params(dqk, dqk, B=B, H=H, N=N, M=M, q_stride_b=0 if bcast else N * H * dqk)
        need = ctypes.c_size_t(0)
        assert handle.pcv_attn_bwd_workspace_bytes(ctypes.byref(p), ctypes.byref(need)) == 0
        nq, nk = (N + TILE - 1) // TILE, (M + TILE - 1) // TILE
        stats = (768 * B * H * 2 * nq + 255) // 256 * 256
        dq_bytes = 4 * Bq * N * H * dqk
        assert dq_bytes % 256 == 0
        tps, splits = dq_split(B * H * nq, nk, KWIDE_SPLIT_SMS)
        parts = (B if Bq == 1 else 1) * splits
        assert need.value == stats + dq_bytes * parts, (B, H, N, M, bcast, need.value, stats, dq_bytes, parts)
        seen.add(splits)
    assert len(seen) >= 4, seen  # the grid walks several split counts


# ---- the gate: calibration on an emulation of the kernels' arithmetic ----
def _round(t, dtype):
    return t.to(dtype).to(t.dtype)


def _filled(B, N, M, pad, causal):
    f = torch.zeros(B, 1, N, M, dtype=torch.bool)
    if pad is not None:
        f = f | pad[:, None, None, :]
    if causal:
        f = f | torch.ones(N, M, dtype=torch.bool).triu(M - N + 1)
    return f


def emulate_kernels(q, k, v, go, H, scale, pad, causal, dtype, keep=None, rp=1.0):
    """The forward and backward kernels' arithmetic in fp32: fp32 scores and statistics (m, l in the log2 domain), the
    forward output from 16-bit P, delta from the 16-bit output, P = 2^(t + nlse) in fp32 (fillp = 1/l on a row without a
    live key), P (times keep / (1 - p)) and dS rounded to 16 bits before the gradient GEMMs, fp32 accumulation, the
    gradients rounded to 16 bits."""
    f32 = torch.float32
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    qh = q.to(f32).expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = k.to(f32).reshape(B, M, H, -1).transpose(1, 2)
    vh = v.to(f32).reshape(B, M, H, -1).transpose(1, 2)
    gh = go.to(f32).reshape(B, N, H, -1).transpose(1, 2)
    kr = torch.ones(B, H, N, M) if keep is None else keep.to(f32) * rp
    filled = _filled(B, N, M, pad, causal).expand(B, H, N, M)
    t = (qh @ kh.transpose(-1, -2)) * f32_(scale * LOG2E)
    dead = filled.all(-1, keepdim=True)
    m = t.masked_fill(filled, -math.inf).amax(-1, keepdim=True)
    m = torch.where(dead, torch.zeros_like(m), m)
    pf = torch.exp2(t - m).masked_fill(filled, 0.0)
    l = torch.where(dead, torch.full_like(m, float(M)), pf.sum(-1, keepdim=True))
    pf = torch.where(dead.expand_as(pf), torch.ones_like(pf), pf)   # the finite fill: uniform
    o = _round((_round(pf * kr, dtype) @ vh) / l, dtype)                      # the forward output, 16-bit
    delta = (gh * o).sum(-1, keepdim=True)
    nlse = -(m + torch.log2(l))
    P = torch.exp2(t + nlse)
    P = torch.where(filled, torch.where(dead, 1.0 / l, torch.zeros_like(l)).expand_as(P), P)
    dv = _round(_round(P * kr, dtype).transpose(-1, -2) @ gh, dtype)
    dp = (gh @ vh.transpose(-1, -2)) * kr
    ds = _round((P * (dp - delta)).masked_fill(filled, 0.0), dtype)
    dk = _round((ds.transpose(-1, -2) @ qh) * f32_(scale), dtype)
    dq = (ds @ kh) * f32_(scale)
    if q.shape[0] == 1 and B > 1:
        dq = dq.sum(0, keepdim=True)
    dq = _round(dq, dtype)

    def merge(x, L):
        return x.transpose(1, 2).reshape(x.shape[0], L, -1)

    return merge(dq, N), merge(dk, M), merge(dv, M)


def f32_(x):
    return torch.tensor(x, dtype=torch.float32)


def _operands(B, N, M, H, dqk, dv, dtype, seed, bcast=False, peaked=False):
    g = torch.Generator().manual_seed(seed)
    sc = 3.0 if peaked else 1.0
    q = (torch.randn(1 if bcast else B, N, H * dqk, generator=g) * sc).to(dtype)
    k = (torch.randn(B, M, H * dqk, generator=g) * sc).to(dtype)
    v = torch.randn(B, M, H * dv, generator=g).to(dtype)
    go = torch.randn(B, N, H * dv, generator=g).to(dtype)
    return q, k, v, go


def _pad(B, M, seed):
    g = torch.Generator().manual_seed(seed)
    pad = torch.rand(B, M, generator=g) < 0.3
    pad[1] = True
    return pad


CALIBRATION = [  # B, N, M, H, dqk, dv, pad, causal, bcast, peaked, dropout p
    (3, 130, 300, 2, 40, 56, True, False, True, False, 0.0),
    (2, 200, 260, 2, 120, 120, False, True, False, False, 0.0),
    (3, 130, 300, 2, 184, 120, True, True, False, False, 0.0),
    (2, 96, 400, 1, 64, 64, False, False, False, True, 0.0),    # peaked softmax
    (2, 100, 200, 2, 40, 184, True, False, True, False, 0.25),
]


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_gate_passes_the_emulated_kernel_arithmetic_with_margin(dt):
    dtype = DTYPE[dt]
    worst = {}
    for i, (B, N, M, H, dqk, dv, with_pad, causal, bcast, peaked, p) in enumerate(CALIBRATION):
        q, k, v, go = _operands(B, N, M, H, dqk, dv, dtype, seed=i, bcast=bcast, peaked=peaked)
        pad = _pad(B, M, seed=i) if with_pad else None
        scale = dqk ** -0.5
        keep, rp = None, 1.0
        if p > 0:
            keep = torch.rand(B, H, N, M, generator=torch.Generator().manual_seed(99)) >= p
            rp = 1.0 / (1.0 - p)
        got = emulate_kernels(q, k, v, go, H, scale, pad, causal, dtype, keep, rp)
        if keep is None:
            ref, eager = _ref_grads(q, k, v, go, H, scale, pad, causal, torch.float64), \
                _ref_grads(q, k, v, go, H, scale, pad, causal, dtype)
        else:
            ref, eager = (_drop_ref(q, k, v, go, H, scale, pad, causal, dt_, keep, rp)[1:]
                          for dt_ in (torch.float64, dtype))
        mags = grad_magnitudes(q, k, v, go, H, scale, pad, causal, keep, rp)
        for name, g_, r_, e_, m_ in zip(("dq", "dk", "dv"), got, ref, eager, mags):
            w = assert_grads(g_, r_, e_, m_, dtype, f"emulated {dt} case {i} {name}")
            worst[name] = max(worst.get(name, 0.0), w)
    print(f"[gate calibration] {dt}: emulated worst err/bound " + ", ".join(f"{n} {w:.3f}" for n, w in worst.items()))
    assert max(worst.values()) <= 0.5, worst


def test_whole_tensor_gate_has_no_yardstick_below_three_keys():
    """Causal rows whose live keys number one or two, as the tile-edge sweep's M <= 2 cases have them (batch row 0
    unpadded, batch row 1 padded past a random length).  With one key, P = 1 and delta = dP, so dS, dQ and dK are 0 in
    exact arithmetic while the kernels' delta from the 16-bit output differs from dP in the last bits; with two, the two
    dS of a row cancel, dQ = scale * dS_0 (K_0 - K_1), and eager's error lands below half the kernels' on some seeds.
    Over 60 seeds, the emulated kernel arithmetic exceeds the whole-tensor gate at M = 1 on nearly every seed and at
    M = 2 on some, passes it on every seed at M = 3, and stays under half of the element-wise bound throughout.  So the GPU
    sweep applies the whole-tensor gate from M = 3 on."""
    B, H, d = 2, 2, 120
    scale = d ** -0.5
    over = {}
    for M in (1, 2, 3):
        for dt in ("bf16", "fp16"):
            dtype = DTYPE[dt]
            count = 0
            for seed in range(60):
                N = (1, 63, 64, 65, 127, 128, 129)[seed % 7]
                g = torch.Generator().manual_seed(seed)
                q, k, v, go = (torch.randn(*sh, generator=g).to(dtype)
                               for sh in ((B, N, H * d), (B, M, H * d), (B, M, H * d), (B, N, H * d)))
                pad = torch.arange(M)[None, :] >= torch.randint(1, M + 1, (B,), generator=g)[:, None]
                pad[0] = False
                got = emulate_kernels(q, k, v, go, H, scale, pad, True, dtype)
                ref = _ref_grads(q, k, v, go, H, scale, pad, True, torch.float64)
                eager = _ref_grads(q, k, v, go, H, scale, pad, True, dtype)
                mags = grad_magnitudes(q, k, v, go, H, scale, pad, True)
                hit = False
                for g_, r_, e_, m_ in zip(got, ref, eager, mags):
                    assert assert_grads(g_, r_, e_, m_, dtype, f"M {M} {dt} seed {seed}", whole=False) <= 0.5
                    try:
                        assert_grads(g_, r_, e_, m_, dtype, f"M {M} {dt} seed {seed}")
                    except AssertionError:
                        hit = True
                count += hit
            over[(M, dt)] = count
    print(f"[whole-tensor gate] seeds (of 60) on which the emulation exceeds it: {over}")
    assert min(over[(1, "bf16")], over[(1, "fp16")]) >= 50  # unless the two fp32 sums happen to round alike
    assert over[(2, "bf16")] + over[(2, "fp16")] > 0
    assert over[(3, "bf16")] == over[(3, "fp16")] == 0


# ---- the gate: power against the bugs it is meant to see ----
def _explicit_grads(q, k, v, go, H, scale, filled_fwd, filled_bwd=None, fillp_zero=False, skip_dkdv=None,
                    skip_dq=None):
    """fp64 backward restated from its formulas, with the kernel's structure exposed to mutation: the statistics and
    delta come from the forward with `filled_fwd`, the backward masks with `filled_bwd` (P = exp(s - lse) where that
    lets a key through), `fillp_zero` drops the uniform P of rows without a live key, `skip_dkdv = (n0, n1, j0, j1)`
    leaves queries [n0, n1) out of dK / dV of keys [j0, j1), `skip_dq = (n, j0, j1)` leaves keys [j0, j1) out of dQ row n."""
    f64 = torch.float64
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    qh = q.to(f64).expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = k.to(f64).reshape(B, M, H, -1).transpose(1, 2)
    vh = v.to(f64).reshape(B, M, H, -1).transpose(1, 2)
    gh = go.to(f64).reshape(B, N, H, -1).transpose(1, 2)
    s = (qh * scale) @ kh.transpose(-1, -2)
    ff = filled_fwd.expand(B, H, N, M)
    sf = s.masked_fill(ff, -torch.finfo(f64).max)
    lse = sf.logsumexp(-1, keepdim=True)
    p_true = sf.softmax(-1)
    delta = (gh * (p_true @ vh)).sum(-1, keepdim=True)
    fb = ff if filled_bwd is None else filled_bwd.expand(B, H, N, M)
    dead = ff.all(-1, keepdim=True).expand_as(fb)
    fill = torch.zeros_like(s) if fillp_zero else torch.where(dead, p_true, torch.zeros_like(s))
    P = torch.where(fb, fill, torch.exp(torch.where(fb, lse, s) - lse))
    dS = torch.where(fb, torch.zeros_like(s), P * (gh @ vh.transpose(-1, -2) - delta))
    Pv, dSk, dSq = P.clone(), dS.clone(), dS.clone()
    if skip_dkdv is not None:
        n0, n1, j0, j1 = skip_dkdv
        Pv[..., n0:n1, j0:j1] = 0
        dSk[..., n0:n1, j0:j1] = 0
    if skip_dq is not None:
        n, j0, j1 = skip_dq
        dSq[..., n, j0:j1] = 0
    dq = scale * dSq @ kh
    if q.shape[0] == 1 and B > 1:
        dq = dq.sum(0, keepdim=True)
    dk = scale * dSk.transpose(-1, -2) @ qh
    dv = Pv.transpose(-1, -2) @ gh
    return tuple(x.transpose(1, 2).reshape(x.shape[0], L, -1) for x, L in ((dq, N), (dk, M), (dv, M)))


def _poisoned(B, N, M, H, dqk, dv, dtype, seed, poison, bcast=False):
    """test_gpu_fwd_variants._operands on the CPU: masked keys score ~12 against every query, their values 500..1000."""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(H, dqk, generator=g)
    u = u / u.norm(dim=-1, keepdim=True)
    q = torch.randn(1 if bcast else B, N, H, dqk, generator=g) + dqk ** 0.5 * u
    k = torch.randn(B, M, H, dqk, generator=g)
    v = torch.randn(B, M, H, dv, generator=g)
    pz = poison[:, :, None, None]
    k = torch.where(pz, 12.0 * u, k)
    big = torch.sign(torch.randn(B, M, H, dv, generator=g)) * (500.0 + 500.0 * torch.rand(B, M, H, dv, generator=g))
    v = torch.where(pz, big, v)
    go = torch.randn(B, N, H * dv, generator=g)
    return (q.reshape(-1, N, H * dqk).to(dtype), k.reshape(B, M, H * dqk).to(dtype), v.reshape(B, M, H * dv).to(dtype),
            go.to(dtype))


MUTANTS = ["leaked_masked_key", "missing_dkdv_substep", "missing_dq_key_tile", "causal_shifted_by_one",
           "fillp_zero"]


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("mutant", MUTANTS)
def test_gate_rejects_each_mutant_of_the_reference(mutant, dt):
    """Each mutant is one of the bugs the backward could have, applied to the fp64 reference at one place.  The
    unmutated restatement passes the gate; the mutant fails it, and fails the element-wise part on its own."""
    dtype = DTYPE[dt]
    B, N, M, H, dqk, dv = 3, 200, 300, 2, 40, 56
    scale = dqk ** -0.5
    pad, causal = None, True
    if mutant in ("leaked_masked_key", "fillp_zero"):  # random pad, batch row 1 wholly padded, batch-1 q, no causal
        pad, causal = _pad(B, M, seed=3), False
        q, k, v, go = _poisoned(B, N, M, H, dqk, dv, dtype, seed=4, poison=pad, bcast=True)
    elif mutant == "causal_shifted_by_one":
        M = N + 62  # keys just past every 64-row warpgroup's diagonal are poisoned, as in the GPU test
        poison = torch.zeros(B, M, dtype=torch.bool)
        poison[:, [j for j in range(M) if (j - 62 - 1) % 64 < 8]] = True
        q, k, v, go = _poisoned(B, N, M, H, dqk, dv, dtype, seed=5, poison=poison)
    else:
        q, k, v, go = _operands(B, N, M, H, dqk, dv, dtype, seed=6)
    filled = _filled(B, N, M, pad, causal)
    ref = _ref_grads(q, k, v, go, H, scale, pad, causal, torch.float64)
    eager = _ref_grads(q, k, v, go, H, scale, pad, causal, dtype)
    mags = grad_magnitudes(q, k, v, go, H, scale, pad, causal)

    plain = _explicit_grads(q, k, v, go, H, scale, filled)
    for g_, r_, e_, m_ in zip(plain, ref, eager, mags):
        assert assert_grads(g_, r_, e_, m_, dtype, f"{mutant} unmutated") < 1e-6

    if mutant == "leaked_masked_key":       # one padded key of batch row 0 let into query row 17
        j0 = int(pad[0].nonzero()[0])
        fb = filled.clone()
        fb[0, 0, 17, j0] = False
        got = _explicit_grads(q, k, v, go, H, scale, filled, filled_bwd=fb)
    elif mutant == "missing_dkdv_substep":  # the last 64-query sub-step (queries 192..199) of key tile 1
        got = _explicit_grads(q, k, v, go, H, scale, filled, skip_dkdv=(192, 200, 128, 256))
    elif mutant == "missing_dq_key_tile":   # key tile 0 (128 of the 141 keys row 40 sees) missing from dQ row 40
        got = _explicit_grads(q, k, v, go, H, scale, filled, skip_dq=(40, 0, 128))
    elif mutant == "causal_shifted_by_one":  # j > n + cshift + 1: the first key past every diagonal let in
        got = _explicit_grads(q, k, v, go, H, scale, filled,
                              filled_bwd=torch.ones(N, M, dtype=torch.bool).triu(M - N + 2).expand(B, 1, N, M))
    else:                                   # fillp = 0 on batch row 1, whose every key is padded
        got = _explicit_grads(q, k, v, go, H, scale, filled, fillp_zero=True)

    rejected = []
    for name, g_, r_, e_, m_ in zip(("dq", "dk", "dv"), got, ref, eager, mags):
        elementwise = bool(((g_.double() - r_).abs() > element_bound(m_, dtype)).any())
        try:
            assert_grads(g_, r_, e_, m_, dtype, f"{mutant} {name}")
            assert not elementwise
        except AssertionError as exc:
            assert elementwise, f"{mutant} {name}: rejected only by the whole-tensor gate: {exc}"
            rejected.append(name)
    print(f"[gate power] {mutant} {dt}: rejected in {rejected}")
    assert rejected, f"{mutant}: no gradient rejected"
