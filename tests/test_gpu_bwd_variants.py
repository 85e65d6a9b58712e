"""-m gpu: every instantiation of the attention backward (bwd_dkdv_kernel, bwd_dq_kernel on 128- and 64-key stages) at
its schedule, tile and mask edges, against fp64 autograd of the reference algorithm, and the dropout forward at the same
head dims up to 128.
The matrix and the schedule shapes live in bwd_variants.py; test_bwd_variants_cpu.py checks that the matrix covers every
instantiation, that the shapes have their plan structure, and that the gate is calibrated and sees the bugs it is for.

Every gradient goes through gpu_util.assert_grads: the derived whole-tensor gate and the element-wise gate
|got - ref| <= KAPPA u |.|-reference, so one wrong key in a small row of a gradient is seen.  Masked keys are poisoned
as in test_gpu_fwd_variants.py (a score of ~12 against every query and values of 500..1000): one let through moves its
row by far more than the bound."""
import pytest
import torch

from bwd_variants import (EDGE_M, EDGE_N, SCHEDULE_CASES, SCHEDULE_SHAPES, VARIANT_CASES, case_id, check_bwd_schedule,
                          edge_variants, is_wide, plan)
from fwd_variants import DIAG_N, DIAG_SHIFTS
from gpu_util import assert_grad_set, assert_rows, grad_magnitudes, torch_core
from perceiver_io_b200 import _lib, ops
from test_gpu_bwd import _case, _ref_grads
from test_gpu_dropout import _core_drop, _drop_ref, _rp
from test_gpu_fwd_variants import _diag_mask, _operands, _pad_mask

pytestmark = pytest.mark.gpu

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
SEED = 0x5EED_B0D5
REF_ELEMS = 1 << 23  # above this many scores (B*H*N*M) the fp64 references are computed one head at a time


def _sms():
    return ops.device_info()["num_sms"]


def _grad_out(B, N, H, dv, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B, N, H * dv, device="cuda", generator=g).to(dtype)


def _host_forward(q, k, v, H, scale, pad, causal):
    """(out, m, l) as the forward kernel defines them, from fp64 on the device: the forward kernel takes causal
    attention with N <= M only, the backward also N > M.  m, l in the log2 domain; a row without a live key has
    m = -FLT_MAX (every score the finite fill) and l = M."""
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    qh = q.double().expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = k.double().reshape(B, M, H, -1).transpose(1, 2)
    t = (qh @ kh.transpose(-1, -2)) * (scale * 1.4426950408889634)
    filled = torch.zeros(B, 1, N, M, dtype=torch.bool, device=q.device)
    if pad is not None:
        filled = filled | pad.to(q.device)[:, None, None, :]
    if causal:
        filled = filled | torch.ones(N, M, dtype=torch.bool, device=q.device).triu(M - N + 1)
    t = t.masked_fill(filled, -torch.finfo(torch.float32).max)
    m = t.amax(-1)
    l = torch.exp2(t - m[..., None]).sum(-1)
    out = torch_core(q, k, v, H, scale, pad, causal, torch.float64).to(q.dtype)
    return out, m.float().contiguous(), l.float().contiguous()


def _forward(q, k, v, H, scale, pad, causal, p=0.0):
    if causal and q.shape[1] > k.shape[1]:
        assert p == 0
        return _host_forward(q, k, v, H, scale, pad, causal)
    po, pm, pl = ops.attention_partial(q, k, v, H, scale, pad_mask=pad, causal=causal,
                                       **({"dropout_p": p, "dropout_seed": SEED} if p > 0 else {}))
    return ops.combine_partials(po[None], pm[None], pl[None], q.dtype), pm, pl


def _backward(q, k, v, go, H, scale, pad, causal, p=0.0, fwd=None):
    out, pm, pl = _forward(q, k, v, H, scale, pad, causal, p) if fwd is None else fwd
    return ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, pad_mask=pad, causal=causal, dropout_p=p,
                                  dropout_seed=SEED)


def _head(t, H, h):
    d = t.shape[-1] // H
    return t[..., h * d:(h + 1) * d]


def _references(q, k, v, go, H, scale, pad, causal, keep=None, rp=1.0):
    """(fp64 gradients, 16-bit eager gradients, magnitudes); one head at a time above REF_ELEMS scores."""
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    if B * H * N * M > REF_ELEMS and H > 1:
        parts = [_references(_head(q, H, h), _head(k, H, h), _head(v, H, h), _head(go, H, h), 1, scale, pad, causal,
                             None if keep is None else keep[:, h:h + 1], rp) for h in range(H)]
        ref, eag, mags = ([[torch.cat([pt[i][j] for pt in parts], -1) for j in range(3)] for i in range(2)]
                          + [[type(parts[0][2][j])(*(torch.cat([getattr(pt[2][j], f) for pt in parts], -1)
                                                    for f in ("abs", "sub"))) for j in range(3)]])
        return ref, eag, mags
    if keep is None:
        ref = _ref_grads(q, k, v, go, H, scale, pad, causal, torch.float64)
        eag = _ref_grads(q, k, v, go, H, scale, pad, causal, q.dtype)
    else:
        ref, eag = (_drop_ref(q, k, v, go, H, scale, pad, causal, dt, keep, rp)[1:] for dt in (torch.float64, q.dtype))
    return ref, eag, grad_magnitudes(q, k, v, go, H, scale, pad, causal, keep, rp)


def _gate(got, q, k, v, go, H, scale, pad, causal, what, keep=None, rp=1.0, whole=True):
    ref, eag, mags = _references(q, k, v, go, H, scale, pad, causal, keep, rp)
    return assert_grad_set(got, ref, eag, mags, q.dtype, what, whole)


def _dq_deterministic(B, H, N, M, dqk, dv, bcast):
    """The wide dQ sums its partials in a fixed order; elsewhere dQ is reduced with fp32 atomics, which give one order
    only when each element receives one contribution: one split and a per-batch q."""
    return is_wide(dqk, dv) or (plan(B, H, N, M, dqk, dv, _sms())["splits"] == 1 and not bcast)


def _dead_rows(pad_b, N, M, causal):
    """Query rows of one batch row without a live key."""
    filled = pad_b.cpu()[None, :].expand(N, M)
    if causal:
        filled = filled | torch.ones(N, M, dtype=torch.bool).triu(M - N + 1)
    return filled.all(-1)


def _assert_masked_keys_get_nothing(grads, pad, N, causal, what):
    """dK of every padded key is exactly 0; so is its dV in batch rows where every query has a live key."""
    _, gk, gv = grads
    padc = pad.to(gk.device)
    assert (gk[padc] == 0).all(), f"{what}: dK of a padded key is not 0"
    for b in range(pad.shape[0]):
        if not _dead_rows(pad[b], N, pad.shape[1], causal).any():
            assert (gv[b][padc[b]] == 0).all(), f"{what}: dV of a padded key of batch row {b} is not 0"


# --------------------------------------------------------------------------------------------------
# every instantiation x four mask regimes, with the exact properties
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", VARIANT_CASES, ids=case_id)
def test_variant_mask_regimes_and_exact_properties(case):
    dqk, dv, dt = case
    dtype, scale, name = DTYPE[dt], dqk ** -0.5, case_id(case)
    B, N, M, H = 3, 200, 300, 2
    pad = _pad_mask(B, M, seed=7)                   # about 30 %, batch row 1 wholly padded
    padc = pad.cuda()
    nopad = torch.zeros(B, M, dtype=torch.bool, device="cuda")
    diag = _diag_mask(B, M, M - N)                  # keys just past each warpgroup's diagonal
    go = _grad_out(B, N, H, dv, dtype, seed=5)

    # no mask; an all-False pad mask and a second call give the same dK / dV bit for bit
    q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=1)
    fwd = _forward(q, k, v, H, scale, None, False)
    got = _backward(q, k, v, go, H, scale, None, False, fwd=fwd)
    _gate(got, q, k, v, go, H, scale, None, False, f"{name} no mask")
    again = _backward(q, k, v, go, H, scale, None, False, fwd=fwd)
    assert torch.equal(again[1], got[1]) and torch.equal(again[2], got[2]), "dK / dV differ between two calls"
    allfalse = _backward(q, k, v, go, H, scale, nopad, False, fwd=fwd)
    assert torch.equal(allfalse[1], got[1]) and torch.equal(allfalse[2], got[2]), "all-False pad != no pad (dK / dV)"
    if _dq_deterministic(B, H, N, M, dqk, dv, False):
        assert torch.equal(allfalse[0], got[0]), "all-False pad != no pad (dQ)"

    # random pad, batch-1 q, padded keys poisoned
    q1, kp, vp = _operands(B, N, M, H, dqk, dv, dtype, seed=2, Bq=1, poison=pad)
    got = _backward(q1, kp, vp, go, H, scale, padc, False)
    _gate(got, q1, kp, vp, go, H, scale, pad, False, f"{name} pad, q broadcast")
    _assert_masked_keys_get_nothing(got, pad, N, False, f"{name} pad")

    # causal, keys just past each warpgroup's diagonal poisoned; all-False pad gives the same dK / dV
    qc, kc, vc = _operands(B, N, M, H, dqk, dv, dtype, seed=3, poison=diag)
    fwd = _forward(qc, kc, vc, H, scale, None, True)
    got = _backward(qc, kc, vc, go, H, scale, None, True, fwd=fwd)
    _gate(got, qc, kc, vc, go, H, scale, None, True, f"{name} causal")
    allfalse = _backward(qc, kc, vc, go, H, scale, nopad, True, fwd=fwd)
    assert torch.equal(allfalse[1], got[1]) and torch.equal(allfalse[2], got[2]), "causal: all-False pad != no pad"

    # causal + pad, per-batch q: the fully padded batch row gets dQ = dK = 0
    qcp, kcp, vcp = _operands(B, N, M, H, dqk, dv, dtype, seed=4, poison=diag | pad)
    got = _backward(qcp, kcp, vcp, go, H, scale, padc, True)
    _gate(got, qcp, kcp, vcp, go, H, scale, pad, True, f"{name} causal + pad")
    _assert_masked_keys_get_nothing(got, pad, N, True, f"{name} causal + pad")
    assert (got[0][1] == 0).all() and (got[1][1] == 0).all(), "dQ / dK of the fully padded batch row are not 0"


# --------------------------------------------------------------------------------------------------
# schedule shapes: the ring phase carried across tiles, the ring's wrap, the dQ split edges
# --------------------------------------------------------------------------------------------------
SCHEDULE_RUNS = [(shape, case) for shape, cases in SCHEDULE_CASES.items() for case in cases]
SCHEDULE_MASKS = {  # pad kind, causal, batch-1 q; "random" pads about 30 % of every key tile
    "dkdv_carry": ("random", False, False),
    "dkdv_wrap": (None, True, False),          # N = 700 > M = 300: rows n < 400 have no live key
    "dq_split": ("random", False, True),
    "wide_dq_items": ("random", False, True),
}


@pytest.mark.parametrize("shape, case", SCHEDULE_RUNS, ids=[f"{s}-{case_id(c)}" for s, c in SCHEDULE_RUNS])
def test_schedule_shapes(shape, case):
    dqk, dv, dt = case
    print(check_bwd_schedule(shape, case, _sms()))
    B, H, N, M = SCHEDULE_SHAPES[shape]
    pad_kind, causal, bcast = SCHEDULE_MASKS[shape]
    q, k, v, go, pad = _case(B, N, M, H, dqk, dv, pad_kind, causal, bcast, dtype=DTYPE[dt], seed=N + M + dqk)
    if pad is not None:  # the last key tile and the last dQ split hold live keys in every batch row
        k0 = plan(B, H, N, M, dqk, dv, _sms())["last_split_key0"]
        assert (~pad[:, k0:]).any(-1).all() and (~pad[:, (M - 1) // 128 * 128:]).any(-1).all()
    scale = dqk ** -0.5
    got = _backward(q, k, v, go, H, scale, pad, causal)
    _gate(got, q, k, v, go, H, scale, pad, causal, f"{shape} {case_id(case)}")
    if causal and N > M:
        assert (got[0][:, :N - M] == 0).all(), "dQ of rows without a live key is not 0"


# --------------------------------------------------------------------------------------------------
# tile edges: every (N, M) pair, with and without causal, on one small and one wide variant.  Without causal there is
# no mask; with it batch row 1 is padded past a random length and batch row 0 not at all, so the last key (the one key
# of the last tile at M = 129 or 257, the last 64-key stage) is live for the last query
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", EDGE_N)
def test_tile_edges(N):
    B, H = 2, 2
    for i, M in enumerate(EDGE_M):
        for case in edge_variants(EDGE_N.index(N) * len(EDGE_M) + i):
            dqk, dv, dt = case
            scale = dqk ** -0.5
            for causal in (False, True):
                q, k, v, go, pad = _case(B, N, M, H, dqk, dv, "ragged" if causal else None, causal, False,
                                         dtype=DTYPE[dt], seed=N * 1000 + M)
                if pad is not None:
                    pad[0] = False
                got = _backward(q, k, v, go, H, scale, pad, causal)
                # M <= 2: the element-wise gate only (gpu_util.assert_grads, `whole`)
                _gate(got, q, k, v, go, H, scale, pad, causal, f"{case_id(case)} N {N} M {M} causal {causal}",
                      whole=M > 2)


# --------------------------------------------------------------------------------------------------
# the causal diagonal: single pass (negative shifts: N > M) and as key shards at even, unaligned cuts
# --------------------------------------------------------------------------------------------------
DIAG_CASES = [(120, 56, "bf16"), (184, 120, "bf16"), (40, 120, "fp16"), (40, 184, "fp16")]
NEG_SHIFTS = (-1, -63, -64, -65, -129)
SHARD_CUTS = (64, 258)


@pytest.mark.parametrize("case", DIAG_CASES, ids=case_id)
def test_causal_diagonal_sweep(case):
    dqk, dv, dt = case
    dtype, scale = DTYPE[dt], dqk ** -0.5
    B, H, N = 2, 2, DIAG_N
    for shift in NEG_SHIFTS + DIAG_SHIFTS:
        M = N + shift
        q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=60 + shift, poison=_diag_mask(B, M, shift))
        go = _grad_out(B, N, H, dv, dtype, seed=61 + shift)
        out, pm, pl = _forward(q, k, v, H, scale, None, True)
        got = _backward(q, k, v, go, H, scale, None, True, fwd=(out, pm, pl))
        ref, eag, mags = _references(q, k, v, go, H, scale, None, True)
        assert_grad_set(got, ref, eag, mags, dtype, f"{case_id(case)} shift {shift}")
        if shift < 0:
            assert (got[0][:, :-shift] == 0).all(), f"shift {shift}: dQ of rows without a live key is not 0"
            continue
        # key shards [0, 64), [64, 258), [258, M) from the merged statistics
        cuts = (0,) + SHARD_CUTS + (M,)
        gq = torch.zeros(q.shape, dtype=torch.float32, device="cuda")
        gks, gvs = [], []
        for a, b in zip(cuts[:-1], cuts[1:]):
            g32, gk, gv = ops.attention_backward_shard(q, k[:, a:b], v[:, a:b], out, go, pm, pl, H, scale, M, a,
                                                       causal=True)
            gq += g32
            gks.append(gk)
            gvs.append(gv)
        assert_grad_set((gq, torch.cat(gks, 1), torch.cat(gvs, 1)), ref, eag, mags, dtype,
                        f"{case_id(case)} shift {shift} shards {cuts}")


# --------------------------------------------------------------------------------------------------
# dropout on the exported mask: the backward, and the dropout forward (attention_dropout_forward)
# --------------------------------------------------------------------------------------------------
DROP_BWD = [(40, 120, "bf16"), (184, 56, "bf16"), (120, 56, "fp16"), (40, 184, "fp16")]


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("case", DROP_BWD, ids=case_id)
def test_dropout_backward(case, p):
    dqk, dv, dt = case
    B, N, M, H = 3, 200, 300, 2
    scale = dqk ** -0.5
    q, k, v, go, pad = _case(B, N, M, H, dqk, dv, "row_full", True, False, dtype=DTYPE[dt], seed=70)
    keep = ops.dropout_keep_mask(B, H, N, M, p, SEED)
    rp = _rp(p)[1]
    got = _backward(q, k, v, go, H, scale, pad, True, p=p)
    _gate(got, q, k, v, go, H, scale, pad, True, f"{case_id(case)} dropout {p}", keep, rp)


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("case", [c for c in VARIANT_CASES if not is_wide(c[0], c[1])], ids=case_id)
def test_dropout_forward_rows(case, p):
    dqk, dv, dt = case
    dtype, scale = DTYPE[dt], dqk ** -0.5
    B, N, M, H = 3, 200, 300, 2
    pad = _pad_mask(B, M, seed=8)
    q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=9, Bq=1, poison=pad)
    keep = ops.dropout_keep_mask(B, H, N, M, p, SEED)
    rp = _rp(p)[1]
    for causal in (False, True):
        _, pm, pl = _forward(q, k, v, H, scale, pad.cuda(), causal)
        out = ops.attention_dropout_forward(q, k, v, pm, pl, H, scale, p, SEED, pad.cuda(), causal)
        ref = _core_drop(q, k, v, H, scale, pad.cuda(), causal, torch.float64, keep, rp)
        eager = _core_drop(q, k, v, H, scale, pad.cuda(), causal, dtype, keep, rp)
        assert torch.isfinite(out).all()
        assert_rows(out, ref, eager, H, f"{case_id(case)} dropout forward p {p} causal {causal}")


def test_zz_watchdog_record_is_clear():
    """No barrier wait of any kernel timed out during this module (runs last in it)."""
    torch.cuda.synchronize()
    assert _lib.debug_read()[0] == 0, _lib.debug_read()
