"""-m gpu: every instantiation of the tensor-core forward kernel (attn_fwd_kernel<NQB, NVB, BF16, PAIR>) at its schedule
and mask edges, against the fp64 reference.  The variant matrix and the schedule shapes live in fwd_variants.py; the
CPU companion (test_fwd_variants_cpu.py) checks that the matrix covers every instantiation and that the shapes have the
plan structure they are meant to exercise.

Masked keys are poisoned where a test looks for a leak: a large score along the direction every query shares and a
value of magnitude 500..1000, so one masked key let through moves its row by O(|v|).  Those rows are gated one by one
(gpu_util.assert_rows), since the poisoned keys are live, and large, in other rows of the same case."""
import pytest
import torch

from fwd_variants import (DIAG_N, DIAG_SHARD_CUTS, DIAG_SHIFTS, DIAG_VARIANTS, SCHEDULE_SHAPES, SCHEDULE_VARIANTS,
                          VARIANT_CASES, case_id, check_schedule, diag_poison_keys, plan_segments, workers_for)
from gpu_util import assert_parity, assert_partial_state

pytestmark = pytest.mark.gpu

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _impl(pair):
    return "tcgen05_pair" if pair else "tcgen05"


def _operands(B, N, M, H, dqk, dv, dtype, seed, Bq=None, poison=None):
    """q (Bq, N, H*dqk), k (B, M, H*dqk), v (B, M, H*dv) on the GPU.  Every query has a component of norm sqrt(dqk)
    along a unit direction u_h of its head, so with scale dqk^-0.5 a key 12 u_h scores about 12 against every row
    while the other keys score N(0, 2).  `poison` (B, M) bool: keys that get 12 u_h and values of magnitude 500..1000."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    Bq = B if Bq is None else Bq
    u = torch.randn(H, dqk, generator=g, device="cuda")
    u = u / u.norm(dim=-1, keepdim=True)
    q = torch.randn(Bq, N, H, dqk, generator=g, device="cuda") + dqk ** 0.5 * u
    k = torch.randn(B, M, H, dqk, generator=g, device="cuda")
    v = torch.randn(B, M, H, dv, generator=g, device="cuda")
    if poison is not None:
        pz = poison.to("cuda")[:, :, None, None]
        k = torch.where(pz, 12.0 * u, k)
        big = torch.sign(torch.randn(B, M, H, dv, generator=g, device="cuda")) * (
            500.0 + 500.0 * torch.rand(B, M, H, dv, generator=g, device="cuda"))
        v = torch.where(pz, big, v)
    return (q.reshape(Bq, N, H * dqk).to(dtype), k.reshape(B, M, H * dqk).to(dtype), v.reshape(B, M, H * dv).to(dtype))


def _pad_mask(B, M, seed):
    """Random padding (about 30 %) with batch row 1 fully padded."""
    g = torch.Generator().manual_seed(seed)
    pad = torch.rand(B, M, generator=g) < 0.3
    pad[1, :] = True
    return pad


def _diag_mask(B, M, shift):
    m = torch.zeros(B, M, dtype=torch.bool)
    m[:, diag_poison_keys(M, shift)] = True
    return m


def _part_equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


# --------------------------------------------------------------------------------------------------
# 1 + 4 + 5: every instantiation, four mask regimes, exact properties, partial state (split plan)
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", VARIANT_CASES, ids=case_id)
def test_variant_masks_exact_properties_and_partial_state(case):
    from perceiver_io_b200 import ops

    dqk, dv, dt, pair = case
    dtype, impl, scale = DTYPE[dt], _impl(pair), dqk ** -0.5
    B, N, M, H = 3, 200, 300, 2
    pad = _pad_mask(B, M, seed=7)
    padc = pad.cuda()
    nopad = torch.zeros(B, M, dtype=torch.bool, device="cuda")
    diag = _diag_mask(B, M, M - N)
    name = case_id(case)

    # no mask: mask-free tiles except the ragged last key tile
    q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=1)
    out = ops.attention(q, k, v, H, scale, impl=impl)
    assert_parity(out, q, k, v, H, scale, what=f"{name} no mask")
    assert torch.equal(ops.attention(q, k, v, H, scale, pad_mask=nopad, impl=impl), out), "all-False pad != no pad"

    # random pad mask, one batch row fully padded, batch-1 queries; padded keys poisoned
    q1, kp, vp = _operands(B, N, M, H, dqk, dv, dtype, seed=2, Bq=1, poison=pad)
    out = ops.attention(q1, kp, vp, H, scale, pad_mask=padc, impl=impl)
    assert_parity(out, q1, kp, vp, H, scale, pad, what=f"{name} pad, q broadcast", per_row=True)

    # causal without a pad mask (the mask-free causal tiles); keys just past warpgroup diagonals poisoned
    qc, kc, vc = _operands(B, N, M, H, dqk, dv, dtype, seed=3, poison=diag)
    out = ops.attention(qc, kc, vc, H, scale, causal=True, impl=impl)
    assert_parity(out, qc, kc, vc, H, scale, None, True, what=f"{name} causal", per_row=True)
    assert torch.equal(ops.attention(qc, kc, vc, H, scale, pad_mask=nopad, causal=True, impl=impl), out), \
        "causal: all-False pad != no pad"

    # causal + pad
    qcp, kcp, vcp = _operands(B, N, M, H, dqk, dv, dtype, seed=4, poison=diag | pad)
    out = ops.attention(qcp, kcp, vcp, H, scale, pad_mask=padc, causal=True, impl=impl)
    assert_parity(out, qcp, kcp, vcp, H, scale, pad, True, what=f"{name} causal + pad", per_row=True)

    # partial state: a causal shard wholly in the past of every row (m_offset + M - 1 == m_total - N) is the
    # non-causal state bit for bit; both match the oracle
    part = ops.attention_partial(q, k, v, H, scale, impl=impl)
    past = ops.attention_partial(q, k, v, H, scale, causal=True, m_total=M + N - 1, m_offset=0, impl=impl)
    assert _part_equal(part, past), "causal shard wholly in the past != non-causal partial state"
    assert_partial_state(part, q, k, v, H, scale, what=f"{name} partial")

    # a shard in the causal future of rows n < 100, with padding (batch row 1: every key); poisoned masked keys
    Ms, m_total, m_off = 100, 300, 200
    ks, vs, ps = kcp[:, :Ms], vcp[:, :Ms], pad[:, :Ms]
    fut = ops.attention_partial(qcp, ks, vs, H, scale, pad_mask=padc[:, :Ms], causal=True, m_total=m_total,
                                m_offset=m_off, impl=impl)
    dead = assert_partial_state(fut, qcp, ks, vs, H, scale, ps, True, m_total, m_off, what=f"{name} future shard")
    assert dead >= H * (B * 100 + (N - 100)), dead


# --------------------------------------------------------------------------------------------------
# 2: schedule shapes (structure asserted from the plan first)
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape_name", list(SCHEDULE_SHAPES))
@pytest.mark.parametrize("case", SCHEDULE_VARIANTS, ids=case_id)
def test_schedule_shapes(case, shape_name):
    from perceiver_io_b200 import ops

    dqk, dv, dt, pair = case
    dtype, impl, scale = DTYPE[dt], _impl(pair), dqk ** -0.5
    print(check_schedule(shape_name, case, workers_for(ops.device_info()["num_sms"], pair)))
    B, H, N, M = SCHEDULE_SHAPES[shape_name]
    name = f"{case_id(case)} {shape_name}"
    if shape_name == "whole_causal":
        diag = _diag_mask(B, M, M - N)
        q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=13, poison=diag)
        out = ops.attention(q, k, v, H, scale, causal=True, impl=impl)
        assert_parity(out, q, k, v, H, scale, None, True, what=f"{name}", per_row=True)
        return
    q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=11)
    out = ops.attention(q, k, v, H, scale, impl=impl)
    assert_parity(out, q, k, v, H, scale, what=f"{name} no mask")
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[:, 1:M:3] = True
    if B > 1:
        pad[-1, :] = True  # a fully padded batch row
    qp, kp, vp = _operands(B, N, M, H, dqk, dv, dtype, seed=12, poison=pad)
    if shape_name == "one_tile":
        out = ops.attention(qp, kp, vp, H, scale, pad_mask=pad.cuda(), causal=True, impl=impl)
        assert_parity(out, qp, kp, vp, H, scale, pad, True, what=f"{name} causal + pad", per_row=True)
    part = ops.attention_partial(qp, kp, vp, H, scale, pad_mask=pad.cuda(), impl=impl)
    dead = assert_partial_state(part, qp, kp, vp, H, scale, pad, what=f"{name} pad partial")
    assert dead == (H * N if B > 1 else 0), dead


# --------------------------------------------------------------------------------------------------
# 3: causal diagonal sweep over the mask-free-tile boundary, single pass and as M-shards
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", DIAG_VARIANTS, ids=case_id)
def test_causal_diagonal_sweep(case):
    from perceiver_io_b200 import ops

    dqk, dv, dt, pair = case
    dtype, impl, scale = DTYPE[dt], _impl(pair), dqk ** -0.5
    B, H, N = 2, 2, DIAG_N
    for shift in DIAG_SHIFTS:
        M = N + shift
        q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=20 + shift, poison=_diag_mask(B, M, shift))
        out = ops.attention(q, k, v, H, scale, causal=True, impl=impl)
        assert_parity(out, q, k, v, H, scale, None, True, what=f"{case_id(case)} shift {shift}", per_row=True)


@pytest.mark.parametrize("case", DIAG_VARIANTS, ids=case_id)
def test_causal_diagonal_sweep_m_shards(case):
    """Shards [0, 64), [64, 259), [259, M): the later ones have a negative causal shift, and rows whose diagonal lies
    before a shard see none of its keys; merged, they give the unsharded result."""
    from perceiver_io_b200 import ops

    dqk, dv, dt, pair = case
    dtype, impl, scale = DTYPE[dt], _impl(pair), dqk ** -0.5
    B, H, N = 2, 2, DIAG_N
    for shift in DIAG_SHIFTS:
        M = N + shift
        q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=40 + shift, poison=_diag_mask(B, M, shift))
        cuts = (0,) + DIAG_SHARD_CUTS + (M,)
        parts = []
        for a, b in zip(cuts[:-1], cuts[1:]):
            part = ops.attention_partial(q, k[:, a:b], v[:, a:b], H, scale, causal=True, m_total=M, m_offset=a, impl=impl)
            assert_partial_state(part, q, k[:, a:b], v[:, a:b], H, scale, None, True, M, a,
                                 what=f"{case_id(case)} shift {shift} shard [{a}, {b})")
            parts.append(part)
        merged = ops.combine_partials(*(torch.stack([p[i] for p in parts]) for i in range(3)), dtype)
        assert_parity(merged, q, k, v, H, scale, None, True, what=f"{case_id(case)} shift {shift} merged shards",
                      per_row=True)


# --------------------------------------------------------------------------------------------------
# 4: exact properties in the whole-unit plan (N > 66 * 128)
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", VARIANT_CASES, ids=case_id)
def test_whole_unit_plan_exact_properties(case):
    from perceiver_io_b200 import ops

    dqk, dv, dt, pair = case
    dtype, impl, scale = DTYPE[dt], _impl(pair), dqk ** -0.5
    B, H, N = 1, 2, 8600
    workers = workers_for(ops.device_info()["num_sms"], pair)
    name = case_id(case)
    for M, causal in ((300, False), (8700, True)):
        counts, _ = plan_segments(B, H, N, M, workers, pair)
        assert counts["slots"] == 0, "expected the whole-unit plan"
        q, k, v = _operands(B, N, M, H, dqk, dv, dtype, seed=30 + M)
        nopad = torch.zeros(B, M, dtype=torch.bool, device="cuda")
        out = ops.attention(q, k, v, H, scale, causal=causal, impl=impl)
        assert torch.equal(ops.attention(q, k, v, H, scale, pad_mask=nopad, causal=causal, impl=impl), out), \
            f"{name} causal={causal}: all-False pad != no pad"
    # q, k, v: M = 8700 now; a 300-key shard wholly in the past of every row, and one in the future of rows < 8300
    ks, vs = k[:, :300], v[:, :300]
    part = ops.attention_partial(q, ks, vs, H, scale, impl=impl)
    past = ops.attention_partial(q, ks, vs, H, scale, causal=True, m_total=300 + N - 1, m_offset=0, impl=impl)
    assert _part_equal(part, past), f"{name}: causal shard wholly in the past != non-causal partial state"
    fut = ops.attention_partial(q, ks, vs, H, scale, causal=True, m_total=8700, m_offset=8400, impl=impl)
    dead = assert_partial_state(fut, q, ks, vs, H, scale, None, True, 8700, 8400, what=f"{name} whole-unit future shard")
    assert dead == B * H * 8300, dead
