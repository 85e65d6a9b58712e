"""-m gpu: every instantiation of the FP8 tensor-core forward (attn_fwd_fp8_kernel<NQB, NVB, BF16>, and
tc_combine_kernel when the plan splits) at its tile, split, mask and descale edges.  The variant matrix, the operand
builders, the exact probes and the per-element gate live in fp8_fwd_variants.py; the CPU companion
(test_fp8_variants_cpu.py) checks that the matrix covers every instantiation, that the shapes have their plan
structure, that the probes are exact by construction and that the gate rejects mutated emulations.

Random operands are gated element by element against the fp64 emulation (fp8_emulation.emulate) with the bound of
fp8_fwd_variants.gate_terms; every gated call prints its worst err / gate and the accumulator precision A it implies.
Masked keys are poisoned (the top score of every row and V codes +-448), so a leaked key moves its row by far more
than the gate.  The needle and count probes are compared bit for bit."""
import pytest
import torch

from fp8_emulation import emulate
from fp8_fwd_variants import (BF16, DIAG_CASES, FLT_MAX, FP16, SCHEDULE_CASES, SCHEDULE_SHAPES, SEC1, U32, VARIANT_CASES,
                              case_id, check_schedule8, gate_report, live_mask, out_to_bhnd, probe_expected, probe_operands,
                              random_operands)
from fwd_variants import DIAG_N, DIAG_SHARD_CUTS, DIAG_SHIFTS, diag_poison_keys

pytestmark = pytest.mark.gpu

OUT = {BF16: torch.bfloat16, FP16: torch.float16}
REGIMES = ("none", "pad", "causal", "causal_pad")


def _sms():
    from perceiver_io_b200 import ops

    return ops.device_info()["num_sms"]


def _call(opnd, H, dt, **kw):
    from perceiver_io_b200 import ops

    q8, k8, vt8, qd, kd, vd = opnd
    with torch.no_grad():
        return ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, (q8.shape[-1] // H) ** -0.5, out_dtype=OUT[dt], **kw)


def _pad_mask(B, M, seed):
    """Random padding (about 30 %), batch row 1 fully padded, batch row 0's first two key tiles fully padded (a
    segment that starts there runs its first tiles at m = -FLT_MAX and rescales by alpha = 0 at the first live key)."""
    g = torch.Generator().manual_seed(seed)
    pad = torch.rand(B, M, generator=g) < 0.3
    pad[1, :] = True
    pad[0, :256] = True
    return pad


def _diag_mask(B, M, shift):
    m = torch.zeros(B, M, dtype=torch.bool)
    m[:, diag_poison_keys(M, shift)] = True
    return m


def _regime(name, B, M, N, seed):
    """(pad mask or None, causal, poisoned keys) of a mask regime; causal with m_total = M (shift M - N)."""
    pad = _pad_mask(B, M, seed) if "pad" in name else None
    causal = name.startswith("causal")
    poison = torch.zeros(B, M, dtype=torch.bool)
    if pad is not None:
        poison |= pad
    if causal:
        poison |= _diag_mask(B, M, M - N)
    return pad, causal, (poison if poison.any() else None)


def _gated(got, opnd, H, dt, what, pad=None, causal=False, m_total=None, m_offset=0, ref=None):
    """got (B, H, N, dv) float64 (the output, or part_o / part_l with dt None) against the emulation; prints the worst
    err / gate and the A it implies.  Returns the emulation."""
    q8, k8, vt8, qd, kd, vd = opnd
    if ref is None:
        ref = emulate(q8, k8, vt8, qd, kd, vd, H, (q8.shape[-1] // H) ** -0.5, None if pad is None else pad.cuda(),
                      causal, m_total, m_offset, workers=_sms())
    worst, a_meas, shares, ok = gate_report(got, ref, dt)
    print(f"{what}: err/gate {worst:.3f}  A measured {a_meas:.2e}  "
          + " ".join(f"{k} {v:.2f}" for k, v in shares.items()))
    assert torch.isfinite(got).all(), what
    assert ok.all(), f"{what}: max err / gate = {worst:.3f} (A measured {a_meas:.2e})"
    return ref


def _gated_partial(part, opnd, H, what, **kw):
    """The partial state: part_o / part_l gated, part_m exactly the fp32 rounding of the emulation's maximum, part_l
    within its fp32 error.  Returns (emulation, number of rows without a live key)."""
    o, m, l = part
    ref = _gated(o.double() / l.double()[..., None], opnd, H, None, what + " partial", **kw)
    assert torch.equal(m, ref["m"].float()), f"{what}: part_m is not fp32(s_max c)"
    tol = ref["l"] * (ref["rho"] + ref["nadd"] * U32 + ref["rho_w"])
    assert ((l.double() - ref["l"]).abs() <= tol).all(), f"{what}: part_l"
    return ref, int((m == -FLT_MAX).sum())


def _part_equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def _probe_check(opnd, H, dt, what, **kw):
    """Both probe outputs bit for bit: the 16-bit output and the partial state."""
    from perceiver_io_b200 import ops

    q8, k8, vt8, qd, kd, vd = opnd
    scale = (q8.shape[-1] // H) ** -0.5
    pad = kw.get("pad_mask")
    kw = dict(kw, pad_mask=None if pad is None else pad.cuda())
    out32, po, pm, pl = probe_expected(q8, k8, vt8, qd, kd, vd, H, scale, kw["pad_mask"], kw.get("causal", False),
                                       kw.get("m_total"), kw.get("m_offset", 0))
    B, Hh, N, dv = out32.shape
    want = out32.to(OUT[dt]).permute(0, 2, 1, 3).reshape(B, N, H * dv)
    with torch.no_grad():
        out = ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, scale, out_dtype=OUT[dt], **kw)
        part = ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, scale, partial=True, **kw)
    bad = (out != want).reshape(B, N, H, dv).any(dim=-1).nonzero()
    assert torch.equal(out, want), f"{what}: {len(bad)} rows differ, first (b, n, h) {bad[:4].tolist()}"
    assert torch.equal(part[0], po), f"{what}: part_o"
    assert torch.equal(part[1], pm), f"{what}: part_m"
    assert torch.equal(part[2], pl), f"{what}: part_l"


# --------------------------------------------------------------------------------------------------
# 1: every instantiation in four mask regimes, exact properties, partial state, a future shard
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", VARIANT_CASES, ids=case_id)
def test_variant_masks_exact_properties_and_partial_state(case):
    from perceiver_io_b200 import ops

    dqk, dv, dt = case
    B, N, M, H = SEC1
    name = case_id(case)
    nopad = torch.zeros(B, M, dtype=torch.bool, device="cuda")

    # no mask: two calls, an all-False pad mask and an expanded copy of a broadcast q give the same bits
    opnd = random_operands(B, N, M, H, dqk, dv, seed=1, Bq=1)
    out = _call(opnd, H, dt)
    _gated(out_to_bhnd(out, H), opnd, H, dt, f"{name} no mask")
    assert torch.equal(_call(opnd, H, dt), out), "two calls differ"
    assert torch.equal(_call(opnd, H, dt, pad_mask=nopad), out), "all-False pad != no pad"
    q8 = opnd[0]
    qx = q8.view(torch.uint8).expand(B, -1, -1).contiguous().view(torch.float8_e4m3fn)
    assert torch.equal(_call((qx,) + opnd[1:], H, dt), out), "broadcast q != expanded q"

    for regime in REGIMES[1:]:
        pad, causal, poison = _regime(regime, B, M, N, seed=7)
        o = random_operands(B, N, M, H, dqk, dv, seed=2 + REGIMES.index(regime), Bq=1 if pad is not None else None,
                            poison=poison)
        out = _call(o, H, dt, pad_mask=None if pad is None else pad.cuda(), causal=causal)
        _gated(out_to_bhnd(out, H), o, H, dt, f"{name} {regime}", pad=pad, causal=causal)
        if regime == "causal":
            assert torch.equal(_call(o, H, dt, pad_mask=nopad, causal=True), out), "causal: all-False pad != no pad"

    # partial state: a causal shard wholly in the past of every row is the non-causal state bit for bit
    part = _call(opnd, H, dt, partial=True)
    past = _call(opnd, H, dt, partial=True, causal=True, m_total=M + N - 1, m_offset=0)
    assert _part_equal(part, past), "causal shard wholly in the past != non-causal partial state"
    _gated_partial(part, opnd, H, f"{name}")

    # a shard in the causal future of rows n < 100, with padding (batch row 1: every key): dead rows average the shard
    pad, _, poison = _regime("causal_pad", B, M, N, seed=7)
    Ms, m_total, m_off = 100, 300, 200
    o = random_operands(B, N, Ms, H, dqk, dv, seed=9, poison=poison[:, :Ms])
    fut = _call(o, H, dt, partial=True, pad_mask=pad[:, :Ms].cuda(), causal=True, m_total=m_total, m_offset=m_off)
    _, dead = _gated_partial(fut, o, H, f"{name} future shard", pad=pad[:, :Ms], causal=True, m_total=m_total,
                             m_offset=m_off)
    # rows n < 100 of every batch row, every row of batch rows 0 and 1 (their first 256 keys are padded)
    assert dead == H * int((~live_mask(B, N, Ms, pad[:, :Ms], True, m_total, m_off).any(dim=-1)).sum()) == H * 500, dead
    assert torch.equal(fut[2][fut[1] == -FLT_MAX], torch.full_like(fut[2][fut[1] == -FLT_MAX], float(Ms)))


# --------------------------------------------------------------------------------------------------
# 2: needle and count probes, every variant and mask regime, bit for bit
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", VARIANT_CASES, ids=case_id)
def test_variant_probes_are_exact(case):
    dqk, dv, dt = case
    B, N, M, H = SEC1
    for regime in REGIMES:
        pad, causal, poison = _regime(regime, B, M, N, seed=7)
        for kind in ("needle", "count"):
            o = probe_operands(kind, B, N, M, H, dqk, dv, Bq=1 if pad is not None else None, poison=poison)
            _probe_check(o, H, dt, f"{case_id(case)} {kind} {regime}", pad_mask=pad, causal=causal)


# --------------------------------------------------------------------------------------------------
# 3: schedule shapes (structure asserted from the plan first)
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape_name", list(SCHEDULE_SHAPES))
@pytest.mark.parametrize("case", SCHEDULE_CASES, ids=case_id)
def test_schedule_shapes(case, shape_name):
    dqk, dv, dt = case
    print(check_schedule8(shape_name, case, _sms()))
    B, H, N, M = SCHEDULE_SHAPES[shape_name]
    name = f"{case_id(case)} {shape_name}"
    causal = shape_name == "whole_causal"
    poison = _diag_mask(B, M, M - N) if causal else None
    o = random_operands(B, N, M, H, dqk, dv, seed=11, poison=poison)
    out = _call(o, H, dt, causal=causal)
    _gated(out_to_bhnd(out, H), o, H, dt, name, causal=causal)
    for kind in ("needle", "count"):
        _probe_check(probe_operands(kind, B, N, M, H, dqk, dv, poison=poison), H, dt, f"{name} {kind}", causal=causal)
    if not causal:
        pad = torch.zeros(B, M, dtype=torch.bool)
        pad[:, 1:M:3] = True
        if B > 1:
            pad[-1, :] = True  # a fully padded batch row
        op = random_operands(B, N, M, H, dqk, dv, seed=12, poison=pad)
        part = _call(op, H, dt, partial=True, pad_mask=pad.cuda())
        _, dead = _gated_partial(part, op, H, f"{name} pad", pad=pad)
        assert dead == (H * N if B > 1 else 0), dead
        _probe_check(probe_operands("needle", B, N, M, H, dqk, dv, poison=pad), H, dt, f"{name} needle pad",
                     pad_mask=pad)
    if shape_name.startswith("whole"):
        # a 300-key shard in the future of rows < 8300: dead rows, gated and probed
        ks = slice(0, 300)
        os_ = random_operands(B, N, 300, H, dqk, dv, seed=14)
        fut = _call(os_, H, dt, partial=True, causal=True, m_total=8700, m_offset=8400)
        _, dead = _gated_partial(fut, os_, H, f"{name} future shard", causal=True, m_total=8700, m_offset=8400)
        assert dead == B * H * 8300, dead
        _probe_check(probe_operands("count", B, N, ks.stop, H, dqk, dv), H, dt, f"{name} future shard count",
                     causal=True, m_total=8700, m_offset=8400)


# --------------------------------------------------------------------------------------------------
# 4: causal diagonal sweep, single pass and as M-shards merged by combine_partials
# --------------------------------------------------------------------------------------------------
def _merge_refs(refs):
    """The emulation of shards merged exactly, with the gate terms carried by each shard's weight."""
    m = torch.stack([r["m"] for r in refs]).amax(dim=0)
    ws = [torch.exp2(r["m"] - m) * r["l"] for r in refs]
    wsum = sum(ws)
    out = {k: sum(w[..., None] * r[k] for w, r in zip(ws, refs)) / wsum[..., None] for k in ("out", "pv_hat", "flip")}
    out["rho"] = torch.stack([r["rho"] for r in refs]).amax(dim=0)
    out["rho_w"] = sum(r["rho_w"] for r in refs) + len(refs) * 2.0 ** -21
    out["nadd"] = sum(r["nadd"] for r in refs)
    return out


@pytest.mark.parametrize("case", DIAG_CASES, ids=case_id)
def test_causal_diagonal_sweep(case):
    from perceiver_io_b200 import ops

    dqk, dv, dt = case
    B, H, N = 2, 2, DIAG_N
    for shift in DIAG_SHIFTS:
        M = N + shift
        o = random_operands(B, N, M, H, dqk, dv, seed=20 + shift, poison=_diag_mask(B, M, shift))
        out = _call(o, H, dt, causal=True)
        _gated(out_to_bhnd(out, H), o, H, dt, f"{case_id(case)} shift {shift}", causal=True)
        _probe_check(probe_operands("needle", B, N, M, H, dqk, dv, poison=_diag_mask(B, M, shift)), H, dt,
                     f"{case_id(case)} shift {shift} needle", causal=True)
        q8, k8, vt8, qd, kd, vd = o
        v8 = vt8[..., :M].permute(0, 3, 1, 2).reshape(B, M, H * dv)
        cuts = (0,) + DIAG_SHARD_CUTS + (M,)
        parts, refs = [], []
        for a, b in zip(cuts[:-1], cuts[1:]):
            sh = (q8, k8[:, a:b].contiguous(), ops.fp8_transpose_v(v8[:, a:b].contiguous(), H), qd, kd, vd)
            part = _call(sh, H, dt, partial=True, causal=True, m_total=M, m_offset=a)
            ref, _ = _gated_partial(part, sh, H, f"{case_id(case)} shift {shift} shard [{a}, {b})", causal=True,
                                    m_total=M, m_offset=a)
            parts.append(part)
            refs.append(ref)
        merged = ops.combine_partials(*(torch.stack([p[i] for p in parts]) for i in range(3)), OUT[dt])
        _gated(out_to_bhnd(merged, H), o, H, dt, f"{case_id(case)} shift {shift} merged shards", ref=_merge_refs(refs))


# --------------------------------------------------------------------------------------------------
# 5: V^T slack past M is never read
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [(48, 112, BF16), (208, 176, FP16)], ids=case_id)
def test_vt_slack_is_never_read(case):
    """V^T with M_pad = roundup16(M) + 32 keys, the slack filled with 0x7F (e4m3 NaN), as a strided view of a larger
    buffer: the same bits as the zero-slack layout, for a ragged M and for M below one key tile."""
    dqk, dv, dt = case
    B, N, H = 2, 130, 2
    for M in (300, 100):
        for kind in ("random", "count"):
            o = (random_operands(B, N, M, H, dqk, dv, seed=50 + M) if kind == "random"
                 else probe_operands("count", B, N, M, H, dqk, dv))
            vt8 = o[2]
            mp = (M + 15) // 16 * 16 + 32
            buf = torch.full((B, H, dv + 16, mp + 48), 0x7F, dtype=torch.uint8, device="cuda")
            buf[:, :, :dv, :M] = vt8[..., :M].view(torch.uint8)
            slack = buf.view(torch.float8_e4m3fn)[:, :, :dv, :mp]
            assert slack.stride(2) == mp + 48 and slack.shape[-1] == mp
            for kw in ({}, {"causal": True, "m_total": M + N}, {"partial": True}):
                want = _call(o, H, dt, **kw)
                got = _call(o[:2] + (slack,) + o[3:], H, dt, **kw)
                same = _part_equal(got, want) if kw.get("partial") else torch.equal(got, want)
                assert same, f"{case_id(case)} M {M} {kind} {kw}: slack past M was read"


# --------------------------------------------------------------------------------------------------
# 6: descale indexing: v_descale[h, dv_off + c] of every pass, q_descale[h] * k_descale[h]
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [BF16, FP16])
def test_descale_indexing_by_needles(dt):
    """dv 304 runs passes at dv_off 0, 128 and 256 and H = 4: a live needle gives v8 * v_descale[h, c] bit for bit
    (v_descale distinct powers of two, so the channel, the pass and the head are all pinned) and part_m = fp32(16 c_h)
    pins q_descale[h] * k_descale[h]."""
    B, N, M, H, dqk, dv = 2, 150, 700, 4, 144, 304
    o = probe_operands("needle", B, N, M, H, dqk, dv)
    _probe_check(o, H, dt, f"needle H {H} dv {dv}")
    # every row's needle is live here: the output is v8[needle] * v_descale, which depends on every (h, c)
    _, po, pm, pl = probe_expected(*o, H, dqk ** -0.5)
    assert torch.equal(pl, torch.ones_like(pl)) and (pm > 160).all()
