"""CPU companion of test_gpu_fp8_variants.py: the variant matrix covers every instantiation of the FP8 tensor-core
forward, the schedule shapes have their work-plan structure, the probes are exact by construction, and the per-element
gate rejects emulations of kernels with a rounding or descale defect that the old 2^-6 gate let through."""
import re

import pytest
import torch

from fp8_emulation import MUTANTS, emulate
from fp8_fwd_variants import (BF16, FP16, OLD_GATE, PROBE_SUM_LIMIT, SCHEDULE_CASES, SCHEDULE_SHAPES, SEC1, TILE,
                              VARIANT_CASES, boxes_per_tile, case_id, check_schedule8, gate_report, nqb8, out_to_bhnd,
                              probe_expected, probe_gap_and_sums, probe_operands, random_operands, reachable_variants,
                              ring_slots, round_out, tiles_per_segment, variants_of)

H100_SMS = 132


def _library_variants():
    """(NQB, NVB, dtype) of every attn_fwd_fp8_kernel instantiation compiled into the library (its symbol names)."""
    from perceiver_io_b200 import _lib

    with open(_lib.LIB_PATH, "rb") as f:
        blob = f.read()
    found = re.findall(rb"19attn_fwd_fp8_kernelILi(\d)ELi(\d)ELb([01])EEEv", blob)
    return {(int(a), int(b), BF16 if c == b"1" else FP16) for a, b, c in found}


def test_dispatch_reaches_eight_variants_and_the_library_has_exactly_those():
    reach = reachable_variants()
    assert len(reach) == 8
    assert _library_variants() == reach


def test_ring_holds_whole_key_tiles():
    for nqb in (1, 2):
        for nvb in (1, 2):
            assert ring_slots(nqb, nvb) == 12
            assert ring_slots(nqb, nvb) % boxes_per_tile(nqb) == 0


def test_variant_matrix_covers_every_variant_with_box_tails():
    covered = set()
    for case in VARIANT_CASES:
        covered |= variants_of(*case)
    assert covered == reachable_variants(), sorted(reachable_variants() - covered)
    # a qk head dim that is not a multiple of 128 zero-fills the tail of the last Q / K box, at NQB 1 and 2
    assert {nqb8(dqk) for dqk, _, _ in VARIANT_CASES if dqk % 128} == {1, 2}
    # one call runs an NVB 2 and an NVB 1 pass; dv 304 runs three passes
    assert any(len({v[1] for v in variants_of(*c)}) == 2 for c in VARIANT_CASES)
    assert any(dv > 256 for _, dv, _ in VARIANT_CASES)


def test_section_one_shape_runs_the_pipelined_loop_and_splits():
    B, N, M, H = SEC1
    lo, hi, _ = tiles_per_segment(B, H, N, M, H100_SMS)
    assert lo >= 3, (lo, hi)
    assert M % TILE


@pytest.mark.parametrize("shape_name", list(SCHEDULE_SHAPES))
@pytest.mark.parametrize("case", SCHEDULE_CASES, ids=case_id)
def test_schedule_shapes_have_their_plan_structure(case, shape_name):
    print(check_schedule8(shape_name, case, H100_SMS))


def test_print_tiles_per_segment_of_the_older_fp8_cases():
    """The cases of test_gpu_fp8.py run one key tile per segment on 132 SMs: no pipelined loop iteration, no rescale of
    O; the schedule shapes and section 1 here run many."""
    old = [(2, 2, 200, 1000), (3, 2, 130, 900), (2, 2, 200, 700), (1, 2, 130, 520), (2, 2, 64, 1500), (2, 4, 100, 300),
           (2, 2, 150, 517), (2, 2, 150, 583)]
    for B, H, N, M in old:
        stats = tiles_per_segment(B, H, N, M, H100_SMS)
        print(f"test_gpu_fp8 B {B} H {H} N {N} M {M}: tiles / segment min {stats[0]} max {stats[1]} mean {stats[2]:.2f}")
        assert stats[1] == 1
    B, N, M, H = SEC1
    print("section 1:", tiles_per_segment(B, H, N, M, H100_SMS))
    for name, (B, H, N, M) in SCHEDULE_SHAPES.items():
        print(name, tiles_per_segment(B, H, N, M, H100_SMS))


@pytest.mark.parametrize("kind", ["needle", "count"])
def test_probes_are_exact_by_construction(kind):
    """Score levels 16 c apart with c >= 10.5 (>= 168 > 160 log2 units: ex2.approx.ftz and exp2f give exactly 0), and
    integer P V sums small enough for the accumulator, for the largest probe shapes the GPU test runs."""
    shapes = [SEC1 + (dqk, dv) for dqk, dv, _ in VARIANT_CASES]
    shapes += [(B, N, M, H, dqk, dv) for (B, H, N, M) in SCHEDULE_SHAPES.values() if M < 10000
               for dqk, dv, _ in SCHEDULE_CASES]
    shapes += [(2, 120, 40000, 4, 208, 48), (2, 150, 700, 4, 144, 304)]
    for B, N, M, H, dqk, dv in shapes:
        poison = torch.zeros(B, M, dtype=torch.bool)
        poison[:, ::5] = True
        q8, k8, vt8, qd, kd, vd = probe_operands(kind, B, min(N, 256), M, H, dqk, dv, poison=poison, device="cpu")
        gap, sums, levels = probe_gap_and_sums(q8, k8, vt8, qd, kd, H, dqk ** -0.5)
        assert set(levels) <= {0.0, 16.0}, levels
        assert kind == "count" or gap >= 160, gap
        assert sums <= PROBE_SUM_LIMIT, (B, N, M, H, dqk, dv, sums)


def test_probe_expectation_on_the_cpu():
    """The probe formula agrees with the fp64 emulation up to its 16-bit rounding, with pad and causal masks."""
    B, N, M, H, dqk, dv = 2, 130, 300, 2, 48, 112
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, 40:200] = True
    pad[1] = True
    for kind in ("needle", "count"):
        o = probe_operands(kind, B, N, M, H, dqk, dv, poison=pad, device="cpu")
        out, po, pm, pl = probe_expected(*o, H, dqk ** -0.5, pad, True)
        ref = emulate(*o, H, dqk ** -0.5, pad, True)
        assert torch.allclose(out.double(), ref["out"], rtol=1e-6, atol=0)
        assert torch.equal(pl.double(), ref["l"])


def _mutant_verdicts(case, seed=1):
    """Worst err / gate of each mutated emulation (its output rounded to the output dtype) against the unmutated
    emulation, with the new gate and the old one, on the section-1 operands of `case`."""
    dqk, dv, dt = case
    B, N, M, H = SEC1
    o = random_operands(B, N, M, H, dqk, dv, seed=seed, Bq=1, device="cpu")
    scale = dqk ** -0.5
    ref = emulate(*o, H, scale, workers=H100_SMS)
    res = {}
    for mutant in (None,) + MUTANTS:
        if mutant == "vd_prev_pass" and dv <= 128:
            continue
        em = ref if mutant is None else emulate(*o, H, scale, workers=H100_SMS, mutant=mutant)
        got = round_out(em["out"], dt)
        worst, _, _, ok = gate_report(got, ref, dt)
        old_ok = bool(((got - ref["out"]).abs() <= OLD_GATE * ref["pv_abs"]).all())
        res[mutant] = (worst, bool(ok.all()), old_ok)
    return res


@pytest.mark.parametrize("case", [(112, 176, BF16), (208, 304, FP16)], ids=case_id)
def test_gate_rejects_every_mutant_the_emulation_passes(case):
    res = _mutant_verdicts(case)
    for mutant, (worst, ok, old_ok) in res.items():
        print(f"{case_id(case)} {mutant}: new gate err/gate {worst:.3g} {'accepts' if ok else 'rejects'}, "
              f"old 2^-6 gate {'accepts' if old_ok else 'rejects'}")
    assert res[None][1], "the unmutated emulation, rounded to the output dtype, fails the gate"
    rejected = {m for m, (_, ok, _) in res.items() if m is not None and not ok}
    assert rejected == set(MUTANTS), sorted(set(MUTANTS) - rejected)
