"""CPU companion of test_gpu_fwd_variants.py: the variant matrix covers every instantiation of the tensor-core forward
kernel, and every schedule shape has the work-plan structure it is meant to exercise (host-only plan, no GPU)."""
import re

import pytest

from fwd_variants import (DIAG_N, DIAG_SHARD_CUTS, DIAG_SHIFTS, SCHEDULE_SHAPES, SCHEDULE_VARIANTS, VARIANT_CASES, BF16,
                          FP16, case_id, check_schedule, nqb_of, reachable_variants, variants_of, workers_for)

H100_SMS = 132


def _library_variants():
    """(NQB, NVB, dtype, pair) of every attn_fwd_kernel instantiation compiled into the library (its symbol names)."""
    from perceiver_io_b200 import _lib

    with open(_lib.LIB_PATH, "rb") as f:
        blob = f.read()
    found = re.findall(rb"15attn_fwd_kernelILi(\d)ELi(\d)ELb([01])ELb([01])EEEv", blob)
    return {(int(a), int(b), BF16 if c == b"1" else FP16, d == b"1") for a, b, c, d in found}


def test_dispatch_reaches_forty_variants_and_the_library_has_exactly_those():
    reach = reachable_variants()
    assert len(reach) == 40
    assert _library_variants() == reach


def test_variant_matrix_covers_every_variant():
    covered = set()
    for dqk, dv, dt, pair in VARIANT_CASES:
        covered |= variants_of(dqk, dv, dt, pair)
    assert covered == reachable_variants(), sorted(reachable_variants() - covered)
    # head dims that are not multiples of 64 reach every NQB (zero-filled tail of the last Q/K box)
    assert {nqb_of(dqk) for dqk, *_ in VARIANT_CASES if dqk % 64} == set(range(1, 9))
    # one call runs two V passes with different NVB
    assert any(len(set(variants_of(*c))) == 2 for c in VARIANT_CASES)


def test_schedule_variants_cover_the_pipelined_kernels_and_two_serial_ones():
    got = set()
    for c in SCHEDULE_VARIANTS:
        got |= variants_of(*c)
    assert {v for v in reachable_variants() if v[0] <= 2} <= got
    assert {3, 7} <= {v[0] for v in got}


@pytest.mark.parametrize("shape_name", list(SCHEDULE_SHAPES))
@pytest.mark.parametrize("case", SCHEDULE_VARIANTS, ids=case_id)
def test_schedule_shapes_have_their_plan_structure(case, shape_name):
    """The same check the GPU test makes with the device's SM count, for an H100 SXM: 132 workers, 66 CTA pairs."""
    print(check_schedule(shape_name, case, workers_for(H100_SMS, case[3])))


def test_diagonal_sweep_crosses_the_mask_free_tile_boundary():
    """Key tile [j0, j0 + 128) is mask-free for the warpgroup starting at row n_wg iff j0 + 127 <= n_wg + shift.  The
    sweep must put a tile's last key exactly on a first row's diagonal and exactly one key past it, single pass and in
    the interior shards (shift - m_offset)."""
    def edges(shift, N):
        on = past = False
        for n_wg in range(0, N, 64):
            for j0 in range(0, N + shift, 128):
                on |= j0 + 127 == n_wg + shift
                past |= j0 + 127 == n_wg + shift + 1
        return on, past

    assert all(any(edges(s, DIAG_N)) for s in DIAG_SHIFTS if s % 64 in (62, 63))
    assert any(edges(s, DIAG_N)[1] for s in DIAG_SHIFTS)
    assert any(edges(s, DIAG_N)[0] for s in DIAG_SHIFTS)
    assert any(edges(s - a, DIAG_N)[1] for s in DIAG_SHIFTS for a in DIAG_SHARD_CUTS)
