"""CPU companion of test_gpu_merge_variants.py: the SIMT variant matrix reaches every (dtype, DVW, mode), the restated plan
is the library's, the count probe marks every split and tile edge, every probe is exact in fp32 (the restated fp32
algorithm equals fp64 bit for bit), and the probes reject mutants of the restated rules."""
import ctypes

import pytest
import torch

import merge_variants as MV
from merge_variants import FLT_MAX, SIMT_CASES, case_id

DT = MV.TORCH_DTYPE


def test_matrix_reaches_every_simt_variant():
    reach = MV.reachable_variants()
    covered = MV.all_cases_variants()
    print(f"[merge matrix] {len(SIMT_CASES)} cases cover {len(covered)} of {len(reach)} (dtype, DVW, mode)")
    assert len(reach) == 2 * 4 * 4 and covered == reach, sorted(reach - covered)
    inst = set().union(*(MV.case_instantiations(c) for c in SIMT_CASES))
    assert {i for i in MV.all_instantiations() if i[0] in ("attn_simt", "combine")} == inst
    assert {c.dqk for c in SIMT_CASES} >= {1, 37, 512, 513, 1024}
    assert {c.dv for c in SIMT_CASES} >= {1, 3, 64, 65, 128, 129, 256, 257, 512}
    assert {c.N for c in SIMT_CASES} == {1, 31, 32, 33}
    assert {c.M for c in SIMT_CASES} >= {1, 31, 32, 33, 255, 257, 511, 513, 767, 769}
    # both sides of every DVW step, and of the 48 KB shared-memory attribute; every plan fits 200 KB
    for lo, hi in ((64, 65), (128, 129), (256, 257)):
        assert MV.dvw_of(lo) * 2 == MV.dvw_of(hi)
    assert MV.dvw_of(512) == 8 and MV.dvw_of(513) is None
    smem = {c.plan.smem > MV.SMEM_DEFAULT for c in SIMT_CASES}
    assert smem == {True, False} and max(c.plan.smem for c in SIMT_CASES) <= MV.SMEM_MAX
    assert MV.simt_plan(1, 1, 1, 1, 1024, 512).smem > MV.SMEM_DEFAULT
    # broadcast q, strided rows, causal key shards, padding, each in every dtype
    for dt in MV.DTYPES:
        cs = [c for c in SIMT_CASES if c.dt == dt]
        assert any(c.Bq == 1 for c in cs) and any(c.strided for c in cs) and any(c.pad for c in cs)
        assert any(c.causal and c.m_offset > 0 for c in cs) and any(c.causal and c.m_offset == 0 for c in cs)


def test_split_plan_edges():
    """make_plan: splits of 32-key multiples, at most ceil(M / 256) of them, none empty; the last one ragged at M = 256k
    +- 1, and a ragged last tile wherever M is not a multiple of 32."""
    for M in [1, 31, 32, 33, 255, 256, 257, 511, 512, 513, 767, 769, 1023, 1025, 4095, 4097]:
        for B, H, N in [(1, 1, 1), (2, 2, 33), (4, 33, 64), (1, 1, 32 * 528)]:
            p = MV.simt_plan(B, H, N, M, 64, 64)
            rs = MV.split_ranges(M, p)
            assert p.kps % 32 == 0 and p.nsplit <= max(1, MV.cdiv(M, 256))
            assert rs[0][0] == 0 and rs[-1][1] == M and all(ke > kb for kb, ke in rs)
            assert all(rs[i][1] == rs[i + 1][0] for i in range(len(rs) - 1))
    assert MV.split_ranges(513, MV.simt_plan(1, 1, 1, 513, 64, 64)) == [(0, 192), (192, 384), (384, 513)]
    assert MV.split_ranges(257, MV.simt_plan(1, 1, 1, 257, 64, 64)) == [(0, 160), (160, 257)]
    assert MV.simt_plan(1, 1, 32 * 528, 4097, 64, 64).nsplit == 1     # enough CTAs: no split


def _params(B, H, N, M, dqk, dv):
    from perceiver_io_b200 import _lib

    p = _lib.AttnParams()
    p.q, p.k, p.v, p.out = 1 << 20, 2 << 20, 3 << 20, 4 << 20   # never dereferenced: the query touches no memory
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.q_stride_b, p.q_stride_n, p.q_stride_h = N * H * dqk, H * dqk, dqk
    p.k_stride_b, p.k_stride_m, p.k_stride_h = M * H * dqk, H * dqk, dqk
    p.v_stride_b, p.v_stride_m, p.v_stride_h = M * H * dv, H * dv, dv
    p.o_stride_b, p.o_stride_n, p.o_stride_h = N * H * dv, H * dv, dv
    p.scale, p.dtype, p.m_total, p.impl = 0.125, _lib.PCV_BF16, M, _lib.PCV_IMPL_SIMT
    return p


def test_restated_plan_matches_the_library():
    """pcv_attn_workspace_bytes with impl = simt is nsplit * R * (dv + 2) floats when the plan splits, else 0."""
    from perceiver_io_b200 import _lib

    lib = _lib.lib()
    shapes = {(c.B, c.H, c.N, c.M, c.dqk, c.dv) for c in SIMT_CASES}
    shapes |= {(1, 1, 1, M, 64, 64) for M in (256, 257, 4096, 4097, 65536, 135169)}
    shapes |= {(B, H, N, 5000, 8, 8) for B, H, N in [(1, 1, 32 * 264), (1, 1, 32 * 263), (2, 66, 64), (1, 1, 16896)]}
    seen = set()
    for B, H, N, M, dqk, dv in sorted(shapes):
        need = ctypes.c_size_t(0)
        assert lib.pcv_attn_workspace_bytes(ctypes.byref(_params(B, H, N, M, dqk, dv)), ctypes.byref(need)) == 0, \
            lib.pcv_last_error()
        assert need.value == MV.workspace_bytes(B, H, N, M, dqk, dv), (B, H, N, M, dqk, dv)
        seen.add(MV.simt_plan(B, H, N, M, dqk, dv).nsplit)
    print(f"[simt plan] {len(shapes)} shapes, split counts {sorted(seen)}")
    assert {1, 2, 3, 4, 256, 470} <= seen


@pytest.mark.parametrize("c", SIMT_CASES[::3], ids=case_id)
def test_count_probe_marks_every_split_and_tile_edge(c):
    marks = set(MV.edge_marks(c))
    rs = MV.split_ranges(c.M, c.plan)
    for kb, ke in rs:
        assert {kb, ke - 1} <= marks
        if (ke - kb) % 32:
            assert kb + (ke - kb - 1) // 32 * 32 in marks   # the ragged tile's first key
    q, k, v = MV.count_operands(c)
    S, L, _ = MV.DV.count_state(v, c.H, *MV.sets_of(c))
    assert S.abs().max().item() < 2 ** 24 and L.max().item() <= c.M


def _exact_cases():
    # one case per (dtype, mode) with every DVW step between them
    return [c for c in SIMT_CASES if c.dqk <= 513][::4]


@pytest.mark.parametrize("c", _exact_cases(), ids=case_id)
def test_simt_probes_are_exact(c):
    """The restated fp32 algorithm on the count and needle probes equals the exact expectations bit for bit."""
    q, k, v = MV.count_operands(c)
    in_range, live = MV.sets_of(c)
    got = MV.simt_emulate(c, q, k, v, 0.25)
    if c.partial:
        want = MV.count_partial_expect(v, c.H, in_range, live)
        for g, w in zip(got, want):
            assert torch.equal(g, w)
    else:
        assert torch.equal(got, MV.simt_count_expect(v, c.H, in_range, live, DT[c.dt]))
    for r in range(MV.needle_rounds(c, cap=1)):
        nd = MV.needle_set(c, r)
        q, k, v = MV.needle_operands(c, nd)
        got = MV.simt_emulate(c, q, k, v, MV.NEEDLE_SCALE)
        if not c.partial:
            assert torch.equal(got, MV.simt_needle_expect(c, v, in_range, live, nd))


@pytest.mark.parametrize("G", [1, 2, 3, 8, 37])
def test_dyadic_merges_are_exact(G):
    """The fp32 merge of the dyadic states equals the fp64 merge bit for bit, in every intermediate: the row max, l,
    the numerator, 1 / l (a power of two) and the normalised rows before their one 16-bit rounding."""
    po, pm, pl = MV.dyadic_states(G, 97, 33, seed=G)
    acc, m, l = MV.merge_state(po, pm, pl)
    racc, rm, rl = MV.merge_reference(po, pm, pl)
    assert torch.equal(acc.double(), racc) and torch.equal(m.double(), rm) and torch.equal(l.double(), rl)
    w, _ = MV.merge_weights(pm.double())
    assert (w[w > 0] >= 2.0 ** MV.MIN_PROBE_EXP).all()
    assert torch.equal(torch.frexp(l)[0].abs(), torch.full_like(l, 0.5)), "merged l must be a power of two"
    assert torch.equal((acc * (1.0 / l)[..., None]).double(), racc / rl[..., None])
    for dt in DT.values():
        assert torch.equal(MV.combine_emulate(po, pm, pl, dt), (racc / rl[..., None]).to(dt))
    kinds = [MV.ROW_KINDS[r % len(MV.ROW_KINDS)] for r in range(97)]
    dead = torch.tensor([k in ("dead", "dead_inf") for k in kinds])
    assert (m[dead] == -FLT_MAX).all() and torch.isfinite(m[~dead]).all()
    if G >= 3:
        assert (pm == float("-inf")).any() and (pm == -FLT_MAX).any()


def test_rescale_probes_are_exact():
    po, pm, pl, new_m = MV.rescale_states(101, 12, seed=3)
    o2, m2, l2 = MV.rescale_emulate(po, pm, pl, new_m)
    w = torch.where(pm.double() == float("-inf"), torch.zeros_like(pm.double()), torch.exp2(pm.double() - new_m.double()))
    assert torch.equal(o2.double(), po.double() * w[:, None]) and torch.equal(l2.double(), pl.double() * w)
    assert set(w.unique().tolist()) >= {0.0, 1.0} and (w < 2.0 ** -90).any() and (w > 0).sum() > 40
    assert (w[w > 0] >= 2.0 ** MV.MIN_PROBE_EXP).all()


def test_alignment_predicates():
    """The fast paths before and after the pointer terms: an odd-offset fp32 view (4-byte aligned) and an output at an
    odd element (2-byte aligned) passed the old predicates, which would have issued 16- and 8-byte accesses at them."""
    base = 1 << 20
    assert MV.rescale_vector(128, base + 4, aligned=False) and not MV.rescale_vector(128, base + 4)
    assert MV.rescale_vector(128, base) and not MV.rescale_vector(130, base)
    parts, outs, strides = [base, base + 4096], [base * 2, base * 3], (4096, 128, 32)
    assert MV.peers_fast_path(32, strides, parts, outs)
    assert not MV.peers_fast_path(132, strides, parts, outs) and not MV.peers_fast_path(30, strides, parts, outs)
    for p2, o2 in [([base, base + 4100], outs), (parts, [base * 2, base * 3 + 2]), (parts, [base * 2 + 4, base * 3])]:
        assert MV.peers_fast_path(32, strides, p2, o2, aligned=False) and not MV.peers_fast_path(32, strides, p2, o2)
    assert not MV.peers_fast_path(32, (4096, 130, 32), parts, outs)


# ---- mutants ----
def _simt_probes():
    """(name, case, operands, scale) of the probes the SIMT mutants meet: count probes of every matrix case with causal
    masking, a key shard, padding or a ragged split, and needles on the split edges of a split case."""
    out = []
    for c in SIMT_CASES:
        if c.dqk > 37:
            continue
        out.append((f"count {case_id(c)}", c, MV.count_operands(c), 0.25))
    for c in [c for c in SIMT_CASES if c.plan.nsplit > 1 and c.dqk <= 37][:4]:
        out.append((f"needle {case_id(c)}", c, MV.needle_operands(c, MV.needle_set(c, 0)), MV.NEEDLE_SCALE))
    return out


def _same(a, b):
    if isinstance(a, tuple):
        return all(_same(x, y) for x, y in zip(a, b))
    return torch.equal(a, b)


@pytest.mark.parametrize("mut", MV.SIMT_MUTANTS)
def test_simt_probes_reject_mutant(mut):
    for name, c, (q, k, v), scale in _simt_probes():
        if not _same(MV.simt_emulate(c, q, k, v, scale, mut), MV.simt_emulate(c, q, k, v, scale)):
            print(f"[mutant] {mut}: rejected by {name}")
            return
    pytest.fail(f"no probe rejects {mut}")


def _merge_probes():
    for G in (1, 2, 3, 8, 37):
        yield f"dyadic G={G}", MV.dyadic_states(G, 60, 5, seed=10 + G)


def test_merge_probes_reject_or_match_mutants():
    """-inf weight taken as 1 is equivalent on valid states: a -inf part holds o = 0, l = 0, so its weight multiplies
    zeros.  The finite fill weighted 0 only against a live part is equivalent too: exp2(-FLT_MAX - m) is 0 for every
    finite m.  The fill weighted 0 everywhere is rejected by the all-filled rows (l = 0)."""
    for mut in MV.MERGE_MUTANTS:
        rejected = None
        for name, (po, pm, pl) in _merge_probes():
            for dt in DT.values():
                a, b = MV.combine_emulate(po, pm, pl, dt, mut), MV.combine_emulate(po, pm, pl, dt)
                if not torch.equal(a, b):
                    rejected = rejected or f"{name} {dt}"
        print(f"[mutant] {mut}: " + (f"rejected by {rejected}" if rejected else "equivalent on every probe"))
        assert (rejected is None) == (mut in ("inf_weight_one", "ffill_weight_zero_vs_live")), mut


def _peer_run(G, dv, mut, call_ranks=None, rows=45, dtype=torch.bfloat16):
    po, pm, pl = MV.dyadic_states(G, rows, dv, seed=G + dv)
    outs = [torch.full((rows, dv), float("nan"), dtype=dtype) for _ in range(G)]
    for rank in (range(G) if call_ranks is None else call_ranks):
        rb, re = MV.peer_rows(rows, G, rank)
        MV.peers_emulate(po, pm, pl, outs, rb, re, rank, dtype, mut)
    return outs, MV.combine_emulate(po, pm, pl, dtype)


@pytest.mark.parametrize("mut", MV.PEER_MUTANTS)
def test_peer_probes_reject_mutant(mut):
    for G in (1, 2, 3, 8):
        for dv in (1, 3, 4, 128, 132):
            outs, want = _peer_run(G, dv, mut)
            if not all(torch.equal(o, want) for o in outs):
                print(f"[mutant] {mut}: rejected by peers G={G} dv={dv}")
                return
    pytest.fail(f"no probe rejects {mut}")


def test_peer_probe_passes_the_rule_and_keeps_other_rows():
    for G in (1, 2, 3, 8):
        outs, want = _peer_run(G, 132, None)
        assert all(torch.equal(o, want) for o in outs)
        outs, want = _peer_run(G, 4, None, call_ranks=[G - 1])
        rb, re = MV.peer_rows(45, G, G - 1)
        for o in outs:
            assert torch.equal(o[rb:re], want[rb:re]) and o[:rb].isnan().all() and o[re:].isnan().all()


@pytest.mark.parametrize("mut", MV.RESCALE_MUTANTS)
def test_rescale_probe_rejects_mutant(mut):
    po, pm, pl, new_m = MV.rescale_states(101, 12, seed=3)
    got = MV.rescale_emulate(po, pm, pl, new_m, mut)
    want = MV.rescale_emulate(po, pm, pl, new_m)
    bad = [n for n, a, b in zip(("o", "m", "l"), got, want) if not torch.equal(a, b)]
    print(f"[mutant] {mut}: rejected by the rescale probe ({', '.join(bad)})")
    assert bad
