"""CPU companion of test_gpu_aux_variants.py: the case matrix reaches all 17 rotary / KV-append / pad-packing
instantiations and both append paths, every large case passes more than one grid sweep under the restated grid
formulas, the library holds exactly these kernels without spills, the exact oracles are exact, and every gate and probe
rejects mutants of the rule it guards (computed in fp64 on the CPU)."""
import os
import re
import subprocess
from types import SimpleNamespace

import pytest
import torch

import aux_variants as AV
from aux_variants import APPEND_CASES, PACK_CASES, ROTARY_CASES
from conftest import ROOT


def test_matrix_reaches_every_instantiation_and_path():
    inst = AV.all_instantiations()
    assert len(inst) == 4 + 6 + 2 + 4 + 1
    assert AV.matrix_instantiations() == inst, sorted(inst - AV.matrix_instantiations())
    paths = {(c.dt, c.at, p) for c in APPEND_CASES if not c.fp8 for p in c.paths}
    for es_dt in (AV.BF16, AV.FP32):
        for at in (False, True):
            assert {(es_dt, at, "vec"), (es_dt, at, "scalar")} <= paths, (es_dt, at)
    print(f"[aux matrix] {len(ROTARY_CASES)} rotary, {len(APPEND_CASES)} append, {len(PACK_CASES)} pack cases; "
          f"append paths {sorted(paths)}")
    # the edges of the issue list, each present
    rc = ROTARY_CASES
    assert any(c.d % 2 and 0 < c.rd < c.d for c in rc if not c.fp8)
    assert {c.rd for c in rc} >= {0, 2} and any(c.rd == c.d for c in rc) and any(c.rd == c.d - 1 for c in rc)
    assert any(c.Ba == c.B > 1 and c.right_align for c in rc)
    assert any(c.Ba == 1 < c.B for c in rc)
    assert any(c.x_pad for c in rc) and any(c.y_pad for c in rc)
    for c in [c for c in rc if c.at and c.B == len(c.bounds)]:
        arow, _, ok = c.rows()
        flat = [r for rr in arow for r in rr]
        assert min(flat) < 0 and max(flat) >= c.capacity and c.capacity - 1 in flat
        assert {f for _, f in c.bounds} == {0, 1}
    for dt in (AV.BF16, AV.FP16, AV.E4M3):
        assert any(c.fp8 and c.dt == dt and c.rd == 0 for c in rc)
    ac = APPEND_CASES
    assert any(c.alias_k for c in ac if c.fp8) and any(c.alias_k for c in ac if not c.fp8)
    assert any(c.L_old == 0 and not c.at for c in ac) and any(c.pad for c in ac)
    tiny = [c for c in ac if min(c.Ck, c.Cv) * AV.ELEM_BYTES[c.dt] < 16]
    assert tiny and all(c.blocks == 1 for c in tiny if max(c.Ck, c.Cv) * AV.ELEM_BYTES[c.dt] < 16)
    assert {AV.ELEM_BYTES[c.dt] for c in tiny} == {2, 4}
    for c in [c for c in ac if c.at]:
        rows = [AV.dst_row(c.bounds[b % len(c.bounds)], r, c.capacity) for b in range(c.B) for r in range(c.n)]
        assert all(ok == (0 <= r < c.capacity) for r, ok in rows)
    assert any(min(c.bounds) < 0 for c in ac if c.at) and any(max(c.bounds) + c.n > c.capacity for c in ac if c.at)


def test_every_kernel_body_has_a_case_past_one_sweep():
    big = {
        "rotary": [c for c in ROTARY_CASES if not c.fp8 and c.sweeps > 1],
        "rotary_fp8": [c for c in ROTARY_CASES if c.fp8 and c.sweeps > 1],
        "kv_append vec": [c for c in APPEND_CASES if not c.fp8 and c.sweeps > 1 and c.paths == {"vec"}],
        "kv_append scalar": [c for c in APPEND_CASES if not c.fp8 and c.sweeps > 1 and c.paths == {"scalar"}],
        "kv_append_fp8": [c for c in APPEND_CASES if c.fp8 and c.sweeps > 1],
        "pack_pad": [c for c in PACK_CASES if c.sweeps > 1],
    }
    for k, cs in big.items():
        print(f"[sweeps] {k}: " + ", ".join(f"{c.name} {c.sweeps}" for c in cs))
        assert cs, k
    assert any(c.at for c in big["rotary"]) and any(c.at for c in big["kv_append vec"])
    # the sweep sizes of the issue's shapes
    assert AV.rotary_blocks(2, 4100, 8, 66) * AV.THREADS == 540_672 and AV.rotary_work(2, 4100, 8, 66) == 2_164_800
    assert AV.APPEND_MAX_BLOCKS * AV.THREADS == 270_336 and AV.PACK_MAX_BLOCKS * AV.THREADS == 262_144
    assert AV.PackCase("x", 1024, 8193).words == 266_240
    assert AV.pad_words_per_row(1) == 4 and AV.pad_words_per_row(128) == 4 and AV.pad_words_per_row(129) == 8


def test_restated_vec_predicate_and_in_place_skip():
    s = AV.Seg(0, 0, 2048, 128, 4096, 128, 5, 128, 0)
    assert AV.vec_path(s)
    for field in ("src", "dst", "s_sb", "s_sl", "d_sb", "d_sl", "row_bytes"):
        assert not AV.vec_path(s._replace(**{field: getattr(s, field) + 8})), field
    c = next(c for c in APPEND_CASES if c.alias_k and not c.fp8)
    segs = c.segments()
    assert segs[0].rows == 0 and segs[0].src == segs[0].dst and segs[2].rows == c.L_old
    assert [s.dst_row0 for s in segs] == [0, c.L_old, 0, c.L_old]
    no_cache = next(c for c in APPEND_CASES if c.L_old == 0 and not c.at)
    assert [s.rows for s in no_cache.segments()] == [0, no_cache.n, 0, no_cache.n]


def test_restated_row_rules():
    assert AV.at_rows((-3, 1), 2, 40) == (-1, -1, False) and AV.at_rows((-3, 0), 3, 40) == (0, 3, True)
    assert AV.at_rows((34, 1), 5, 40) == (39, 39, True) and AV.at_rows((38, 0), 2, 40) == (40, 2, False)
    assert AV.dst_row(-2, 1, 40) == (-1, False) and AV.dst_row(-2, 2, 40) == (0, True)
    assert AV.dst_row(36, 4, 40)[1] is False
    assert AV.angle_row0(50, 37, True) == 13 and AV.angle_row0(50, 37, False) == 0
    assert AV.a_stride_b(1, 3, 99) == 0 and AV.a_stride_b(1, 1, 99) == 99 and AV.a_stride_b(3, 3, 99) == 99


def test_restated_rules_match_the_host_layer():
    """ops._rotary_params sets angle_row0 and a_stride_b by the restated rules (checked on CPU tensors: the function
    only reads shapes, strides and pointers)."""
    from perceiver_io_b200 import _lib, ops

    for B, Ba, n, extra, ra in ((3, 1, 7, 4, True), (3, 3, 7, 4, True), (1, 1, 5, 0, False), (2, 2, 6, 3, False)):
        x = torch.zeros(B, n, 2 * 10)
        ang = torch.zeros(Ba, n + extra, 6)
        p = ops._rotary_params(x, x, 2, ang, ra, _lib.PCV_BF16)
        assert p.angle_row0 == AV.angle_row0(n + extra, n, ra) and p.a_stride_b == AV.a_stride_b(Ba, B, ang.stride(0))
        assert p.rotate_dim == 6 and p.d == 10


def test_angle_tables_distinguish_pair_channels():
    a = AV.angle_table(2, 30, 16, seed=1)
    z = AV.zero_angle_rows(a)
    assert z[:, 3].all() and z[:, 10].all() and int(z.sum()) == 2 * 4
    live = ~z
    assert (a[..., 0::2] != a[..., 1::2])[live].all()
    assert (a[:, 5] > 1e5).all() and (a[:, 6] > 1e8).all() and (a[:, 0].abs() < 8).all()
    assert not torch.equal(a[0], a[1])


# ---- the library's kernels ----
def _aux_entries():
    log = os.path.join(ROOT, "build", "pcv_aux.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was not built in this tree")
    out = {}
    for e in open(log).read().split("Compiling entry function")[1:]:
        mangled = e.split("'")[1]
        name = subprocess.run(["c++filt", mangled], capture_output=True, text=True).stdout.strip()
        name = re.sub(r"^(void )?(pcv::\(anonymous namespace\)::)?", "", name).split("(")[0]
        own = next(line for line in e.split("\n") if "spill" in line)
        stack, stores, loads = map(int, re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes "
                                                   r"spill loads", own).groups())
        out[name] = (stack, stores, loads)
    return out


def test_library_holds_exactly_the_17_aux_kernels_without_spills():
    """pcv_aux.cu compiles to these 17 kernels next to the 5 merge kernels (combine_kernel<T>, combine_peers_kernel<T>,
    rescale_kernel), nothing else.  None spills.  The ten rotary kernels keep a 32-byte stack frame: sincosf's
    large-argument (Payne-Hanek) reduction stores its partial products in a local array, the path the angles above 1e5
    of angle_table exercise; the append and pack kernels have no frame."""
    entries = _aux_entries()
    inst = {}
    merge = set()
    for name, v in entries.items():
        i = AV.instantiation_of(name)
        if i is None:
            merge.add(name.split("<")[0])
        else:
            assert i not in inst, name
            inst[i] = (name, v)
    assert set(inst) == AV.all_instantiations(), sorted(set(map(str, AV.all_instantiations())) ^ set(map(str, inst)))
    assert merge == {"combine_kernel", "combine_peers_kernel", "rescale_kernel"} and len(entries) == 17 + 5
    for i, (name, (stack, stores, loads)) in inst.items():
        assert stores == 0 and loads == 0, name
        assert stack == (32 if i[0].startswith("rotary") else 0), (name, stack)
    print(f"[aux ptxas] {len(inst)} kernels, no spills; rotary stack frames "
          f"{sorted({v[1][0] for i, v in inst.items() if i[0].startswith('rotary')})}")


# ---- exact oracles ----
def test_rd0_requantisation_emulation_is_the_kernel_arithmetic():
    """requant_rd0 forms (code * descale) * inv as two rounded fp32 products, then RNE e4m3 with saturation: checked
    against an fp64 evaluation of the same two roundings, and the saturation / zero / subnormal codes are reached."""
    g = torch.Generator().manual_seed(3)
    codes = (torch.randn(4, 3, 16, generator=g) * 60).to(torch.float8_e4m3fn)
    codes[0, 0, :4] = torch.tensor([448.0, -448.0, 0.0, -0.0]).to(torch.float8_e4m3fn)
    codes[1, 0, :4] = torch.tensor([2.0 ** -9, -3 * 2.0 ** -9, 5 * 2.0 ** -9, 2.0 ** -7]).to(torch.float8_e4m3fn)
    descale = torch.tensor([0.37, 1.0, 2.0 ** -5])
    inv = torch.tensor([3.1, 1.0, 2.0 ** 7])
    got = AV.requant_rd0(codes, descale, inv)
    p1 = (codes.double() * descale.double()[:, None]).float().double()
    p2 = (p1 * inv.double()[:, None]).float()
    want = p2.clamp(-448, 448).to(torch.float8_e4m3fn)
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
    vals = got.float()
    assert (vals.abs() == 448).any() and (vals == 0).any() and ((vals.abs() > 0) & (vals.abs() < 2.0 ** -6)).any()


def test_e4m3_codes_ties_saturation_and_infinities():
    """The torch expression rounds ties to even, flushes nothing, saturates past 464 and maps +-inf to +-448: the
    edges the GPU probes of kv_append_fp8_kernel use."""
    v = torch.tensor([1.0625, 1.1875, 2.0 ** -10, 3 * 2.0 ** -10, 2.0 ** -9, 463.0, 464.0, 466.0, float("inf"),
                      float("-inf"), -0.0, 432.0])
    got = AV.e4m3_codes(v, torch.ones_like(v)).float()
    want = torch.tensor([1.0, 1.25, 0.0, 2.0 ** -8, 2.0 ** -9, 448, 448, 448, 448, -448, -0.0, 448])
    assert torch.equal(got, want)
    assert torch.signbit(got[10])


# ---- mutants ----
def _rotary_probe(c: AV.RotaryCase, seed=0):
    """A CPU-size copy of the case (n <= 40) with the GPU test's operands: (case, x64 (B, n, H, d), angles)."""
    small = c._replace(n=min(c.n, 40), B=min(c.B, 4))
    if small.at:
        small = small._replace(bounds=small.bounds[:small.B])
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(small.B, small.n, small.H, small.d, generator=g, dtype=torch.float64)
    x = x.to(AV.TORCH_DTYPE[AV.BF16 if small.dt == AV.E4M3 else small.dt]).double()
    angles = AV.angle_table(small.Ba, small.n_angles, small.rd, seed)
    return small, x, angles


def _rotary_excess(c, x, angles, mut):
    """The GPU gate applied to the mutant: the mutant's output, rounded to the output type, against the correct fp64
    rotation."""
    _, _, ok = c.rows()
    ok = torch.tensor(ok)
    ref, mag = AV.rotate64(x, AV.select_angles(c, angles), c.rd)
    bad, _ = AV.rotate64(x, AV.select_angles(c, angles, mut if mut in ("angle_row_plus_1", "broadcast_batch_ignored")
                                             else None), c.rd, mut)
    out_dt = AV.E4M3 if c.fp8 else c.dt
    got = bad.to(AV.TORCH_DTYPE[out_dt]).double()
    return AV.rotary_excess(got, ref, mag, out_dt)[ok]


def test_rotary_gate_passes_the_rule():
    for c in ROTARY_CASES:
        c, x, angles = _rotary_probe(c)
        if c.fp8:
            continue   # e4m3 output is gated at the scale the GPU test picks
        assert _rotary_excess(c, x, angles, None).max().item() <= 0, c.name


@pytest.mark.parametrize("mut", AV.ROTARY_MUTANTS)
def test_rotary_gate_rejects_mutant(mut):
    for c in ROTARY_CASES:
        if c.fp8:
            continue
        c, x, angles = _rotary_probe(c)
        if _rotary_excess(c, x, angles, mut).max().item() > 0:
            print(f"[mutant] {mut}: rejected by {c.name}")
            return
    pytest.fail(f"no rotary case rejects {mut}")


def _append_probe(c: AV.AppendCase, seed=0):
    small = c._replace(n=min(c.n, 9), L_old=min(c.L_old, 12), Ck=min(c.Ck, 64), Cv=min(c.Cv, 64))
    g = torch.Generator().manual_seed(seed)
    dt = AV.TORCH_DTYPE[c.dt]
    cdt = torch.float8_e4m3fn if c.fp8 else dt
    rnd = lambda *s: torch.randn(*s, generator=g).to(dt)   # noqa: E731
    dst = [torch.randn(small.B, small.dst_rows, C, generator=g).to(cdt) for C in (small.Ck, small.Cv)]
    caches = [torch.randn(small.B, small.L_old, C, generator=g).to(cdt) for C in (small.Ck, small.Cv)]
    new = [rnd(small.B, small.n, C) for C in (small.Ck, small.Cv)]
    inv = [torch.rand(C, generator=g) * 30 + 1 for C in (small.Ck, small.Cv)] if c.fp8 else [None, None]
    return small, dst, caches, new, inv


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


@pytest.mark.parametrize("mut", AV.APPEND_MUTANTS)
def test_append_probe_rejects_mutant(mut):
    for c in APPEND_CASES:
        c, dst, caches, new, inv = _append_probe(c)
        want = AV.append_oracle(c, dst, *caches, *new, *inv)
        got = AV.append_oracle(c, dst, *caches, *new, *inv, mut=mut)
        if not all(torch.equal(_bits(a), _bits(b)) for a, b in zip(want, got)):
            print(f"[mutant] {mut}: rejected by {c.name}")
            return
    pytest.fail(f"no append case rejects {mut}")


@pytest.mark.parametrize("mut", AV.PACK_MUTANTS)
def test_pad_count_probe_rejects_mutant(mut):
    for c in PACK_CASES:
        pad = AV.probe_mask(min(c.B, 4), c.M, seed=c.M, stride_pad=c.stride_pad)
        want = AV.count_expect(pad, c.dv)
        assert torch.equal(AV.unpack_words(AV.pack_words(pad), c.M), pad)
        got = AV.count_expect(AV.unpack_words(AV.pack_words(pad, mut), c.M), c.dv)
        if not all(torch.equal(a, b) for a, b in zip(want, got)):
            print(f"[mutant] {mut}: rejected by {c.name}")
            return
    pytest.fail(f"no pack case rejects {mut}")


def test_pad_words_keep_the_bits_past_M_zero():
    for M in (1, 31, 33, 129, 4097):
        w = AV.pack_words(torch.ones(2, M, dtype=torch.bool))
        assert w.shape == (2, AV.pad_words_per_row(M))
        assert int(w[0].sum()) == sum(0xFFFFFFFF if 32 * (i + 1) <= M else (1 << max(0, M - 32 * i)) - 1
                                      for i in range(w.shape[1]))


# ---- the backward shim, on the CPU ----
def _shim_grad(gy, angles, H, right_align):
    from perceiver_io_b200 import ops

    ctx = SimpleNamespace(saved_tensors=(angles,), meta=(H, right_align))
    return ops._Rotary.backward(ctx, gy)[0]


SHIM_CASES = [(3, 7, 2, 9, 8, 3, 5, True), (2, 6, 3, 10, 10, 1, 0, False), (2, 5, 1, 33, 16, 2, 4, True)]


@pytest.mark.parametrize("B,n,H,d,f,Ba,extra,ra", SHIM_CASES)
def test_rotary_backward_shim_matches_fp64_autograd(B, n, H, d, f, Ba, extra, ra):
    """_Rotary.backward (an fp32 torch shim) against fp64 autograd of the rotation, with a[2p] != a[2p+1], odd d,
    right_align and broadcast angles: within 2^-20 of sum |gy| |J| per element (fp32 cos / sin and two products)."""
    g = torch.Generator().manual_seed(B * 100 + d)
    angles = AV.angle_table(Ba, n + extra, f, seed=d)[..., :f]
    angles = torch.where(angles.abs() > 1e4, angles * 1e-6, angles)       # the shim's torch.cos runs in fp32 too
    x = torch.randn(B, n, H * d, generator=g, dtype=torch.float64, requires_grad=True)
    gy = torch.randn(B, n, H * d, generator=g, dtype=torch.float64)
    AV.rotary_autograd64(x, angles, H, ra).backward(gy)
    got = _shim_grad(gy.float(), angles, H, ra).double()
    err = (got - x.grad).abs().max().item()
    print(f"[rotary shim] B{B} n{n} H{H} d{d} f{f} Ba{Ba}: max |err| {err:.2e}")
    assert err <= 2.0 ** -20 * 2 * gy.abs().max().item() * 4
    for mut in ("swapped_pair_angles", "one_angle_per_pair"):
        bad = AV.rotary_backward_mutant(gy, angles, H, ra, mut)
        assert (bad - x.grad).abs().max().item() > 1e-3, mut
