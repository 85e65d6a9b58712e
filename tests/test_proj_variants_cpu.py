"""CPU companion of test_gpu_proj_variants.py (no GPU): the matrix reaches all 42 restated instantiations of the
LayerNorm-folded projection kernels (the GPU module's profiler check confirms them in the binary), the named shapes have
their structure, the restated backward split is the library's, the probes keep every intermediate exact, an fp32
emulation of the kernels' arithmetic stays within half of the element gates, and mutants of the kernels' indexing are
rejected by them."""
import ctypes

import pytest
import torch

import proj_variants as PV
from gpu_util import (UNIT_ROUNDOFF, lnlin_element_bounds, lnlin_magnitudes, proj_reference)

F32 = torch.float32


def test_matrix_reaches_every_instantiation():
    """The matrix, mapped through the restated launch rules, reaches the 42 restated instantiations.  This checks the
    matrix against the restatement only: the rules are applied to themselves, so it cannot disagree with the library.
    The evidence that the library launches exactly these 42 is test_gpu_proj_variants.py's profiler check."""
    want = PV.all_instantiations()
    assert len(want) == 42
    assert PV.matrix_instantiations() == want


@pytest.mark.parametrize("name", list(PV.PRODUCER_SHAPES))
def test_producer_shapes_have_their_structure(name):
    PV.check_producer_shape(name, cg=2)


@pytest.mark.parametrize("name", list(PV.STATS_SHAPES))
def test_stats_shapes_have_their_structure(name):
    PV.check_stats_shape(name)


@pytest.mark.parametrize("name", list(PV.BWD_SHAPES))
def test_bwd_shapes_have_their_structure(name):
    PV.check_bwd_shape(name)


def test_needs_subsets_cover_every_kernel_set():
    import itertools

    sets = {frozenset(PV.bwd_kernels(n)) for n in PV.NEEDS_SUBSETS.values()}
    every = {frozenset(PV.bwd_kernels(n)) for n in itertools.product((False, True), repeat=5) if any(n)}
    assert sets == every
    assert frozenset(PV.bwd_kernels((True, False, False, False, False))) == {"dx", "dx_fixup"}   # col_part = nullptr
    assert "dx_fixup" not in PV.bwd_kernels((False, False, False, True, False))                 # want_x = false


@pytest.mark.parametrize("shape", list(PV.BWD_SHAPES.values()) + [(1024, 1024, 1024, 2048), (2000, 64, 64, 0)])
def test_restated_plan_matches_the_library(shape):
    from perceiver_io_b200 import _lib

    rows, C, n_k, n_v = shape
    p = _lib.LnLinearBwdParams()
    p.rows, p.C, p.n_k, p.n_v, p.dtype = rows, C, n_k, n_v, _lib.PCV_BF16
    need = ctypes.c_size_t(0)
    assert _lib.lib().pcv_ln_linear_bwd_workspace_bytes(ctypes.byref(p), ctypes.byref(need)) == 0
    pl = PV.make_plan(rows, C, n_k, n_v)
    assert need.value == pl["bytes"]
    # the workspace grows by n * C * 4 bytes (+ n * 4) per split: a split count one off would not match
    for ds in (-1, 1):
        s = pl["splits"] + ds
        if s >= 1:
            up = lambda b: -(-b // 256) * 256
            other = (up(pl["tiles_c"] * rows * 8) + up(pl["m_blocks"] * C * 8) + up(s * (n_k + n_v) * C * 4)
                     + up(s * (n_k + n_v) * 4))
            assert other != need.value


def test_splits_reach_one_the_cap_and_kb_rows():
    assert PV.make_plan(*PV.BWD_SHAPES["splits1"])["splits"] == 1
    assert PV.make_plan(*PV.BWD_SHAPES["splits32"])["splits"] == 32
    pl = PV.make_plan(*PV.BWD_SHAPES["splits_kb_rows"])
    assert pl["splits"] == pl["kb_rows"]
    ranges = PV.split_rows(4000, PV.make_plan(4000, 128, 64, 64)["kb_rows"], 32)
    assert ranges[0][0] == 0 and ranges[-1][1] == 4000 and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_constant_row_mean_is_exact_at_every_register_width(dtype):
    """The producer writes t for a row whose separate statistics have var = 0, which needs the mean of a constant row
    to be exactly its value.  Both statistics kernels sum the row exactly (C copies of a 16-bit value fit in fp32) and
    then divide by C, which is exact.  Multiplying by the fp32 reciprocal instead is not: at C = 1792 (NCH 7) it moves
    the mean of 48, 100 and 1000 one ulp, and the row escapes the rule."""
    vals = torch.tensor([1.0, 1.5, 48.0, 100.0, 1000.0, -1000.0, 3.0, 65504.0 / 64]).to(dtype).float()
    for C in [256 * k for k in range(1, 9)] + [200, 2304]:
        total = vals * C
        assert torch.equal(total.double(), vals.double() * C)
        assert torch.equal(total / C, vals), C
    recip = (vals * 1792) * torch.tensor(1.0 / 1792, dtype=F32)
    assert not torch.equal(recip, vals)


# ---- probes ----
@pytest.mark.parametrize("C", [128, 256, 1024])
def test_producer_probe_keeps_intermediates_exact(C):
    rows, n = 64, 96
    x, gamma, beta, w, bias, mu, k = PV.producer_probe(rows, C, n, seed=1, ln=True)
    xd = x.double()
    assert torch.equal(xd.mean(1), mu) and torch.equal(((xd - mu[:, None]) ** 2).mean(1), 4.0 ** k)
    wc = (w.double() * gamma.double()[None])
    assert torch.equal(wc.to(torch.bfloat16).double(), wc), "gamma W exact in 16 bits"
    xw = xd @ wc.T
    assert xw.abs().max() < 2 ** 23 and torch.equal(xw.float().double(), xw)
    s = wc.float().sum(1).double()
    assert torch.equal(s, wc.sum(1))
    t = w.double() @ beta.double() + bias.double()
    assert torch.equal(t.float().double(), t)
    out = (xw - mu[:, None] * s) * (2.0 ** -k)[:, None] + t
    assert torch.equal(out.float().double(), out)


def test_backward_probe_keeps_intermediates_exact():
    rows, C, n = 300, 256, 200
    x, gamma, beta, w, G, mu, k = PV.bwd_probe(rows, C, n, seed=2)
    xh = (x.double() - mu[:, None]) * (2.0 ** -k)[:, None]
    assert torch.equal(xh.abs(), torch.ones_like(xh))
    dxh = (G.double() @ w.double()) * gamma.double()
    assert torch.equal(dxh.to(torch.bfloat16).double(), dxh) and torch.equal(dxh.to(torch.float16).double(), dxh)
    a, b = dxh.sum(1, keepdim=True), (dxh * xh).sum(1, keepdim=True)
    dx = (2.0 ** -k)[:, None] * (dxh - (a + xh * b) / C)
    assert torch.equal(dx.float().double(), dx)


def test_vt_probe_digits_identify_every_coordinate():
    rows, M, n_k, n_v, dv = 300, 100, 64, 128, 64
    coords = PV.vt_coords(rows, M, n_k, n_v, dv)
    flat = coords.reshape(-1, 4)
    assert torch.unique(flat, dim=0).shape[0] == flat.shape[0]
    assert int(coords[..., 3].max()) < 256 and int(coords[..., 2].max()) < 256
    # b and m swapped (the mutant) writes elsewhere
    mut = flat[:, [3, 1, 2, 0]]
    assert not torch.equal(mut, flat)


# ---- fp32 emulation of the kernels' arithmetic ----
def _tc_sum(a, b):
    """a (rows, C) @ b (n, C)^T as the tensor core accumulates: exact k16 partial sums added in fp32 in k order."""
    C = a.shape[1]
    parts = torch.einsum("rkc,nkc->rnk", a.double().reshape(a.shape[0], -1, 16), b.double().reshape(b.shape[0], -1, 16))
    acc = torch.zeros(a.shape[0], b.shape[0], dtype=F32)
    for j in range(C // 16):
        acc = acc + parts[:, :, j].float()
    return acc


def _emulate_producer(x, w_cat, col_st, eps, fuse):
    xf = x.float()
    C = xf.shape[1]
    if fuse:
        x0 = xf[:, :1]
        s1 = torch.zeros(x.shape[0], 2, dtype=F32)
        s2 = torch.zeros(x.shape[0], 2, dtype=F32)
        for c in range(C):
            h = (c // 32) % 2   # each thread of a pair reads half of every 64-channel line
            d = xf[:, c] - x0[:, 0]
            s1[:, h] += d
            s2[:, h] = s2[:, h] + d * d
        s1, s2 = s1.sum(1, keepdim=True), s2.sum(1, keepdim=True)
        dm = s1 * (1.0 / C)
        var = (s2 * (1.0 / C) - dm * dm).clamp_min(0)
        mean, rstd = x0 + dm, torch.where(var > 0, torch.rsqrt(var + eps), torch.zeros_like(var))
    else:
        mean = xf.sum(1, keepdim=True) / C
        var = ((xf - mean) ** 2).sum(1, keepdim=True) * (1.0 / C)
        rstd = 1.0 / torch.sqrt(var + eps)
    acc = _tc_sum(x, w_cat)
    s, t = col_st[:, 0].float(), col_st[:, 1].float()
    return (rstd * (acc - mean * s) + t).to(x.dtype)


def _proj_operands(rows, C, n, dtype, mean):
    g = torch.Generator().manual_seed(C + int(mean))
    x = (torch.randn(rows, C, generator=g) * 1.3 + mean).to(dtype)
    gamma = (1.0 + 0.2 * torch.randn(C, generator=g)).to(dtype)
    beta = (0.3 * torch.randn(C, generator=g)).to(dtype)
    w = (torch.randn(n, C, generator=g) * C ** -0.5).to(dtype)
    b = (0.1 * torch.randn(n, generator=g)).to(dtype)
    from perceiver_io_b200 import ops
    w_cat, col_st = ops.fold_ln_linear(gamma, beta, [w], [b], dtype)
    return x, w_cat, col_st


def _ratio(got, ref, e32, dtype):
    bound = 2.0 * (UNIT_ROUNDOFF[dtype] * ref.abs() + e32) + (2.0 ** -24 if dtype == torch.float16 else 0.0)
    return ((got.double() - ref).abs() / bound).max().item()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("fuse", [False, True], ids=["separate", "fused"])
@pytest.mark.parametrize("mean", [0.7, 48.0])
def test_emulated_producer_stays_within_half_the_gate(mean, fuse, dtype):
    x, w_cat, col_st = _proj_operands(96, 256, 64, dtype, mean)
    ref, e32 = proj_reference(x, w_cat, col_st, 1e-5, fuse=fuse)
    r = _ratio(_emulate_producer(x, w_cat, col_st, 1e-5, fuse), ref, e32, dtype)
    print(f"[emulation] producer mean={mean} fuse={fuse} {dtype}: worst err/bound {r:.3f}")
    assert r <= 0.55


def _emulate_dx(x, st, w, gamma, G):
    dtype = x.dtype
    C = x.shape[1]
    mean, rstd = st[:, :1].float(), st[:, 1:].float()
    xh = (x.float() - mean) * rstd
    dy = _tc_sum(G, w.T.contiguous())
    dxh = (dy * gamma.float()).to(dtype).float()
    a = torch.zeros(x.shape[0], 1)
    b = torch.zeros(x.shape[0], 1)
    for c0 in range(0, C, 128):
        a = a + (dy[:, c0:c0 + 128] * gamma.float()[c0:c0 + 128]).sum(1, keepdim=True)
        b = b + (dy[:, c0:c0 + 128] * gamma.float()[c0:c0 + 128] * xh[:, c0:c0 + 128]).sum(1, keepdim=True)
    return (rstd * (dxh - (a + xh * b) * (1.0 / C))).to(dtype)


def _bwd_operands(rows, C, n, dtype):
    g = torch.Generator().manual_seed(rows)
    x = (torch.randn(rows, C, generator=g) * 1.3 + 3.0).to(dtype)
    gamma = (torch.rand(C, generator=g) + 0.5).to(dtype)
    beta = (torch.randn(C, generator=g) * 0.5).to(dtype)
    w = (torch.randn(n, C, generator=g) / C ** 0.5).to(dtype)
    G = torch.randn(rows, n, generator=g).to(dtype)
    xf = x.float()
    mean = xf.mean(1, keepdim=True)
    st = torch.cat([mean, 1.0 / torch.sqrt(((xf - mean) ** 2).mean(1, keepdim=True) + 1e-5)], 1)
    return x, gamma, beta, w, G, st


def _fp64_grads(x, gamma, beta, w, G):
    import torch.nn.functional as F
    leaves = [t.double().requires_grad_() for t in (x, w, gamma, beta)]
    F.linear(F.layer_norm(leaves[0], (x.shape[1],), leaves[2], leaves[3], 1e-5), leaves[1]).backward(G.double())
    return [leaves[0].grad, leaves[1].grad, G.double().sum(0), leaves[2].grad, leaves[3].grad]


def _bwd_bounds(x, st, w, gamma, beta, G):
    rows, C = x.shape
    n = w.shape[0]
    pl = PV.make_plan(rows, C, n, 0)
    mags, rstd = lnlin_magnitudes(x, st, w, gamma, beta, G)
    return lnlin_element_bounds(mags, rstd, x.dtype, rows, C, n, pl["splits"], pl["m_blocks"]), pl


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_emulated_fixup_stays_within_half_the_gate(dtype):
    x, gamma, beta, w, G, st = _bwd_operands(200, 384, 128, dtype)
    ref = _fp64_grads(x, gamma, beta, w, G)
    bounds, _ = _bwd_bounds(x, st, w, gamma, beta, G)
    r = ((_emulate_dx(x, st, w, gamma, G).double() - ref[0]).abs() / bounds[0]).max().item()
    print(f"[emulation] fixup dx {dtype}: worst err/bound {r:.3f}")
    assert r <= 0.55


# ---- mutants ----
def _worst(got, ref, bound):
    return ((got.double() - ref.double()).abs() / bound).max().item()


def test_producer_mutants_are_rejected():
    dtype = torch.bfloat16
    x, w_cat, col_st = _proj_operands(150, 448, 128, dtype, 0.7)
    n_k = 64
    ref, e32 = proj_reference(x, w_cat, col_st, 1e-5)
    bound = 2.0 * (UNIT_ROUNDOFF[dtype] * ref.abs() + e32)
    good = _emulate_producer(x, w_cat, col_st, 1e-5, False)
    assert _worst(good, ref, bound) <= 1
    xd = x.double()
    mean = xd.mean(1, keepdim=True)
    rstd = 1 / (xd.var(1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    s, t = col_st[:, 0].double(), col_st[:, 1].double()
    xw = xd @ w_cat.double().T
    mutants = {
        "neighbour statistics": rstd.roll(-1, 0) * (xw - mean.roll(-1, 0) * s) + t,
        "K/V swapped at n_k": ref[:, torch.cat([torch.arange(n_k - 2), torch.tensor([n_k, n_k + 1, n_k - 2, n_k - 1]),
                                                torch.arange(n_k + 2, 128)])],
        "last C block dropped": rstd * (xd[:, :384] @ w_cat.double()[:, :384].T - mean * s) + t,
    }
    for name, m in mutants.items():
        r = _worst(m, ref, bound)
        print(f"[mutant] {name}: worst err/bound {r:.1f}")
        assert r > 1, name


def test_fuse_without_the_shift_is_rejected():
    dtype = torch.bfloat16
    x, w_cat, col_st = _proj_operands(64, 1024, 64, dtype, 200.0)
    ref, e32 = proj_reference(x, w_cat, col_st, 1e-5, fuse=True)
    bound = 2.0 * (UNIT_ROUNDOFF[dtype] * ref.abs() + e32)
    xf = x.float()
    C = x.shape[1]
    s1 = torch.zeros(64)
    s2 = torch.zeros(64)
    for c in range(C):
        s1 += xf[:, c]
        s2 = s2 + xf[:, c] * xf[:, c]
    m = s1 / C
    rstd = torch.rsqrt((s2 / C - m * m).clamp_min(0) + 1e-5)[:, None]
    mut = rstd.double() * (_tc_sum(x, w_cat).double() - m[:, None].double() * col_st[:, 0].double()) + col_st[:, 1].double()
    r = _worst(mut, ref, bound)
    print(f"[mutant] FUSE shifted by 0: worst err/bound {r:.1f}")
    assert r > 1


def test_backward_mutants_are_rejected():
    dtype = torch.bfloat16
    rows, C, n = 700, 256, 64
    x, gamma, beta, w, G, st = _bwd_operands(rows, C, n, dtype)
    ref = _fp64_grads(x, gamma, beta, w, G)
    bounds, pl = _bwd_bounds(x, st, w, gamma, beta, G)
    xd, Gd = x.double(), G.double()
    xh = (xd - xd.mean(1, keepdim=True)) / (xd.var(1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    dy = Gd @ w.double()
    # one dW split missing
    r0, r1 = PV.split_rows(rows, pl["kb_rows"], pl["splits"])[1]
    keep = torch.ones(rows, dtype=torch.bool)
    keep[r0:r1] = False
    dbm = Gd[keep].sum(0)
    dw_m = (xh[keep].T @ Gd[keep]).T * gamma.double() + dbm[:, None] * beta.double()
    # one colsum range missing (row blocks of range 3)
    b0, b1 = PV.colsum_ranges(pl["m_blocks"])[3]
    keep2 = torch.ones(rows, dtype=torch.bool)
    keep2[b0 * 128:b1 * 128] = False
    dg_m = (dy * xh)[keep2].sum(0)
    # the fixup with the first column tile's partials only
    rstd = 1 / (xd.var(1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    dxh = dy * gamma.double()
    a, b = dxh[:, :128].sum(1, keepdim=True), (dxh * xh)[:, :128].sum(1, keepdim=True)
    dx_m = rstd * (dxh - (a + xh * b) / C)
    for name, m, i in (("dW split missing", dw_m, 1), ("colsum range missing", dg_m, 3), ("fixup one tile", dx_m, 0)):
        r = _worst(m, ref[i], bounds[i])
        print(f"[mutant] {name}: worst err/bound {r:.1f}")
        assert r > 1, name
