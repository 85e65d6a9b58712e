"""-m gpu: every instantiation of the LayerNorm-folded projection kernels (csrc/pcv_kvproj.cu, csrc/pcv_lnlin_bwd.cu)
at its tile, split and statistics edges.  The rules, the matrix and the probes live in proj_variants.py;
test_proj_variants_cpu.py checks that the matrix reaches all 42 instantiations, that the shapes have their structure,
that the restated split is the library's, and that the gates see the bugs they are for.

Exact probes (small integers, power-of-two gamma, rows mu +- 2^k with eps = 0) must equal RN16 of the fp64 value bit
for bit; random operands go through the element-wise gates of gpu_util (proj_reference, lnlin_element_bounds) and the
whole-tensor derived gate together."""
import pytest
import torch
import torch.nn.functional as F

import proj_variants as PV
from test_gpu_ln_linear_bwd import route  # noqa: F401 (fixture: the training route and the fp64 attention)
from gpu_util import (UNIT_ROUNDOFF, assert_e4m3_codes, assert_lnlin_elements, assert_proj_elements, derived_bound,
                      fold_term, lnlin_element_bounds, lnlin_magnitudes, proj_reference)

pytestmark = pytest.mark.gpu

DEV = "cuda"
DT = PV.TORCH_DTYPE
MODES = ("none", "separate", "fused")


def _ops():
    from perceiver_io_b200 import ops
    return ops


def _x_rows(x, stride):
    """x (rows, C) as a view of a (rows, stride) buffer."""
    rows, C = x.shape
    if stride == C:
        return x.contiguous()
    buf = torch.zeros(rows, stride, dtype=x.dtype, device=x.device)
    buf[:, :C] = x
    return buf[:, :C]


def _project(x, w_cat, col_st, n_k, n_v, mode, cg):
    ops = _ops()
    eps = None if mode == "none" else 1e-5
    k, v = ops.kv_project(x, w_cat, col_st, n_k, n_v, eps=eps, cta_group=cg,
                          stats=None if mode == "none" else mode)
    parts = [t for t in (k, v) if t is not None]
    return torch.cat(parts, 1)


def _random_case(rows, C, n, dtype, seed, mean=0.7):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(rows, C, generator=g) * 1.3 + mean).to(dtype)
    gamma = (1.0 + 0.2 * torch.randn(C, generator=g)).to(dtype)
    beta = (0.3 * torch.randn(C, generator=g)).to(dtype)
    w = (torch.randn(n, C, generator=g) * C ** -0.5).to(dtype)
    b = (0.1 * torch.randn(n, generator=g)).to(dtype)
    return [t.to(DEV) for t in (x, gamma, beta, w, b)]


def _bits(a, b, what):
    a, b = a.contiguous(), b.to(a.device).contiguous()
    eq = (a.view(torch.int16) == b.view(torch.int16)) | ((a == 0) & (b == 0))
    if not bool(eq.all()):
        i = (~eq).nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int((~eq).sum())} of {eq.numel()} differ; first at {i}: got "
                             f"{a[tuple(i)].item()!r} want {b[tuple(i)].item()!r}")


# ---- producer: random operands, every shape x mode x CG x dtype, both gates ----
@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", list(PV.PRODUCER_SHAPES))
def test_producer_random_operands(shape, mode, cg, dt):
    rows, C, n_k, n_v, xs = PV.PRODUCER_SHAPES[shape]
    dtype = DT[dt]
    PV.check_producer_shape(shape, cg=2)
    x, gamma, beta, w, b = _random_case(rows, C, n_k + n_v, dtype, seed=rows + C)
    ln = mode != "none"
    ops = _ops()
    w_cat, col_st = ops.fold_ln_linear(gamma if ln else None, beta if ln else None, [w], [b], dtype)
    xv = _x_rows(x, xs)
    got = _project(xv, w_cat, col_st, n_k, n_v, mode, cg)
    ref, e32 = proj_reference(x, w_cat, col_st, 1e-5 if ln else None, fuse=mode == "fused")
    inst = PV.case_instantiations("proj", dt, has_stats=mode == "separate", ln_eps=1e-5 if ln else 0.0, cg=cg)
    what = f"{shape} {mode} cg={cg} {dt} {sorted(inst)}"
    assert_proj_elements(got, ref, e32, dtype, what)
    if ln:   # module semantics: fp64 LayerNorm -> Linear on the 16-bit parameters, plus the fold's rounding
        sem = F.linear(F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-5), w.double(), b.double())
        assert_proj_elements(got, sem, e32 + fold_term(x, gamma, w, 1e-5, dtype) / 2, dtype, what + " vs LayerNorm")
        eager = F.linear(F.layer_norm(x, (C,), gamma, beta, 1e-5), w, b)
        bound, eerr, _ = derived_bound(sem, eager)
        err = (got.double() - sem).abs().max().item()
        assert err <= bound, f"{what}: whole-tensor err {err:.3e} > {bound:.3e}"
    # two calls are bitwise equal
    _bits(got, _project(xv, w_cat, col_st, n_k, n_v, mode, cg), what + " determinism")


# ---- producer: exact probes ----
def _probe_ref(x, mu, k, gamma, beta, w, bias):
    """LayerNorm -> Linear of a probe in closed form: x_hat = (x - mu) 2^-k = +-1 exactly, so every term is exact in
    fp64 (fp64 layer_norm leaves a residue of ~1e-16 where the exact value is 0)."""
    xh = (x.double() - mu[:, None]) * (2.0 ** -k)[:, None]
    return xh @ (w.double() * gamma.double()[None]).T + w.double() @ beta.double() + bias.double()


def _bwd_probe_ref(x, mu, k, gamma, beta, w, G):
    """(dx, dW, db, dgamma, dbeta) of a backward probe in closed form (exact in fp64)."""
    xh = (x.double() - mu[:, None]) * (2.0 ** -k)[:, None]
    g, b, W, Gd = gamma.double(), beta.double(), w.double(), G.double()
    C = x.shape[1]
    dy = Gd @ W
    dxh = dy * g
    dx = (2.0 ** -k)[:, None] * (dxh - (dxh.sum(1, keepdim=True) + xh * (dxh * xh).sum(1, keepdim=True)) / C)
    db = Gd.sum(0)
    return [dx, (xh.T @ Gd).T * g + db[:, None] * b, db, (dy * xh).sum(0), dy.sum(0)]



PROBE_SHAPES = [(1, 256, 128, 64), (129, 128, 64, 72), (300, 512, 192, 128), (260, 1024, 128, 256)]


@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("shape", PROBE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_producer_probe_without_layernorm_is_exact(shape, cg, dt):
    rows, C, n_k, n_v = shape
    dtype = DT[dt]
    x, _, _, w, bias, _, _ = PV.producer_probe(rows, C, n_k + n_v, seed=rows, ln=False, dtype=dtype)
    ops = _ops()
    w_cat, col_st = ops.fold_ln_linear(None, None, [w.to(DEV)], [bias.to(DEV)], dtype)
    got = _project(x.to(DEV), w_cat, col_st, n_k, n_v, "none", cg)
    want = (x.double() @ w.double().T + bias.double()).to(dtype)
    _bits(got, want, f"no-LN probe {shape} cg={cg} {dt}")


@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("shape", PROBE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_producer_probe_with_separate_statistics_is_exact(shape, cg, dt):
    """Rows mu +- 2^k, eps = 0: pcv_ln_stats returns (mu, 2^-k) exactly, and the output is RN16 of the fp64 value."""
    rows, C, n_k, n_v = shape
    dtype = DT[dt]
    x, gamma, beta, w, bias, mu, k = PV.producer_probe(rows, C, n_k + n_v, seed=rows + 1, ln=True, dtype=dtype)
    ops = _ops()
    xd = x.to(DEV)
    st = ops.ln_stats(xd, 0.0).cpu()
    assert torch.equal(st[:, 0].double(), mu) and torch.equal(st[:, 1].double(), 2.0 ** -k), "probe statistics"
    w_cat, col_st = ops.fold_ln_linear(gamma.to(DEV), beta.to(DEV), [w.to(DEV)], [bias.to(DEV)], dtype)
    got = torch.cat([t for t in ops.kv_project(xd, w_cat, col_st, n_k, n_v, eps=0.0, cta_group=cg) if t is not None], 1)
    ref = _probe_ref(x, mu, k, gamma, beta, w, bias)
    _bits(got, ref.to(dtype), f"LN probe {shape} cg={cg} {dt}")


@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("mode", ["none", "separate"])
def test_e4m3_producer_probe_is_exact(mode, dt):
    """The e4m3 producer on the probes: power-of-two inv_scale keeps (acc + t) inv exact, so every code is the e4m3
    RN code of the fp64 value; V^T holds the same codes as K at the transposed place (K and V share their weights)."""
    dtype = DT[dt]
    B, M, C, n_k, H, dv = 3, 100, 256, 128, 4, 32
    rows = B * M
    x, gamma, beta, w, bias, mu, k = PV.producer_probe(rows, C, n_k, seed=5, ln=mode == "separate", dtype=dtype)
    ops = _ops()
    eps = None if mode == "none" else 0.0
    wk = w.to(DEV)
    w_cat, col_st = ops.fold_ln_linear(None if eps is None else gamma.to(DEV), None if eps is None else beta.to(DEV),
                                       [wk, wk], [bias.to(DEV), bias.to(DEV)], dtype)
    inv = torch.full((2 * n_k,), 2.0 ** -4, device=DEV)
    k8, vt8 = ops.kv_project_fp8(x.to(DEV).view(B, M, C), w_cat, col_st, inv, n_k, n_k, H, eps=eps)
    if eps is None:
        ref = x.double() @ w.double().T + bias.double()
    else:
        ref = _probe_ref(x, mu, k, gamma, beta, w, bias)
    want = (ref * 2.0 ** -4).clamp(-448, 448).float().to(torch.float8_e4m3fn)
    want = want.view(torch.uint8) & torch.where(ref == 0, 0x7F, 0xFF).to(torch.uint8)   # +0 for an exact 0
    got_k = k8.reshape(rows, n_k).view(torch.uint8).cpu()
    got_k = torch.where(got_k == 0x80, 0, got_k).to(torch.uint8)
    assert torch.equal(got_k, want), "K codes"
    vt_want = want.reshape(B, M, H, dv).permute(0, 2, 3, 1)
    got_vt = vt8[..., :M].view(torch.uint8).cpu()
    assert torch.equal(torch.where(got_vt == 0x80, 0, got_vt).to(torch.uint8), vt_want), "V^T codes"


def test_e4m3_vt_lands_at_its_coordinates():
    """Each V^T element's (b, h, c, m) written digit by digit (base 16, exact in e4m3): M = 100 (not a multiple of 16),
    so 128-row tiles cross batch boundaries."""
    ops = _ops()
    B, M, C, n_k, n_v, H = 3, 100, 64, 64, 128, 2
    dv = n_v // H
    rows = B * M
    coords = PV.vt_coords(rows, M, n_k, n_v, dv)
    inv = torch.ones(n_k + n_v, device=DEV)
    col_st = torch.zeros(n_k + n_v, 2, device=DEV)
    got = torch.zeros(B, H, dv, M, 4, dtype=torch.int64)
    for coord in range(4):
        for digit in range(2):
            x, w = PV.vt_digit_probe(coord, digit, rows, C, n_k, n_v, M, dv)
            _, vt8 = ops.kv_project_fp8(x.to(DEV).view(B, M, C), w.to(DEV), col_st, inv, n_k, n_v, H, eps=None)
            got[..., coord] += vt8[..., :M].float().cpu().long() << (4 * digit)
    want = torch.zeros(B, H, dv, M, 4, dtype=torch.int64)
    b, h, c, m = coords.reshape(-1, 4).unbind(-1)
    want[b, h, c, m] = coords.reshape(-1, 4)
    assert torch.equal(got, want)


@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", ["rows127_c200", "pair_spare", "c1024_ring", "nk0", "kv_split64"])
def test_e4m3_producer_random_operands(shape, mode, dt):
    rows, C, n_k, n_v, _ = PV.PRODUCER_SHAPES[shape]
    n_k, n_v = n_k // 16 * 16, n_v // 16 * 16 or 16
    dtype = DT[dt]
    H = 1
    B, M = 1, rows
    x, gamma, beta, w, b = _random_case(rows, C, n_k + n_v, dtype, seed=C)
    ln = mode != "none"
    ops = _ops()
    w_cat, col_st = ops.fold_ln_linear(gamma if ln else None, beta if ln else None, [w], [b], dtype)
    inv = torch.full((n_k + n_v,), 16.0, device=DEV)
    old = ops.kv_project_config["stats"]
    ops.kv_project_config["stats"] = "fused" if mode == "fused" else "separate"
    try:
        k8, vt8 = ops.kv_project_fp8(x.view(B, M, C), w_cat, col_st, inv, n_k, n_v, H, eps=1e-5 if ln else None)
    finally:
        ops.kv_project_config["stats"] = old
    ref, e32 = proj_reference(x, w_cat, col_st, 1e-5 if ln else None, fuse=mode == "fused")
    parts = ([k8.reshape(rows, n_k)] if n_k else []) + [vt8[0, 0, :, :M].T]
    codes = torch.cat(parts, 1)
    inst = PV.case_instantiations("proj", dt, has_stats=mode == "separate", ln_eps=1e-5 if ln else 0.0, fp8=True)
    assert_e4m3_codes(codes, ref, e32, inv, f"{shape} e4m3 {mode} {dt} {sorted(inst)}")


# ---- row statistics ----
@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("shape", list(PV.STATS_SHAPES))
def test_ln_stats_variants(shape, dt):
    """Every register width, the generic vector and scalar paths, past both grid-stride sweeps: mean within (C / 32 + 8)
    u32 mean|x| and rstd within (C / 32 + 16) u32 relative of fp64; the exact probe rows (eps = 0) bit for bit."""
    rows, C, stride, off = PV.STATS_SHAPES[shape]
    route = PV.check_stats_shape(shape)
    dtype = DT[dt]
    ops = _ops()
    g = torch.Generator().manual_seed(rows + C)
    x = (torch.randn(rows, C, generator=g) * 2 + 5).to(dtype).to(DEV)
    buf = torch.zeros(rows * stride + off + 8, dtype=dtype, device=DEV)
    xv = buf[off:off + rows * stride].view(rows, stride)[:, :C]
    xv.copy_(x)
    assert (xv.data_ptr() % 16 == 0) == (off % 8 == 0)
    st = ops.ln_stats(xv, 1e-5).double()
    xd = x.double()
    mean = xd.mean(1)
    rstd = (xd.var(1, unbiased=False) + 1e-5).rsqrt()
    u32 = 2.0 ** -24
    merr = ((st[:, 0] - mean).abs() / ((C / 32 + 8) * u32 * xd.abs().mean(1))).max().item()
    rerr = ((st[:, 1] - rstd).abs() / ((C / 32 + 16) * u32 * rstd)).max().item()
    print(f"[ln_stats] {shape} {dt} {route}: mean err/bound {merr:.3f} rstd err/bound {rerr:.3f}")
    assert merr <= 1 and rerr <= 1
    if C & (C - 1) == 0:   # the exact probe
        xp, _, _, _, _, mu, k = PV.producer_probe(min(rows, 300), C, 8, seed=3, ln=True, dtype=dtype)
        sp = ops.ln_stats(xp.to(DEV), 0.0).cpu().double()
        assert torch.equal(sp[:, 0], mu) and torch.equal(sp[:, 1], 2.0 ** -k)


# ---- backward ----
def _bwd_ref(x, gamma, beta, w, G, eps):
    leaves = [t.detach().double().requires_grad_() if t is not None else None for t in (x, w, gamma, beta)]
    xx, ww, gg, be = leaves
    out = F.linear(F.layer_norm(xx, (xx.shape[1],), gg, be, eps), ww)
    bb = torch.zeros(w.shape[0], dtype=torch.float64, device=x.device, requires_grad=True)
    (out + bb).backward(G.double())
    return [xx.grad, ww.grad, bb.grad, None if gg is None else gg.grad, None if be is None else be.grad]


def _bwd_run(x, st, w, gamma, beta, G, n_k, n_v, needs, g_layout="plain"):
    ops = _ops()
    gk, gv = (G[:, :n_k] if n_k else None), (G[:, n_k:] if n_v else None)
    if g_layout == "wide":   # row strides larger than the widths
        gk = None if gk is None else torch.cat([gk, torch.zeros_like(gk[:, :8])], 1)[:, :n_k]
        gv = None if gv is None else torch.cat([gv, torch.zeros_like(gv[:, :8])], 1)[:, :n_v]
    elif g_layout == "copied":   # transposed storage: must be copied to rows
        gk = None if gk is None else gk.t().contiguous().t()
        gv = None if gv is None else gv.t().contiguous().t()
    return ops.ln_linear_backward(x, st, w, gamma, beta, gk, gv, n_k, n_v, needs)


BWD_CASES = ([(s, "all", True, "plain") for s in PV.BWD_SHAPES]
             + [("mblocks5", nd, True, "plain") for nd in PV.NEEDS_SUBSETS if nd != "all"]
             + [("mblocks11", "all", False, "plain"), ("nk0", "all", True, "wide"), ("mblocks5", "all", True, "copied")])


@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: "-".join(map(str, c)))
def test_backward_random_operands(case, dt):
    shape, needs_name, affine, layout = case
    rows, C, n_k, n_v = PV.BWD_SHAPES[shape]
    pl = PV.check_bwd_shape(shape)
    needs = PV.NEEDS_SUBSETS[needs_name]
    if not affine:
        needs = (needs[0], needs[1], needs[2], False, False)
    dtype = DT[dt]
    n = n_k + n_v
    g = torch.Generator(device=DEV).manual_seed(rows + C)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=g)
    x = (rnd(rows, C) * 1.3 + 3.0).to(dtype)
    gamma = (torch.rand(C, device=DEV, generator=g) + 0.5).to(dtype) if affine else None
    beta = (rnd(C) * 0.5).to(dtype) if affine else None
    w = (rnd(n, C) / C ** 0.5).to(dtype)
    G = rnd(rows, n).to(dtype)
    ops = _ops()
    st = ops.ln_stats(x, 1e-5)
    from perceiver_io_b200 import _lib
    l0 = _lib.launch_count()
    got = _bwd_run(x, st, w, gamma, beta, G, n_k, n_v, needs, layout)
    assert _lib.launch_count() - l0 == len(PV.bwd_kernels(needs)), "launched kernels"
    assert all((o is None) != bool(nd) for o, nd in zip(got, needs))
    ref = _bwd_ref(x, gamma, beta, w, G, 1e-5)
    mags, rstd = lnlin_magnitudes(x, st, w, gamma, beta, G)
    bounds = lnlin_element_bounds(mags, rstd, dtype, rows, C, n, pl["splits"], pl["m_blocks"])
    what = f"{case} {dt} splits={pl['splits']} kernels={sorted(PV.bwd_kernels(needs))}"
    assert_lnlin_elements(got, ref, bounds, ("dx", "dW", "db", "dgamma", "dbeta"), what)
    # the whole-tensor derived gate beside it, as test_gpu_ln_linear_bwd states it (eager: 16-bit autograd)
    leaves = [t.detach().clone().requires_grad_() if t is not None else None for t in (x, w, gamma, beta)]
    out = F.linear(F.layer_norm(leaves[0], (C,), leaves[2], leaves[3], 1e-5), leaves[1])
    out.backward(G)
    eager = [leaves[0].grad, leaves[1].grad, G.float().sum(0).to(dtype),
             None if leaves[2] is None else leaves[2].grad, None if leaves[3] is None else leaves[3].grad]
    for name, gv_, r, e in zip(("dx", "dW", "db", "dgamma", "dbeta"), got, ref, eager):
        if gv_ is None:
            continue
        bound = derived_bound(r, e)[0]
        err = (gv_.double() - r).abs().max().item()
        assert err <= bound, f"{what} {name}: whole-tensor err {err:.3e} > {bound:.3e}"
    again = _bwd_run(x, st, w, gamma, beta, G, n_k, n_v, needs, layout)
    for a, b_ in zip(got, again):
        if a is not None:
            _bits(a, b_, what + " determinism")


@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("shape", [(1, 64, 64, 8), (300, 64, 64, 0), (637, 256, 128, 64), (4000, 128, 64, 64),
                                   (9000, 128, 0, 64)], ids=lambda s: "x".join(map(str, s)))
def test_backward_probe_is_exact(shape, dt):
    rows, C, n_k, n_v = shape
    dtype = DT[dt]
    x, gamma, beta, w, G, mu, k = PV.bwd_probe(rows, C, n_k + n_v, seed=rows, dtype=dtype)
    ops = _ops()
    xd = x.to(DEV)
    st = ops.ln_stats(xd, 0.0)
    assert torch.equal(st[:, 1].cpu().double(), 2.0 ** -k)
    got = _bwd_run(xd, st, w.to(DEV), gamma.to(DEV), beta.to(DEV), G.to(DEV), n_k, n_v, PV.ALL_NEEDS)
    ref = _bwd_probe_ref(x, mu, k, gamma, beta, w, G)
    for name, g_, r in zip(("dx", "dW", "db", "dgamma", "dbeta"), got, ref):
        _bits(g_, r.to(dtype), f"backward probe {shape} {dt} {name}")


# ---- LayerNorm with eps = 0 and constant rows ----
@pytest.mark.parametrize("stats", ["fused", "separate"])
def test_eps_zero_is_layernorm(stats):
    """eps = 0 is a legal LayerNorm; the in-kernel statistics only run for eps > 0, so it must still normalise."""
    ops = _ops()
    dtype = torch.bfloat16
    rows, C, n = 300, 256, 128
    x, gamma, beta, w, b = _random_case(rows, C, n, dtype, seed=11, mean=1.0)
    w_cat, col_st = ops.fold_ln_linear(gamma, beta, [w], [b], dtype)
    k, _ = ops.kv_project(x, w_cat, col_st, n, 0, eps=0.0, stats=stats)
    ref, e32 = proj_reference(x, w_cat, col_st, 0.0)
    assert_proj_elements(k, ref, e32, dtype, f"eps=0 kv_project {stats}")
    old = ops.kv_project_config["stats"]
    ops.kv_project_config["stats"] = stats
    try:
        k8, _ = ops.kv_project_fp8(x.view(1, rows, C), w_cat, col_st, torch.full((n,), 16.0, device=DEV), n, 0, 1,
                                   eps=0.0)
    finally:
        ops.kv_project_config["stats"] = old
    assert_e4m3_codes(k8.view(rows, n), ref, e32, torch.full((n,), 16.0, device=DEV), f"eps=0 kv_project_fp8 {stats}")


@pytest.mark.parametrize("dt", PV.DTYPES)
@pytest.mark.parametrize("C", [256 * k for k in range(1, 9)] + [200])
@pytest.mark.parametrize("stats", ["fused", "separate"])
def test_constant_rows_write_the_folded_bias(stats, C, dt):
    """A zero-variance row normalises to 0, so LayerNorm -> Linear gives t = W beta + b: the output must be t within its
    one rounding (rows mixed with random ones, |mu| in {0, 1, 48, 1000}), for both statistics modes and e4m3.  C runs
    over every register width of ln_stats_reg_kernel (NCH 1..8) and one width of the generic kernel: the separate
    statistics reach the producer's zero-variance rule only when their mean of a constant row is exact."""
    ops = _ops()
    dtype = DT[dt]
    rows, n = 256, 512
    x, gamma, beta, w, b = _random_case(rows, C, n, dtype, seed=C)
    consts = torch.tensor([0.0, 1.0, 48.0, 1000.0, -48.0, -1000.0], device=DEV)
    cr = torch.arange(0, rows, 5, device=DEV)
    x[cr] = consts[torch.arange(cr.numel(), device=DEV) % consts.numel()].to(dtype)[:, None]
    w_cat, col_st = ops.fold_ln_linear(gamma, beta, [w], [b], dtype)
    t = w.double() @ beta.double() + b.double()
    got = torch.cat([o for o in ops.kv_project(x, w_cat, col_st, n // 2, n // 2, stats=stats) if o is not None], 1)
    err = (got[cr].double() - t).abs()
    ratio = (err / (UNIT_ROUNDOFF[dtype] * t.abs() + 2.0 ** -24)).max().item()
    print(f"[constant rows] {stats} C={C} {dt}: max err {err.max().item():.3e}, err / (u |t|) {ratio:.2f}")
    assert ratio <= 1.0
    ref, e32 = proj_reference(x, w_cat, col_st, 1e-5, fuse=stats == "fused")
    live = torch.ones(rows, dtype=torch.bool, device=DEV)
    live[cr] = False
    assert_proj_elements(got[live], ref[live], e32[live], dtype, f"constant-row case, other rows ({stats})")
    inv = torch.full((n,), 16.0, device=DEV)
    old = ops.kv_project_config["stats"]
    ops.kv_project_config["stats"] = stats
    try:
        k8, _ = ops.kv_project_fp8(x.view(1, rows, C), w_cat, col_st, inv, n, 0, 1)
    finally:
        ops.kv_project_config["stats"] = old
    # the e4m3 epilogue writes RN(t * inv) of the kernel's own fp32 t exactly
    want = (col_st[:, 1] * 16).to(torch.float8_e4m3fn).view(torch.uint8)
    assert torch.equal(k8.view(rows, n)[cr].view(torch.uint8), want.expand(cr.numel(), n)), "e4m3 constant rows"


# ---- the binary: every restated instantiation is launched ----
def test_profiler_sees_every_instantiation():
    import re

    from torch.profiler import ProfilerActivity, profile

    ops = _ops()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for dt in PV.DTYPES:
            dtype = DT[dt]
            x, gamma, beta, w, b = _random_case(200, 256, 192, dtype, seed=1)
            w_cat, col_st = ops.fold_ln_linear(gamma, beta, [w], [b], dtype)
            for mode in MODES:
                for cg in (1, 2):
                    _project(x, w_cat, col_st, 128, 64, mode, cg)
                old = ops.kv_project_config["stats"]
                ops.kv_project_config["stats"] = "fused" if mode == "fused" else "separate"
                try:
                    ops.kv_project_fp8(x.view(1, 200, 256), w_cat, col_st, torch.ones(192, device=DEV), 128, 64, 1,
                                       eps=None if mode == "none" else 1e-5)
                finally:
                    ops.kv_project_config["stats"] = old
            for rows, C, stride, off in PV.STATS_SHAPES.values():
                buf = torch.randn(min(rows, 64) * stride + off + 8, device=DEV).to(dtype)
                ops.ln_stats(buf[off:off + min(rows, 64) * stride].view(-1, stride)[:, :C], 1e-5)
            st = ops.ln_stats(x, 1e-5)
            G = torch.randn(200, 192, device=DEV).to(dtype)
            for needs in PV.NEEDS_SUBSETS.values():
                ops.ln_linear_backward(x, st, w, gamma, beta, G[:, :128], G[:, 128:], 128, 64, needs)
        torch.cuda.synchronize()
    seen = set()
    tname = {"__nv_bfloat16": PV.BF16, "__half": PV.FP16, "true": PV.BF16, "false": PV.FP16}
    for ev in prof.key_averages():
        m = re.search(r"(kvproj_fp8_kernel|kvproj_kernel|ln_stats_reg_kernel|ln_stats_kernel|lnlin_\w+?_kernel)<([^>]*)>",
                      ev.key)
        if not m:
            continue
        name, args = m[1][: -len("_kernel")], [a.strip() for a in m[2].split(",")]
        dt = tname[args[0]]
        if name == "kvproj":
            seen.add((name, dt, args[1] == "true", int(args[2])))
        elif name == "kvproj_fp8":
            seen.add((name, dt, args[1] == "true"))
        elif name == "ln_stats_reg":
            seen.add((name, dt, int(args[1])))
        else:
            seen.add((name, dt))
    want = PV.all_instantiations()
    print(f"[proj variants] profiler saw {len(seen & want)} of {len(want)} instantiations")
    assert seen == want, (sorted(want - seen, key=str), sorted(seen - want, key=str))


# ---- the module-level xfail, with gamma = 1 ----
def test_perceiver_encoder_training_route_with_unit_gamma(route):
    """The encoder case of test_gpu_ln_linear_bwd with every LayerNorm weight 1: round(gamma W) = W, so the fold adds no
    rounding.  Strict: the routed gradients must pass the derived gate of the fp64 model.

    This test records an open problem; it does not guard a fix.  On one H100 this seed passes at 0.98 of the gate
    (the self-attention k_proj gradients at 1.95 x eager's error), where the random-gamma case of the xfail reaches 1.06
    (2.12 x).  So the fold's rounding explains little of the excess, and its cause is not known.  The margin is 2 %: the
    test fails if the routed gradients drift further from fp64, and it would also fail if the eager yardstick's cuBLAS
    algorithms changed.  A failure here means the excess grew, not that the fold explanation was confirmed."""
    import test_gpu_ln_linear_bwd as T

    enc, x, go = T._small_encoder()
    with torch.no_grad():
        for m in enc.modules():
            if isinstance(m, torch.nn.LayerNorm):
                m.weight.fill_(1.0)
    T._check_module(enc, [x], go, route, ["_pcv_q_fold", "_pcv_kv_fold", "_pcv_qkv_fold", "_pcv_qkv_fold"])
