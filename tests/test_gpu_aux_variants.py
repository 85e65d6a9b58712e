"""-m gpu: every rotary, KV-append and pad-packing kernel of csrc/pcv_aux.cu at its instantiation, alignment,
grid-stride and device-row edges.  The rules, the case matrix and the oracles live in aux_variants.py;
test_aux_variants_cpu.py checks that the matrix reaches all 17 instantiations and both append paths, that the large
cases pass more than one grid sweep, and that the gates reject mutants of the rules.

- rotary: within half an output ulp of the fp64 rotation of the fp32 angles (plus the fp32 slack of sincosf and the
  products); pass-through channels are exact (e4m3 output: the exact requantisation); rows at angle 0 keep their values.
- append: bit for bit what torch.cat / indexed writes give (e4m3 arenas: the header's clamp-and-round expression).
- pack_pad: through the tensor-core forward and backward, with exact count probes.
Outputs live inside larger buffers filled with a byte pattern: every byte a launch must not write is checked unchanged,
so skipped rows, guard rows and padding columns are verified, and nothing is written outside the allocation even if a
row rule were wrong."""
import pytest
import torch

import aux_variants as AV
from aux_variants import APPEND_CASES, PACK_CASES, ROTARY_CASES

pytestmark = pytest.mark.gpu

DEV = "cuda"
F8 = torch.float8_e4m3fn
GUARD = 4          # rows before and after every output
PATTERN = 0x7B     # the byte every output buffer starts as


def _ops():
    from perceiver_io_b200 import ops
    return ops


def _lib():
    from perceiver_io_b200 import _lib
    return _lib


def _buffer(B, rows, width, dtype):
    """(B, GUARD + rows + GUARD, width) of `dtype`, every byte PATTERN."""
    es = torch.empty(0, dtype=dtype).element_size()
    return torch.full((B, 2 * GUARD + rows, width * es), PATTERN, dtype=torch.uint8, device=DEV).view(dtype)


def _bytes(t):
    return t.view(torch.uint8)


# ---- rotary ----
def _rotary_operands(c: AV.RotaryCase, seed):
    g = torch.Generator().manual_seed(seed)
    C = c.H * c.d
    xw = torch.randn(c.B, c.n, C + c.x_pad, generator=g) * 2
    descale = None
    if c.dt == AV.E4M3:
        codes = (xw * 40).clamp(-448, 448).to(F8)
        descale = torch.rand(c.H, generator=g) * 0.05 + 0.02
        x_full = codes
        x64 = (codes[..., :C].double().reshape(c.B, c.n, c.H, c.d) * descale.double()[:, None])
    else:
        x_full = xw.to(AV.TORCH_DTYPE[c.dt])
        x64 = x_full[..., :C].double().reshape(c.B, c.n, c.H, c.d)
    ang = AV.angle_table(1 if c.at else c.Ba, c.n_angles, max(c.rd, 2), seed)
    return x_full.to(DEV), x64.to(DEV), ang.to(DEV), descale


def _run_rotary(c: AV.RotaryCase, seed=0):
    """One launch of the case through the C entry points -> (output buffer, y view, x (the input tensor before the
    column slice), x64, angles, y_inv_scale or None, x_descale or None)."""
    ops, lib = _ops(), _lib()
    C = c.H * c.d
    x_full, x64, ang, descale = _rotary_operands(c, seed)
    x = x_full[..., :C]
    out_dt = F8 if c.fp8 else AV.TORCH_DTYPE[c.dt]
    buf = _buffer(c.B, c.out_rows, C + c.y_pad, out_dt)
    y = buf[:, GUARD:GUARD + c.out_rows, :C]
    angles = ang[0][None].contiguous() if c.at else ang
    code = {AV.BF16: lib.PCV_BF16, AV.FP16: lib.PCV_F16, AV.E4M3: lib.PCV_E4M3}[c.dt]
    p = ops._rotary_params(x, y, c.H, angles, c.right_align, code)
    p.rotate_dim = c.rd
    f, inv = None, None
    keep = []
    if c.fp8:
        amax = x64.abs().amax(dim=(0, 1, 3)).float().cpu()
        inv = (150.0 / amax).to(DEV)
        ds = descale.to(DEV) if descale is not None else None
        keep += [inv, ds]
        f = lib.RotaryFp8(x_descale=None if ds is None else ds.data_ptr(), y_inv_scale=inv.data_ptr())
    rows = None
    if c.at:
        b = torch.tensor([[r0, fl, 0] for r0, fl in c.bounds], dtype=torch.int32, device=DEV)
        b = b[0, :2].contiguous() if len(c.bounds) == 1 else b        # shared (1-D) or per row at row stride 3
        keep.append(b)
        rows = ops._dev_rows(b, c.capacity, c.B, 2, "rotary test")
    with torch.cuda.device(x.device):
        ops._launch_rotary(p, f, rows)
    torch.cuda.synchronize()
    return buf, y, x_full, x64, angles, inv, descale


def _written_mask(c: AV.RotaryCase, buf_shape, C):
    _, yrow, ok = c.rows()
    m = torch.zeros(buf_shape[:2], dtype=torch.bool)
    for b in range(c.B):
        for i in range(c.n):
            if ok[b][i]:
                m[b, GUARD + yrow[b][i]] = True
    return m


@pytest.mark.parametrize("c", ROTARY_CASES, ids=lambda c: c.name)
def test_rotary_matches_fp64(c):
    C = c.H * c.d
    buf, y, x_full, x64, angles, inv, descale = _run_rotary(c, seed=len(c.name))
    _, yrow, ok = c.rows()
    ok = torch.tensor(ok, device=DEV)
    yrow = torch.tensor(yrow, device=DEV).clamp(0, c.out_rows - 1)
    bi = torch.arange(c.B, device=DEV)[:, None].expand(-1, c.n)
    got = y[bi, yrow].reshape(c.B, c.n, c.H, c.d)           # (B, n, H, d): the output row of every input row
    A = AV.select_angles(c, angles[..., :c.rd])
    ref, mag = AV.rotate64(x64, A, c.rd)
    out_dt = AV.E4M3 if c.fp8 else c.dt
    scale = inv.double()[None, None, :, None] if c.fp8 else 1.0
    excess = AV.rotary_excess(got.float().double(), ref, mag, out_dt, scale)[ok]
    worst = excess.max().item() if excess.numel() else float("-inf")
    # pass-through channels: exact copies (e4m3: one fp32 product, or two for e4m3 input, rounded once)
    xv = x_full[..., :C].reshape(c.B, c.n, c.H, c.d)
    if c.fp8:
        if c.dt == AV.E4M3:
            want = AV.requant_rd0(xv.cpu(), descale, inv.cpu()).to(DEV)
        else:
            want = AV.e4m3_codes(xv, inv[None, None, :, None].expand_as(xv))
        same = _bytes(got[..., c.rd:])[ok] == _bytes(want[..., c.rd:].contiguous())[ok]
    else:
        same = _bytes(got[..., c.rd:].contiguous())[ok] == _bytes(xv[..., c.rd:].contiguous())[ok]
        want = xv
    assert same.all(), f"{c.name}: pass-through channels differ from the exact value"
    # rows at angle 0: the rotated channels keep their values.  Signed zeros may differ: y1 = x1 * 1 + x0 * 0 turns
    # x1 = -0 into +0 when x0 >= 0
    zero = (A[..., :c.rd] == 0).all(-1) & ok if c.rd else torch.zeros_like(ok)
    zero = zero.to(DEV)
    if zero.any():
        assert (got[..., :c.rd].float() == want[..., :c.rd].float())[zero].all(), f"{c.name}: angle-0 rows changed"
    # every byte outside the written rows and columns keeps its pattern
    written = _written_mask(c, buf.shape, C).to(DEV)
    raw = _bytes(buf)
    es = buf.element_size()
    assert (raw[~written] == PATTERN).all(), f"{c.name}: a skipped or guard row was written"
    assert (raw[written][:, C * es:] == PATTERN).all(), f"{c.name}: the row padding was written"
    print(f"[rotary] {c.name} ({'x'.join(map(str, c.instantiation[1:]))}, {c.work} pairs, {c.sweeps} sweeps): "
          f"worst excess over the half-ulp gate {worst:.3e}; {int(zero.sum())} angle-0 rows; "
          f"{int((~ok).sum())} rows skipped")
    assert worst <= 0, f"{c.name}: an element is more than half an ulp + slack from the fp64 rotation"


# ---- the rotary backward shim, end to end ----
@pytest.mark.parametrize("B,n,H,d,f,Ba,extra,ra", [(3, 37, 2, 9, 8, 3, 5, True), (2, 64, 4, 66, 32, 1, 0, False),
                                                   (2, 20, 1, 33, 32, 2, 7, True)])
def test_rotary_autograd_matches_fp64(B, n, H, d, f, Ba, extra, ra):
    ops = _ops()
    g = torch.Generator().manual_seed(n + d)
    angles = AV.angle_table(Ba, n + extra, f, seed=d)
    angles = torch.where(angles.abs() > 1e4, angles * 1e-6, angles).to(DEV)
    x = (torch.randn(B, n, H * d, generator=g)).bfloat16().to(DEV).requires_grad_()
    gy = torch.randn(B, n, H * d, generator=g).bfloat16().to(DEV)
    y = ops.rotary(x, H, angles, ra)
    y.backward(gy)
    x64 = x.detach().double().requires_grad_()
    y64 = AV.rotary_autograd64(x64, angles, H, ra)
    y64.backward(gy.double())
    for name, got, ref, mag in (("y", y.detach(), y64.detach(), x64.detach().abs()),
                                ("grad", x.grad, x64.grad, gy.double().abs())):
        m = mag.reshape(B, n, H, d)
        m2 = m.clone()
        m2[..., :f] = (m[..., 0:f:2] + m[..., 1:f:2]).repeat_interleave(2, -1)
        ex = AV.rotary_excess(got.double(), ref, m2.reshape(B, n, -1), AV.BF16)
        print(f"[rotary autograd] B{B} n{n} H{H} d{d} f{f} Ba{Ba} {name}: worst excess {ex.max().item():.3e}")
        assert ex.max().item() <= 0, name


# ---- kv_append ----
def _append_operands(c: AV.AppendCase, seed):
    g = torch.Generator().manual_seed(seed)
    dt = AV.TORCH_DTYPE[c.dt]
    ddt = F8 if c.fp8 else dt
    view = lambda t, C: t[..., c.shift:c.shift + C]   # noqa: E731
    new = [view(torch.randn(c.B, c.n, C + c.pad, generator=g).to(dt).to(DEV), C) for C in (c.Ck, c.Cv)]
    caches = [view((torch.randn(c.B, c.L_old, C + c.pad, generator=g) * 20).to(ddt).to(DEV), C) if c.L_old else None
              for C in (c.Ck, c.Cv)]
    bufs = [_buffer(c.B, c.dst_rows, C + c.pad, ddt) for C in (c.Ck, c.Cv)]
    noise = [torch.randint(0, 256, b.view(torch.uint8).shape, generator=g, dtype=torch.uint8) for b in bufs]
    for b, z in zip(bufs, noise):
        b.view(torch.uint8)[:, GUARD:GUARD + c.dst_rows] = z[:, GUARD:GUARD + c.dst_rows].to(DEV)
    dsts = [view(b[:, GUARD:GUARD + c.dst_rows], C) for b, C in zip(bufs, (c.Ck, c.Cv))]
    if c.alias_k:   # a cache view at k_dst's pointer with a dense cache's batch stride: the launch skips it
        row = c.Ck + c.pad
        caches[0] = torch.as_strided(bufs[0], (c.B, c.L_old, c.Ck), (c.L_old * row, row, 1), dsts[0].storage_offset())
    inv = [None, None]
    if c.fp8:
        ch = torch.arange(c.Ck)
        inv[0] = torch.exp2(((ch * 5) % 7 - 2).float()).to(DEV)               # powers of two, 7 values per vector
        inv[1] = (torch.rand(c.Cv, generator=g) * 40 + 0.5).to(DEV)
        probes = _fp8_probes(c.dt)
        k0 = (probes[ch % len(probes)] / inv[0].cpu()).to(dt)
        assert torch.equal(k0.double() * inv[0].cpu().double(), probes[ch % len(probes)])   # exact in dt
        new[0][:, 0] = k0.to(DEV)
    return new, caches, bufs, dsts, inv


def _fp8_probes(dt):
    """e4m3 values after scaling: ties between adjacent codes (normal and subnormal), codes, subnormals, signed zeros,
    values on both sides of the saturation boundary 464 and +-inf (-> +-448 under satfinite)."""
    s = 2.0 ** -9
    v = [1.0625, -1.1875, 17.0, 208.0, -432.0, s, 1.5 * s, 0.5 * s, 0.25 * s, 2.5 * s, -3.5 * s, 0.0, -0.0, 448.0,
         462.0, 464.0, 466.0, -466.0, 12288.0, float("inf"), float("-inf"), 2.0 ** -6 + 2.0 ** -10, 3.0]
    if dt == AV.FP16:
        v += [447.0, 449.0, 463.5, 464.5]
    return torch.tensor(v, dtype=torch.float64)


def _run_append(c: AV.AppendCase, new, caches, dsts, inv):
    ops = _ops()
    rows = None
    keep = None
    if c.at:
        keep = torch.tensor([[r, 0] for r in c.bounds], dtype=torch.int32, device=DEV)
        keep = keep[0, :1].contiguous() if len(c.bounds) == 1 else keep              # per row at row stride 2
        rows = ops._dev_rows(keep, c.capacity, c.B, 1, "append test")
    ops._launch_kv_append(caches[0], caches[1], new[0], new[1], dsts[0], dsts[1], False, False,
                          (inv[0], inv[1]) if c.fp8 else None, rows)
    torch.cuda.synchronize()


@pytest.mark.parametrize("c", APPEND_CASES, ids=lambda c: c.name)
def test_kv_append_is_bit_exact(c):
    new, caches, bufs, dsts, inv = _append_operands(c, seed=len(c.name) + c.n)
    before = [b.clone() for b in bufs]
    cache_vals = [None if t is None else t.clone() for t in caches]
    _run_append(c, new, caches, dsts, inv)
    want_bufs = [b.clone() for b in before]
    want_dst = [w[:, GUARD:GUARD + c.dst_rows, c.shift:c.shift + C] for w, C in zip(want_bufs, (c.Ck, c.Cv))]
    res = AV.append_oracle(c, want_dst, *cache_vals, *new, *inv)
    for w, r in zip(want_dst, res):
        w.copy_(r)
    for half, (got, want) in enumerate(zip(bufs, want_bufs)):
        diff = (_bytes(got) != _bytes(want))
        assert not diff.any(), (f"{c.name}: {'KV'[half]} differs from the oracle at {int(diff.sum())} bytes, first "
                                f"{diff.nonzero()[0].tolist()}")
    print(f"[append] {c.name} ({c.instantiation}, paths {sorted(c.paths)}, {c.blocks} blocks, {c.sweeps} sweeps): "
          f"bit-exact, guards and padding untouched")


# ---- pack_pad, through the tensor-core attention ----
@pytest.mark.parametrize("c", PACK_CASES, ids=lambda c: c.name)
def test_pad_bits_count_probe(c):
    """q = 0 and v_j = e_(j mod dv): every live score is 0, so l is the count of unpadded keys and part_o[..., c] the
    count of unpadded keys = c (mod dv), integers below 2^24 and exact in fp32; a fully padded row takes the finite
    fill (m = -FLT_MAX, l = M, o the counts of all keys)."""
    ops = _ops()
    H, d, N = 1, c.dv, 3
    pad = AV.probe_mask(c.B, c.M, seed=c.M, device=DEV, stride_pad=c.stride_pad)
    assert pad.stride(0) == c.M + c.stride_pad
    q = torch.zeros(1, N, H * d, dtype=torch.bfloat16, device=DEV)
    k = torch.randn(c.B, c.M, H * d, dtype=torch.bfloat16, device=DEV)
    j = torch.arange(c.M, device=DEV)
    v = torch.nn.functional.one_hot(j % c.dv, c.dv).to(torch.bfloat16)[None].expand(c.B, -1, -1).contiguous()
    po, pm, pl = ops.attention_partial(q, k, v, H, 0.125, pad_mask=pad, impl="tcgen05")
    o, m, l = AV.count_expect(pad, c.dv)
    B = c.B
    assert torch.equal(pl.double(), l[:, None, None].expand(B, H, N)), f"{c.name}: l is not the unpadded key count"
    assert torch.equal(pm.double(), m[:, None, None].expand(B, H, N)), f"{c.name}: m"
    assert torch.equal(po.double(), o[:, None, None, :].expand(B, H, N, c.dv)), f"{c.name}: per-residue counts"
    print(f"[pack_pad] {c.name}: B{B} M{c.M} stride_b {pad.stride(0)}, {c.words} words, {c.sweeps} sweeps: counts "
          f"exact, {int((~(~pad).any(-1)).sum())} fully padded rows")


@pytest.mark.parametrize("M", AV.PACK_BWD_MS)
def test_pad_bits_in_the_backward(M):
    """The backward's pad bits at the word edges: grad_k and grad_v of padded keys are exactly zero, those of unpadded
    keys are not, in every batch row with a live key (a fully padded row takes the finite fill instead)."""
    ops = _ops()
    B, H, N, d = 3, 2, 40, 32
    g = torch.Generator().manual_seed(M)
    q, k, v, go = ((torch.randn(B, L, H * d, generator=g)).bfloat16().to(DEV) for L in (N, M, M, N))
    pad = AV.probe_mask(B, M, seed=M + 1, device=DEV)
    scale = d ** -0.5
    po, pm, pl = ops.attention_partial(q, k, v, H, scale, pad_mask=pad, impl="tcgen05")
    out = ops.combine_partials(po[None], pm[None], pl[None], q.dtype)
    _, gk, gv = ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, pad_mask=pad)
    live_rows = (~pad).any(-1)
    for b in range(B):
        if not live_rows[b]:
            continue
        pb = pad[b]
        assert (gk[b][pb] == 0).all() and (gv[b][pb] == 0).all(), f"M{M} b{b}: a padded key has a gradient"
        assert (gk[b][~pb] != 0).any(-1).all() and (gv[b][~pb] != 0).any(-1).all(), f"M{M} b{b}: a live key has none"
    print(f"[pack_pad bwd] M{M}: padded keys {int(pad[live_rows].sum())} with zero gradients, live keys "
          f"{int((~pad).sum())} with nonzero ones")
