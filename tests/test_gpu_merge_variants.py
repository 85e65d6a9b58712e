"""-m gpu: every instantiation of the CUDA-core attention kernel (csrc/pcv_attn_simt.cu) and of the partial-state merge
kernels (csrc/pcv_aux.cu: combine_kernel, combine_peers_kernel, rescale_kernel) at its split, tile, alignment and
finite-fill edges.  The rules, the matrix and the probes live in merge_variants.py; test_merge_variants_cpu.py checks
that the matrix reaches every (dtype, DVW, mode), that the restated plan is the library's, that the probes are exact
in fp32 and that they reject mutants of the rules.

Count, needle and dyadic probes must equal their exact expectations bit for bit; random operands go through the
element-wise gates (gpu_util.decode_element_bound for the SIMT kernel, merge_variants.merge_element_bound for the
merges) beside the whole-tensor derived gate."""
import ctypes as C
import zlib

import pytest
import torch

import merge_variants as MV
from gpu_util import assert_decode_elements, assert_partial_state
from merge_variants import SIMT_CASES, case_id

pytestmark = pytest.mark.gpu

DEV = "cuda"
DT = MV.TORCH_DTYPE


def _ops():
    from perceiver_io_b200 import ops
    return ops


def _lib():
    from perceiver_io_b200 import _lib
    return _lib


def _rows(t, strided):
    """t (B, L, C) on the device, as a slice of (B, L, C + 3) rows when `strided`."""
    t = t.to(DEV)
    if not strided:
        return t.contiguous()
    buf = torch.zeros(t.shape[0], t.shape[1], t.shape[2] + 3, dtype=t.dtype, device=DEV)
    buf[..., :t.shape[2]] = t
    return buf[..., :t.shape[2]]


def _run(c, q, k, v, scale):
    ops = _ops()
    pad = MV.pad_mask(c)
    q, k, v = (_rows(t, c.strided) for t in (q, k, v))
    pad = None if pad is None else pad.to(DEV)
    if c.partial:
        return tuple(t.cpu() for t in ops.attention_partial(q, k, v, c.H, scale, pad_mask=pad, causal=c.causal,
                                                            m_total=c.m_total, m_offset=c.m_offset, impl="simt"))
    return ops.attention(q, k, v, c.H, scale, pad_mask=pad, causal=c.causal, impl="simt").cpu()


def _bits(got, want, what):
    got, want = got.cpu(), want.cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype in (torch.bfloat16, torch.float16):
        g16, w16 = got.view(torch.int16), want.view(torch.int16)
        bad = (g16 != w16).nonzero()
    else:
        bad = (got != want).nonzero()
    assert bad.shape[0] == 0, (f"{what}: {bad.shape[0]} of {got.numel()} elements differ; first at {bad[0].tolist()}: "
                               f"got {got[tuple(bad[0])].item()} want {want[tuple(bad[0])].item()}")


# ---- exp2f of an integer is exact on the device: the probes below rest on it ----
def test_exp2f_of_integers_is_exact():
    """rescale_partial_ with o = 1, l = 1, m = k, new_m = 0 stores exp2f(k) for every integer k in [-149, 0].  Exact on
    the normal range [-126, 0], where every probe of this file keeps its weights (merge_variants.MIN_PROBE_EXP); the
    subnormal results are reported, not gated (on an H100, exp2f(-127) was the one inexact value of the 150)."""
    ops = _ops()
    ks = torch.arange(-149, 1, dtype=torch.float32)
    po = torch.ones(ks.numel(), 1, device=DEV)
    pm, pl = ks.to(DEV).clone(), torch.ones(ks.numel(), device=DEV)
    ops.rescale_partial_(po, pm, pl, torch.zeros_like(pm))
    got = po[:, 0].cpu()
    want = torch.tensor([2.0 ** int(k) for k in ks], dtype=torch.float64).float()
    bad = [(int(k), a.item()) for k, a, b in zip(ks, got, want) if a.item() != b.item()]
    print(f"[exp2f] exact for {ks.numel() - len(bad)} of {ks.numel()} integers in [-149, 0]; inexact: "
          + ", ".join(f"exp2f({k}) = {a!r} (2^{k} = {2.0 ** k!r})" for k, a in bad))
    normal = ks >= -126
    assert torch.equal(got[normal], want[normal]) and torch.equal(pl.cpu(), got) and (pm == 0).all()
    assert all(k < MV.MIN_PROBE_EXP for k, _ in bad)


# ---- the SIMT kernel, every (dtype, DVW, mode) ----
@pytest.mark.parametrize("c", SIMT_CASES, ids=case_id)
def test_simt_count_probe(c):
    q, k, v = MV.count_operands(c)
    in_range, live = MV.sets_of(c)
    got = _run(c, q, k, v, 0.25)
    if c.partial:
        for name, g, w in zip("oml", got, MV.count_partial_expect(v, c.H, in_range, live)):
            _bits(g, w, f"count {case_id(c)} {name}")
    else:
        _bits(got, MV.simt_count_expect(v, c.H, in_range, live, DT[c.dt]), f"count {case_id(c)}")


@pytest.mark.parametrize("c", SIMT_CASES, ids=case_id)
def test_simt_needle_probe(c):
    in_range, live = MV.sets_of(c)
    for r in range(MV.needle_rounds(c)):
        nd = MV.needle_set(c, r)
        q, k, v = MV.needle_operands(c, nd, seed=r)
        got = _run(c, q, k, v, MV.NEEDLE_SCALE)
        if not c.partial:
            _bits(got, MV.simt_needle_expect(c, v, in_range, live, nd), f"needle {case_id(c)} round {r}")
            continue
        o, m, l = MV.count_partial_expect(v, c.H, in_range, live)
        found = MV.needle_found(c, live, nd)                                     # (B, H, N)
        bi, hi = torch.arange(c.B)[:, None, None], torch.arange(c.H)[None, :, None]
        vn = v.float().reshape(c.B, c.M, c.H, -1)[bi, nd, hi]                   # (B, H, N, dv)
        o = torch.where(found[..., None], vn, o)
        m = torch.where(found, torch.full_like(m, MV.needle_score()), m)
        l = torch.where(found, torch.ones_like(l), l)
        for name, g, w in zip("oml", got, (o, m, l)):
            _bits(g, w, f"needle {case_id(c)} round {r} {name}")


@pytest.mark.parametrize("c", SIMT_CASES, ids=case_id)
def test_simt_random_operands(c):
    g = torch.Generator().manual_seed(zlib.crc32(case_id(c).encode()))
    dtype = DT[c.dt]
    q = torch.randn(c.Bq, c.N, c.H * c.dqk, generator=g).to(dtype)
    k = torch.randn(c.B, c.M, c.H * c.dqk, generator=g).to(dtype)
    v = torch.randn(c.B, c.M, c.H * c.dv, generator=g).to(dtype)
    scale = c.dqk ** -0.5
    got = _run(c, q, k, v, scale)
    pad = MV.pad_mask(c)
    if c.partial:
        assert_partial_state(tuple(t.to(DEV) for t in got), q.to(DEV), k.to(DEV), v.to(DEV), c.H, scale,
                             None if pad is None else pad.to(DEV), c.causal, c.m_total, c.m_offset, what=case_id(c))
    else:
        assert_decode_elements(got.to(DEV), q.to(DEV), k.to(DEV), v.to(DEV), c.H, scale,
                               None if pad is None else pad.to(DEV), c.causal, dtype, MV.serial_depth(c.plan),
                               what=case_id(c))


SHARDINGS = [   # (dt, B, H, N, m_total, dqk, dv, causal, shard edges): causal shards in the rows' future, N > m_total
    ("bf16", 2, 2, 300, 400, 40, 24, True, (0, 128, 256, 384, 400)),
    ("fp16", 2, 3, 33, 700, 64, 130, True, (0, 256, 512, 700)),
    ("bf16", 1, 2, 40, 33, 17, 64, False, (0, 16, 33)),
    ("fp16", 2, 1, 65, 70, 9, 7, True, (0, 5, 6, 70)),
]


@pytest.mark.parametrize("sh", SHARDINGS, ids=lambda s: f"{s[0]}-N{s[3]}-M{s[4]}-{len(s[8]) - 1}shards")
def test_simt_key_shards_merge_to_the_single_pass(sh):
    """attention_partial on each key shard (m_offset / m_total), merged by combine_partials: bitwise the single pass on
    the count probe, every shard's partial state within assert_partial_state, and the merged random output within the
    element-wise gate."""
    ops = _ops()
    dt, B, H, N, M, dqk, dv, causal, edges = sh
    dtype = DT[dt]
    c = MV.SimtCase(dt, B, B, H, N, M, dqk, dv, causal, True, False, M, 0, False)
    pad = MV.pad_mask(c).to(DEV)
    in_range, live = MV.sets_of(c)
    g = torch.Generator().manual_seed(N)
    count = MV.count_operands(c)
    rand = (torch.randn(B, N, H * dqk, generator=g).to(dtype), torch.randn(B, M, H * dqk, generator=g).to(dtype),
            torch.randn(B, M, H * dv, generator=g).to(dtype))
    for name, (q, k, v) in (("count", count), ("random", rand)):
        q, k, v = q.to(DEV), k.to(DEV), v.to(DEV)
        scale = 0.25 if name == "count" else dqk ** -0.5
        parts, depth = [], 0
        for a, b in zip(edges[:-1], edges[1:]):
            part = ops.attention_partial(q, k[:, a:b], v[:, a:b], H, scale, pad_mask=pad[:, a:b].contiguous(), causal=causal,
                                         m_total=M, m_offset=a, impl="simt")
            dead = assert_partial_state(part, q, k[:, a:b], v[:, a:b], H, scale, pad[:, a:b], causal, M, a,
                                        what=f"{name} shard [{a}, {b})")
            parts.append(part)
            depth = max(depth, MV.serial_depth(MV.simt_plan(B, H, N, b - a, dqk, dv)))
            print(f"[shards] {name} [{a}, {b}): {dead} rows without a live key")
        merged = ops.combine_partials(*(torch.stack([p[i] for p in parts]) for i in range(3)), out_dtype=dtype)
        single = ops.attention(q, k, v, H, scale, pad_mask=pad, causal=causal, impl="simt")
        if name == "count":
            want = MV.simt_count_expect(count[2], H, in_range, live, dtype)
            _bits(merged, want, "count shards merged")
            _bits(single, want, "count single pass")
        else:
            assert_decode_elements(merged, q, k, v, H, scale, pad, causal, dtype, depth + len(parts), what="merged")


def test_simt_grid_above_65535_heads():
    """B*H = 65536 (and a 2-tile query axis): the (b, h) index shares gridDim.x with the query tile, so it is not bound
    by gridDim.y's 65535.  The count probe on two keys: every row is RN16((v0 + v1) / 2)."""
    ops = _ops()
    B, H, N, M = 32768, 2, 33, 2
    for dtype in (torch.bfloat16, torch.float16):
        q = torch.zeros(1, N, H, device=DEV, dtype=dtype)
        k = torch.randn(B, M, H, device=DEV).to(dtype)
        v = torch.randint(-64, 65, (B, M, H), device=DEV).to(dtype)
        out = ops.attention(q, k, v, H, 0.5, impl="simt")
        want = ((v[:, 0].float() + v[:, 1].float()) * 0.5).to(dtype)[:, None, :].expand(B, N, H)
        _bits(out, want, f"B*H = {B * H} {dtype}")


def test_auto_routes_uncovered_calls_to_simt():
    """`auto` takes the SIMT kernel for dqk in 513..1024 and for scale <= 0 (the tensor-core kernel refuses both, the
    decode kernel takes neither N = 33 nor M = 300): the same bits as impl = "simt"."""
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    for dqk, scale in ((513, 0.04), (1024, 0.03), (64, -0.125), (64, 0.0)):
        q = torch.randn(2, 33, 2 * dqk, generator=g).bfloat16().to(DEV)
        k = torch.randn(2, 300, 2 * dqk, generator=g).bfloat16().to(DEV)
        v = torch.randn(2, 300, 2 * 64, generator=g).bfloat16().to(DEV)
        _bits(ops.attention(q, k, v, 2, scale), ops.attention(q, k, v, 2, scale, impl="simt"), f"auto dqk={dqk} s={scale}")


# ---- combine_partials, merge_partials, rescale_partial_ ----
GS = (1, 2, 3, 8, 37)
MERGE_DVS = (1, 3, 4, 128, 132, 512)


def _states(G, B, H, N, dv, seed, fn=MV.dyadic_states):
    po, pm, pl = fn(G, B * H * N, dv, seed)
    return (po.reshape(G, B, H, N, dv).to(DEV), pm.reshape(G, B, H, N).to(DEV), pl.reshape(G, B, H, N).to(DEV))


@pytest.mark.parametrize("G", GS)
@pytest.mark.parametrize("dv", MERGE_DVS)
def test_merges_on_dyadic_states(G, dv):
    """combine_partials (bf16 and fp16) is RN16 of the fp64 merge bit for bit, merge_partials the fp64 (o, m, l) bit for
    bit, on rows that are live, all filled, filled + live, filled + -inf and live + -inf."""
    ops = _ops()
    B, H, N = 2, 3, 11
    po, pm, pl = _states(G, B, H, N, dv, seed=G * 1000 + dv)
    acc, m, l = MV.merge_reference(po.cpu(), pm.cpu(), pl.cpu())
    for dtype in (torch.bfloat16, torch.float16):
        out = ops.combine_partials(po, pm, pl, out_dtype=dtype)
        want = (acc / l[..., None]).to(dtype).transpose(1, 2).reshape(B, N, H * dv)
        _bits(out, want, f"combine G={G} dv={dv} {dtype}")
    mo, mm, ml = ops.merge_partials(po, pm, pl)
    for name, g, w in zip("oml", (mo, mm, ml), (acc, m, l)):
        _bits(g, w.float(), f"merge_partials G={G} dv={dv} {name}")


@pytest.mark.parametrize("dv", (3, 128, 132))
def test_combine_into_strided_outputs(dv):
    """pcv_attn_combine into the H*dv columns of a wider (B, N, W) buffer at a column offset: the columns are the
    dense call's bit for bit, every other element keeps its NaN."""
    lib, ops = _lib(), _ops()
    G, B, H, N = 5, 2, 3, 7
    po, pm, pl = _states(G, B, H, N, dv, seed=dv)
    for dtype in (torch.bfloat16, torch.float16):
        dense = ops.combine_partials(po, pm, pl, out_dtype=dtype)
        W, off = H * dv + 13, 5
        buf = torch.full((B, N, W), float("nan"), dtype=dtype, device=DEV)
        p = lib.CombineParams()
        p.part_o, p.part_m, p.part_l = po.data_ptr(), pm.data_ptr(), pl.data_ptr()
        p.out = buf.data_ptr() + off * buf.element_size()
        p.o_stride_b, p.o_stride_n, p.o_stride_h = N * W, W, dv
        p.num_parts, p.B, p.H, p.N, p.dv = G, B, H, N, dv
        p.dtype = ops._pcv_dtype(dtype)
        lib.check(lib.lib().pcv_attn_combine(C.byref(p), ops._stream()), "pcv_attn_combine")
        _bits(buf[..., off:off + H * dv], dense, f"strided combine dv={dv}")
        rest = torch.cat([buf[..., :off], buf[..., off + H * dv:]], -1)
        assert rest.isnan().all(), "combine wrote outside the output columns"


@pytest.mark.parametrize("G", (1, 3, 37))
@pytest.mark.parametrize("dv", (3, 128))
def test_merges_on_random_states(G, dv):
    ops = _ops()
    B, H, N = 2, 2, 13
    po, pm, pl = _states(G, B, H, N, dv, seed=7 * G + dv, fn=MV.random_states)
    for dtype in (torch.bfloat16, torch.float16):
        out = ops.combine_partials(po, pm, pl, out_dtype=dtype).cpu().double()
        bound, ref = MV.merge_element_bound(po.cpu(), pm.cpu(), pl.cpu(), dtype)
        ref = ref.transpose(1, 2).reshape(B, N, -1)
        bound = bound.transpose(1, 2).reshape(B, N, -1)
        ratio = ((out - ref).abs() / bound).max().item()
        print(f"[merge random] G={G} dv={dv} {dtype}: worst err / bound {ratio:.3f}")
        assert ratio <= 1.0
    mo, mm, ml = ops.merge_partials(po, pm, pl)
    acc, m, l = MV.merge_reference(po.cpu(), pm.cpu(), pl.cpu())
    assert torch.equal(mm.cpu().double(), m)
    assert ((ml.cpu().double() - l).abs() <= (G + 2) * 2.0 ** -21 * l).all()
    scale = (po.cpu().double().abs() * torch.exp2(pm.cpu().double() - m).nan_to_num(0.0)[..., None]).sum(0)
    assert ((mo.cpu().double() - acc).abs() <= (G + 2) * 2.0 ** -21 * scale + 1e-30).all()


@pytest.mark.parametrize("dv", (1, 3, 4, 128, 132, 512))
def test_rescale_on_dyadic_states(dv):
    """rescale_partial_ is exact on the dyadic states (w = 2^-e, 1 and 0), and the same on a part_o at an odd float
    offset (4-byte aligned: the element-wise path) as on an aligned copy."""
    ops = _ops()
    po, pm, pl, new_m = (t.to(DEV) for t in MV.rescale_states(203, dv, seed=dv))
    want = MV.rescale_emulate(po.cpu(), pm.cpu(), pl.cpu(), new_m.cpu())
    w = torch.where(pm.cpu().double() == float("-inf"), torch.zeros(()).double(),
                    torch.exp2(pm.cpu().double() - new_m.cpu().double()))
    assert torch.equal(want[0].double(), po.cpu().double() * w[:, None])
    a = [t.clone() for t in (po, pm, pl)]
    ops.rescale_partial_(*a, new_m)
    for name, g, x in zip("oml", a, want):
        _bits(g, x, f"rescale dv={dv} {name}")
    buf = torch.zeros(po.numel() + 1, device=DEV)
    mis = buf[1:].view(po.shape)
    mis.copy_(po)
    assert mis.data_ptr() % 16 == 4 and MV.rescale_vector(dv, mis.data_ptr()) is False
    b = [mis, pm.clone(), pl.clone()]
    ops.rescale_partial_(*b, new_m)
    for name, g, x in zip("oml", b, a):
        _bits(g, x, f"rescale dv={dv} misaligned part_o {name}")


# ---- combine_peers on one GPU: G local buffers stand for the ranks' mapped buffers ----
def _peer_call(po_list, pm_list, pl_list, outs, B, H, N, dv, dtype, rank, G, strides):
    lib, ops = _lib(), _ops()
    p = lib.PeerCombineParams()
    for g in range(G):
        p.part_o[g], p.part_m[g], p.part_l[g] = po_list[g].data_ptr(), pm_list[g].data_ptr(), pl_list[g].data_ptr()
        p.out[g] = outs[g].data_ptr()
    p.o_stride_b, p.o_stride_n, p.o_stride_h = strides
    p.row_begin, p.row_end = MV.peer_rows(B * H * N, G, rank)
    p.num_peers, p.rank = G, rank
    p.B, p.H, p.N, p.dv = B, H, N, dv
    p.dtype = ops._pcv_dtype(dtype)
    lib.check(lib.lib().pcv_attn_combine_peers(C.byref(p), ops._stream()), "pcv_attn_combine_peers")


def _offset_copy(t, elems):
    """t's values in a new buffer at `elems` elements past its start (4-byte aligned for fp32 at elems = 1)."""
    buf = torch.full((t.numel() + elems,), float("nan"), dtype=t.dtype, device=DEV)
    v = buf[elems:].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("G", (1, 2, 3, 8))
@pytest.mark.parametrize("dv", (3, 4, 128, 132))
def test_combine_peers_on_one_gpu(G, dv):
    """Called once per rank with dist.PeerMerger's row slices: every out[g] holds every row, equal to combine_partials
    bit for bit; a single rank's call leaves the other rows' NaN untouched.  dv in (4, 128) with aligned buffers takes
    the fast path, dv in (3, 132) and the misaligned buffers (part_o at an odd float, out at an odd element) the general
    path, with the same bits."""
    ops = _ops()
    B, H, N = 2, 3, 15
    strides = (N * H * dv, H * dv, dv)
    for dtype in (torch.bfloat16, torch.float16):
        po, pm, pl = _states(G, B, H, N, dv, seed=G * 31 + dv)
        want = ops.combine_partials(po, pm, pl, out_dtype=dtype)
        acc, _, l = MV.merge_reference(po.cpu(), pm.cpu(), pl.cpu())
        _bits(want, (acc / l[..., None]).to(dtype).transpose(1, 2).reshape(B, N, -1), "combine_partials")
        po_l = [po[g].contiguous() for g in range(G)]
        pm_l, pl_l = [pm[g].contiguous() for g in range(G)], [pl[g].contiguous() for g in range(G)]
        for layout in ("aligned", "misaligned"):
            if layout == "aligned":
                parts = po_l
                outs = [torch.full((B, N, H * dv), float("nan"), dtype=dtype, device=DEV) for _ in range(G)]
            else:
                parts = [_offset_copy(t, 1) for t in po_l]
                outs = [_offset_copy(torch.full((B, N, H * dv), float("nan"), dtype=dtype, device=DEV), 1)
                        for _ in range(G)]
            fast = MV.peers_fast_path(dv, strides, [t.data_ptr() for t in parts], [t.data_ptr() for t in outs])
            assert fast == (layout == "aligned" and dv in (4, 128)), (layout, dv, fast)
            # one rank's call first: only its rows are written, in every output
            _peer_call(parts, pm_l, pl_l, outs, B, H, N, dv, dtype, G - 1, G, strides)
            rb, re = MV.peer_rows(B * H * N, G, G - 1)
            rowmask = torch.zeros(B * H * N, dtype=torch.bool)
            rowmask[rb:re] = True
            rowmask = rowmask.view(B, H, N).transpose(1, 2).to(DEV)         # (B, N, H): the (b, h, n) row order
            for g in range(G):
                o = outs[g].view(B, N, H, dv)
                assert o[~rowmask].isnan().all(), f"{layout} G={G}: rows outside [{rb}, {re}) written into out[{g}]"
                _bits(o[rowmask], want.view(B, N, H, dv)[rowmask], f"{layout} G={G} rank {G - 1} out[{g}]")
            for rank in range(G - 1):
                _peer_call(parts, pm_l, pl_l, outs, B, H, N, dv, dtype, rank, G, strides)
            for g in range(G):
                _bits(outs[g], want, f"peers {layout} G={G} dv={dv} {dtype} out[{g}]")


# ---- the binary: every instantiation is launched ----
def test_profiler_sees_every_instantiation():
    """Every one of the 13 instantiations is launched: the attention calls run two splits (combine_kernel<T> too).
    The operands are built before the profiler starts. Inside the session a batch of warm-up kernels is synchronized
    first, and the launches run twice: a session can miss the records of the first kernels it sees (in a long pytest
    process, the first SIMT launch of a session once went unrecorded), and no launch here may depend on that window."""
    import re

    from torch.profiler import ProfilerActivity, profile

    ops = _ops()
    calls = []
    for dt in MV.DTYPES:
        dtype = DT[dt]
        for dv in (1, 65, 129, 257):
            q = torch.randn(1, 1, 16, device=DEV).to(dtype)
            k = torch.randn(1, 300, 16, device=DEV).to(dtype)
            v = torch.randn(1, 300, dv, device=DEV).to(dtype)
            calls.append(lambda q=q, k=k, v=v: ops.attention(q, k, v, 1, 0.25, impl="simt"))
        po, pm, pl = _states(2, 1, 1, 8, 4, seed=1)
        outs = [torch.empty(1, 8, 4, dtype=dtype, device=DEV) for _ in range(2)]
        calls.append(lambda po=po, pm=pm, pl=pl, outs=outs, dtype=dtype: _peer_call(
            [po[0], po[1]], [pm[0], pm[1]], [pl[0], pl[1]], outs, 1, 1, 8, 4, dtype, 0, 2, (32, 4, 4)))
    state = [t.clone() for t in (po[0], pm[0], pl[0])]
    new_m = pm[0] + 1
    calls.append(lambda: ops.rescale_partial_(*state, new_m))
    scratch = torch.zeros(1024, device=DEV)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(64):
            scratch.add_(1.0)
        torch.cuda.synchronize()
        for _ in range(2):
            for call in calls:
                call()
        torch.cuda.synchronize()
    seen = set()
    tname = {"__nv_bfloat16": MV.BF16, "__half": MV.FP16}
    for ev in prof.key_averages():
        m = re.search(r"(?<!\w)(attn_simt_kernel|combine_kernel|combine_peers_kernel|rescale_kernel)(?:<([^>]*)>)?",
                      ev.key)
        if not m:
            continue
        name = m[1][: -len("_kernel")]
        args = [a.strip() for a in (m[2] or "").split(",") if a.strip()]
        if name == "attn_simt":
            seen.add((name, tname[args[0]], int(args[1])))
        elif name == "rescale":
            seen.add((name,))
        else:
            seen.add((name, tname[args[0]]))
    want = MV.all_instantiations()
    print(f"[merge variants] profiler saw {len(seen & want)} of {len(want)} instantiations")
    assert seen == want, (sorted(want - seen, key=str), sorted(seen - want, key=str))
