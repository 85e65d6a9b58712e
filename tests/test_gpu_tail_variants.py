"""-m gpu: the M-sharded forward's fused merge (peer_tail_kernel<BF16>, csrc/pcv_attn_tc.cu:171-269) on ONE GPU, at every
peer count, row slice and V-pass edge of tail_variants.TAIL_CASES.

G ranks are simulated with ordinary device buffers: part[g], out[g] and a (G, 64) flag block, rank g's words in row g.
Before rank r's launch, the flag words its tail waits on are written (tail_variants.preset_flags) and checked on the
host (wait_set_satisfied); then the ranks are launched one after another on one stream, rank G-1 first.  Two
simulated ranks must never run at once: each tail spins until its whole grid has arrived.

Per case and per epoch (three calls on the same buffers, q changed between them):
  - own state: part[r] after rank r's launch is ops.attention_partial of its shard bit for bit (part[r] is NaN
    before: every rank that reads it has run or runs after);
  - one rank alone: after rank G-1's launch every out[g] holds exactly its rows of the final result, all other rows
    and the stride padding are still NaN;
  - complete: after all G launches the out[g] are the same bits, without NaN, padding untouched;
  - against pcv_attn_combine_peers on the same states, bit for bit, where its fast path applies (the same fmaf
    arithmetic in rank order);
  - against fp64: gpu_util.assert_parity per row, with masks that make uniform rows (every shard padded), a
    finite-fill part beside live ones (one shard padded) and -inf parts (causal shards in a row's future);
  - the flag words: all G "complete" and "pushed" words of every block equal the epoch, every arrival counter is
    epoch * grid, the phase stamps are ordered and no other word changed."""
import ctypes as C
import re

import pytest
import torch

import fwd_variants as FV
import merge_variants as MV
import tail_variants as TV
from gpu_util import assert_parity
from tail_variants import TAIL_CASES, case_id

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENTINEL = 0x5A5A5A5A
EPOCHS = 3


def _ops():
    from perceiver_io_b200 import ops
    return ops


def _lib():
    from perceiver_io_b200 import _lib
    return _lib


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _operands(c, seed):
    """qs (EPOCHS of (1 or B, N, H*dqk)), k (B, m_total, H*dqk), v (B, m_total, H*dv), pad: as
    test_gpu_fwd_variants._operands, every query has a component of norm sqrt(dqk) along a unit direction u_h of its
    head, and padded keys are poisoned (12 u_h, values of magnitude 500..1000), so that one leaked key moves its row."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    B, M, H, dtype = c.B, c.m_total, c.H, TV.TORCH_DTYPE[c.dt]
    u = torch.randn(H, c.dqk, generator=g, device=DEV)
    u = u / u.norm(dim=-1, keepdim=True)
    Bq = 1 if c.G % 2 else B           # a broadcast latent array in half of the cases
    qs = [(torch.randn(Bq, c.N, H, c.dqk, generator=g, device=DEV) + c.dqk ** 0.5 * u).reshape(Bq, c.N, -1).to(dtype)
          for _ in range(EPOCHS)]
    k = torch.randn(B, M, H, c.dqk, generator=g, device=DEV)
    v = torch.randn(B, M, H, c.dv, generator=g, device=DEV)
    pad = TV.pad_mask(c, seed)
    if pad is not None:
        pad = pad.to(DEV)
        pz = pad[:, :, None, None]
        k = torch.where(pz, 12.0 * u, k)
        big = torch.sign(torch.randn(B, M, H, c.dv, generator=g, device=DEV)) * (
            500.0 + 500.0 * torch.rand(B, M, H, c.dv, generator=g, device=DEV))
        v = torch.where(pz, big, v)
    return qs, k.reshape(B, M, -1).to(dtype), v.reshape(B, M, -1).to(dtype), pad


def _rows(out, c):
    """(B, N, W) output buffer -> its (R, dv) rows in (b, h, n) order."""
    d = out[..., :c.H * c.dv].reshape(c.B, c.N, c.H, c.dv)
    return d.permute(0, 2, 1, 3).reshape(c.R, c.dv)


def _flat(state):
    return torch.cat([t.reshape(-1) for t in state])


def _shard_args(c, k, v, pad, g):
    a, b = c.shards[g]
    return (k[:, a:b], v[:, a:b], dict(pad_mask=None if pad is None else pad[:, a:b].contiguous(),
                                      causal=c.mask == "causal", m_total=c.m_total, m_offset=a))


def _fuse(c, r, e, parts, outs, flags):
    f = _lib().ShardFuse()
    for g in range(c.G):
        f.part[g], f.out[g], f.flags[g] = parts[g].data_ptr(), outs[g].data_ptr(), flags[g].data_ptr()
    f.o_stride_b, f.o_stride_n, f.o_stride_h = c.strides
    f.num_peers, f.rank, f.epoch = c.G, r, e
    return f


def _combine_peers(c, parts, outs):
    lib, ops = _lib(), _ops()
    for r in range(c.G):
        p = lib.PeerCombineParams()
        for g in range(c.G):
            base = parts[g].data_ptr()
            p.part_o[g], p.part_m[g], p.part_l[g] = base, base + 4 * c.R * c.dv, base + 4 * (c.R * c.dv + c.R)
            p.out[g] = outs[g].data_ptr()
        p.o_stride_b, p.o_stride_n, p.o_stride_h = c.strides
        p.row_begin, p.row_end = TV.rank_rows(c.R, c.G, r)
        p.num_peers, p.rank = c.G, r
        p.B, p.H, p.N, p.dv = c.B, c.H, c.N, c.dv
        p.dtype = ops._pcv_dtype(TV.TORCH_DTYPE[c.dt])
        lib.check(lib.lib().pcv_attn_combine_peers(C.byref(p), ops._stream()), "pcv_attn_combine_peers")


def _check_flags(flags, before, c, e, grid):
    """After epoch e: every "complete" / "pushed" word is e, every arrival counter e * grid, the stamps ordered, and
    no other word changed."""
    G = c.G
    got = flags.cpu().long()
    assert (got[:, :2 * G] == e).all(), f"{case_id(c)} epoch {e}: flag words {got[:, :2 * G].tolist()}"
    assert (got[:, TV.ARRIVE_WORD] == e * grid).all(), f"{case_id(c)} epoch {e}: arrivals {got[:, TV.ARRIVE_WORD].tolist()}"
    stamps = got[:, list(TV.STAMP_WORDS)] & 0xFFFFFFFF
    assert (stamps[:, 1:] >= stamps[:, :-1]).all(), f"{case_id(c)} epoch {e}: phase stamps {stamps.tolist()}"
    rest = [w for w in range(TV.FLAG_WORDS) if w >= 2 * G and w != TV.ARRIVE_WORD and w not in TV.STAMP_WORDS]
    assert torch.equal(got[:, rest], before.cpu().long()[:, rest]), f"{case_id(c)} epoch {e}: a foreign flag word changed"


@pytest.mark.parametrize("c", TAIL_CASES, ids=case_id)
def test_fused_tail_on_one_gpu(c):
    ops = _ops()
    dtype = TV.TORCH_DTYPE[c.dt]
    grid = _sms()
    G, R = c.G, c.R
    counts, _ = FV.plan_segments(c.B, c.H, c.N, c.Ms, grid, False)
    print(f"[tail] {case_id(c)}: R={R} slices {[TV.rank_rows(R, G, r) for r in range(G)][:4]}... "
          f"plan {'split' if counts['slots'] else 'whole'} ({counts['ctas']} CTAs), "
          f"warp loop wraps: {TV.warp_loop_wraps(R, G, grid)}")
    qs, k, v, pad = _operands(c, seed=G * 1000 + c.N)
    scale = c.dqk ** -0.5
    parts = [torch.empty(R * c.dv + 2 * R, dtype=torch.float32, device=DEV) for _ in range(G)]
    outs = [torch.empty(c.B, c.N, c.W, dtype=dtype, device=DEV) for _ in range(G)]
    flags = torch.zeros(G, TV.FLAG_WORDS, dtype=torch.int32, device=DEV)
    flags[:, 2 * G:] = SENTINEL
    flags[:, TV.ARRIVE_WORD] = 0
    flags[:, list(TV.STAMP_WORDS)] = 0
    initial = flags.clone()
    order = [G - 1] + list(range(G - 1))
    for e in range(1, EPOCHS + 1):
        q = qs[e - 1]
        want_parts = []
        for g in range(G):   # the same plan and kernel as the fused launch, without the tail
            ks, vs, kw = _shard_args(c, k, v, pad, g)
            want_parts.append(_flat(ops.attention_partial(q, ks, vs, c.H, scale, impl="tcgen05", **kw)))
            parts[g].copy_(want_parts[g])
            outs[g].fill_(float("nan"))
        first = None
        for i, r in enumerate(order):
            parts[r].fill_(float("nan"))   # ranks that read part[r] before this launch have run; the rest run after it
            TV.preset_flags(flags, r, G, e)
            assert TV.wait_set_satisfied(flags.cpu(), r, G, e, grid), f"{case_id(c)}: rank {r} epoch {e} could block"
            ks, vs, kw = _shard_args(c, k, v, pad, r)
            ops.attention_sharded_fused(q, ks, vs, c.H, scale, _fuse(c, r, e, parts, outs, flags), **kw)
            assert torch.equal(parts[r].view(torch.int32), want_parts[r].view(torch.int32)), \
                f"{case_id(c)} epoch {e}: rank {r}'s own state differs from attention_partial"
            if i == 0:
                first = [o.clone() for o in outs]
        rows = [_rows(o, c) for o in outs]
        what = f"{case_id(c)} epoch {e}"
        TV.gate_complete(rows, what=what)
        TV.gate_one_rank([_rows(o, c) for o in first], *TV.rank_rows(R, G, G - 1), rows[0], what=what + " rank G-1")
        for o in first + outs:
            assert o[..., c.H * c.dv:].isnan().all(), f"{what}: the stride padding was written"
        _check_flags(flags, initial, c, e, grid)

        sep = [torch.full_like(o, float("nan")) for o in outs]
        fast = MV.peers_fast_path(c.dv, c.strides, [t.data_ptr() for t in parts], [t.data_ptr() for t in sep])
        _combine_peers(c, parts, sep)
        same = torch.equal(_rows(sep[0], c).view(torch.int16), rows[0].view(torch.int16))
        print(f"[tail] {what}: combine_peers ({'fast' if fast else 'general'} path) {'equal' if same else 'DIFFERS'}")
        if fast:
            TV.gate_complete(rows, want=_rows(sep[0], c), what=what + " vs combine_peers")

        out = outs[0][..., :c.H * c.dv]
        assert_parity(out, q, k, v, c.H, scale, pad, c.mask == "causal", what=what, per_row=True)
    torch.cuda.synchronize()


def test_matrix_edges_hold_on_this_device():
    """The warp loop wraps at G = 1 and G = 8 and the split plan is taken, with this device's SM count."""
    grid = _sms()
    for G in (1, 8):
        assert any(c.G == G and TV.warp_loop_wraps(c.R, G, grid) for c in TAIL_CASES), (G, grid)
    split = [c for c in TAIL_CASES if FV.plan_segments(c.B, c.H, c.N, c.Ms, grid, False)[0]["slots"] > 0]
    assert {c.dt for c in split} == set(TV.DTYPES) and any(c.dv > TV.MAX_DV_PASS for c in split), grid


def test_profiler_sees_both_instantiations():
    """peer_tail_kernel<true> (bf16) and <false> (fp16) are launched: one G = 1 call per dtype, twice, after a synchronized
    warm-up batch (a profiler session can miss the first kernels it sees)."""
    from torch.profiler import ProfilerActivity, profile

    ops = _ops()
    c0 = TV.TailCase(TV.BF16, 1, 1, 1, 16, 64, 16, 8, "none", 0)
    calls = []
    flags = torch.zeros(2, TV.FLAG_WORDS, dtype=torch.int32, device=DEV)
    for i, dt in enumerate(TV.DTYPES):
        c = c0._replace(dt=dt)
        qs, k, v, _ = _operands(c, seed=i)
        part = torch.empty(c.R * c.dv + 2 * c.R, device=DEV)
        out = torch.empty(c.B, c.N, c.W, dtype=TV.TORCH_DTYPE[dt], device=DEV)

        def call(e, c=c, q=qs[0], k=k, v=v, part=part, out=out, fl=flags[i:i + 1]):
            assert TV.wait_set_satisfied(fl.cpu(), 0, 1, e, _sms())
            ops.attention_sharded_fused(q, k, v, 1, 0.25, _fuse(c, 0, e, [part], [out], fl), m_total=c.m_total)
        calls.append(call)
    scratch = torch.zeros(1024, device=DEV)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(64):
            scratch.add_(1.0)
        torch.cuda.synchronize()
        for e in (1, 2):
            for call in calls:
                call(e)
        torch.cuda.synchronize()
    seen = {m[1] for ev in prof.key_averages() for m in [re.search(r"peer_tail_kernel<(true|false)>", ev.key)] if m}
    assert seen == {"true", "false"}, seen


def test_zz_watchdog_record_is_clear():
    """No barrier or flag wait of any kernel timed out during this module (runs last in it); the tail's wait sites are
    41, 42 and 43."""
    torch.cuda.synchronize()
    assert _lib().debug_read()[0] == 0, _lib().debug_read()
