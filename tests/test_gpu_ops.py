"""-m gpu parity tests of the C-ABI ops against the CPU oracle (same seeded, bf16-rounded operands)."""
import pytest
import torch

from gpu_util import assert_close, assert_parity, assert_partial_state, oracle_core, torch_core
from oracle import mha_oracle as O

pytestmark = pytest.mark.gpu

# Parity of the attention kernels is gated by gpu_util.assert_parity: the DERIVED bound of BASELINE.md §3 /
# SURVEY.md §8(d), 2 * max|ref_bf16_eager - ref_fp64| + 1e-3 * max|ref_fp64|, measured per case.  The two
# constants below only remain for comparisons that have no eager counterpart (kernel vs kernel, merged vs single).
REL_SIMT = 6e-3
REL_TC = 1.2e-2


def test_torch_reference_on_device_is_the_cpu_oracle():
    """gpu_util.torch_core (the fp64 / eager-bf16 yardstick evaluated on the GPU) restates the same lines as
    oracle/mha_oracle.py; pin one to the other on a case with every mask type."""
    q, k, v = _qkv(3, 40, 300, 2, 64, 64, Bq=1, seed=3)
    pad = torch.zeros(3, 300, dtype=torch.bool)
    pad[0, :37] = True
    pad[1, :] = True
    for causal in (False, True):
        a = torch_core(q, k, v, 2, 0.125, pad, causal, torch.float64).cpu()
        b = oracle_core(q, k, v, 2, 0.125, pad, causal)
        assert (a - b).abs().max().item() <= 1e-12 * max(b.abs().max().item(), 1.0)


def _qkv(B, N, M, H, dqk, dv, Bq=None, seed=0, q_gain=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    Bq = B if Bq is None else Bq
    q = (torch.randn(Bq, N, H * dqk, generator=g) * q_gain).to(dtype).cuda()
    k = torch.randn(B, M, H * dqk, generator=g).to(dtype).cuda()
    v = torch.randn(B, M, H * dv, generator=g).to(dtype).cuda()
    return q, k, v


SHAPES = [
    # B, N, M, H, dqk, dv
    (2, 8, 24, 4, 8, 8),
    (1, 33, 100, 2, 16, 16),
    (2, 64, 257, 8, 32, 160),     # MLM encoder head dims
    (1, 32, 784, 1, 131, 131),    # MNIST encoder: odd head dim
    (2, 1, 77, 4, 24, 24),        # decode step: one query
    (1, 130, 200, 2, 96, 96),     # Perceiver AR head dim
    (1, 40, 96, 1, 322, 322),     # optical-flow encoder head dim
    (1, 70, 64, 1, 512, 512),     # optical-flow decoder head dim
    (2, 256, 512, 2, 128, 128),   # north-star head dim, small
    (1, 300, 2048, 2, 64, 192),   # wide-dv single-tile mode, split over key ranges
    (1, 130, 300, 2, 128, 256),   # widest v head the tcgen05 family covers
]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_attention_matches_oracle(shape, impl):
    from perceiver_io_b200 import ops

    B, N, M, H, dqk, dv = shape
    q, k, v = _qkv(B, N, M, H, dqk, dv)
    scale = dqk ** -0.5
    out = ops.attention(q, k, v, H, scale, impl=impl)
    assert out.shape == (B, N, H * dv) and out.dtype == torch.bfloat16
    assert_parity(out, q, k, v, H, scale, what=f"{impl} {shape}")


@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_masks_broadcast_and_degenerate_rows(impl):
    from perceiver_io_b200 import ops

    B, N, M, H, d = 3, 40, 300, 2, 64
    q, k, v = _qkv(B, N, M, H, d, d, Bq=1, seed=3)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, :37] = True            # left padding
    pad[1, :] = True              # fully padded row -> uniform average over ALL M values
    pad[2, 250:] = True           # right padding across a tile boundary
    for causal in (False, True):
        out = ops.attention(q, k, v, H, d ** -0.5, pad_mask=pad.cuda(), causal=causal, impl=impl)
        assert_parity(out, q, k, v, H, d ** -0.5, pad, causal, what=f"{impl} causal={causal}")
    # the fully padded batch row equals the plain mean of its values
    mean_v = v[1].float().mean(0).cpu()
    assert_close(out[1, 0], mean_v, 2e-2, "uniform row")


@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_peaked_and_flat_softmax_regimes(impl):
    from perceiver_io_b200 import ops

    B, N, M, H, d = 1, 128, 4096, 2, 128
    for gain, name in ((0.02, "flat"), (6.0, "peaked")):
        q, k, v = _qkv(B, N, M, H, d, d, seed=11, q_gain=gain)
        out = ops.attention(q, k, v, H, d ** -0.5, impl=impl)
        assert_parity(out, q, k, v, H, d ** -0.5, what=f"{impl} {name}")


def test_fp32_inputs_are_rounded_to_bf16_at_the_boundary():
    from perceiver_io_b200 import ops

    q, k, v = _qkv(1, 16, 64, 2, 32, 32, dtype=torch.float32)
    out = ops.attention(q, k, v, 2, 32 ** -0.5)
    assert out.dtype == torch.float32
    assert_parity(out, q.bfloat16(), k.bfloat16(), v.bfloat16(), 2, 32 ** -0.5, what="fp32 boundary")


def test_fp16_inputs():
    from perceiver_io_b200 import ops

    q, k, v = _qkv(2, 16, 100, 2, 64, 64, dtype=torch.float16)
    out = ops.attention(q, k, v, 2, 0.125)
    assert out.dtype == torch.float16
    assert_parity(out, q, k, v, 2, 0.125, what="fp16")


@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("causal", [False, True])
def test_m_shards_merge_to_the_unsharded_result(impl, causal):
    """Partial states of uneven M-shards (one of them fully padded for batch row 0) merged by
    pcv_attn_combine equal the single-pass output and the oracle."""
    from perceiver_io_b200 import ops

    B, N, M, H, d = 2, 48, 1000, 4, 64
    q, k, v = _qkv(B, N, M, H, d, d, seed=5, q_gain=3.0)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, 300:700] = True
    pad[1, :10] = True
    padc = pad.cuda()
    cuts = [0, 300, 700, 1000]
    parts = [ops.attention_partial(q, k[:, a:b], v[:, a:b], H, d ** -0.5, pad_mask=padc[:, a:b], causal=causal,
                                   m_total=M, m_offset=a, impl=impl) for a, b in zip(cuts[:-1], cuts[1:])]
    merged = ops.combine_partials(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]),
                                  torch.stack([p[2] for p in parts]))
    ref = oracle_core(q, k, v, H, d ** -0.5, pad, causal)
    rel = REL_SIMT if impl == "simt" else REL_TC
    assert_close(merged, ref, rel, "merged shards")
    single = ops.attention(q, k, v, H, d ** -0.5, pad_mask=padc, causal=causal, impl=impl)
    assert_close(merged, single.double(), 1e-2, "merged vs single pass")
    # every shard's partial state (o, log2-domain row max, denominator) is the oracle's; the kernels keep the exact
    # running max, and the fully padded shard of batch row 0 has the finite-fill state (m = -FLT_MAX, l = 400)
    for (a, b), part in zip(zip(cuts[:-1], cuts[1:]), parts):
        assert_partial_state(part, q, k[:, a:b], v[:, a:b], H, d ** -0.5, pad[:, a:b], causal, M, a,
                             what=f"{impl} causal={causal} shard [{a}, {b})")


def test_rotary_matches_oracle():
    from perceiver_io_b200 import ops

    g = torch.Generator().manual_seed(2)
    B, n, H, d, f = 2, 37, 4, 24, 12
    x = torch.randn(B, n, H * d, generator=g).bfloat16()
    pos = O.positions(B, n + 5, torch.tensor([[0], [7]]))
    angles = O.frequency_angles(pos, f)
    for right in (True, False):
        y = ops.rotary(x.cuda(), H, angles.cuda(), right)
        ref = O.merge_heads(O.rotate(O.split_heads(x.double(), H), angles.double(), right))
        assert_close(y, ref, 5e-3, f"rotary right_align={right}")
    # batch-1 angles broadcast, full-width rotation
    y = ops.rotary(x.cuda(), H, O.frequency_angles(O.positions(1, n), d).cuda(), False)
    ref = O.merge_heads(O.rotate(O.split_heads(x.double(), H), O.frequency_angles(O.positions(1, n), d).double(), False))
    assert_close(y, ref, 5e-3, "rotary broadcast")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_kv_append_is_bit_exact(dtype):
    from perceiver_io_b200 import ops

    g = torch.Generator().manual_seed(4)
    for (B, L, n, Ck, Cv) in [(2, 0, 5, 64, 96), (3, 17, 1, 64, 64), (1, 9, 4, 20, 6)]:
        kc, vc = torch.randn(B, L, Ck, generator=g).to(dtype), torch.randn(B, L, Cv, generator=g).to(dtype)
        kn, vn = torch.randn(B, n, Ck, generator=g).to(dtype), torch.randn(B, n, Cv, generator=g).to(dtype)
        k, v = ops.kv_append(kc.cuda(), vc.cuda(), kn.cuda(), vn.cuda())
        assert torch.equal(k.cpu(), torch.cat([kc, kn], 1)) and torch.equal(v.cpu(), torch.cat([vc, vn], 1))
    # strided (sliced) cache views, as produced by the HF-side truncation (core/huggingface.py:146-156)
    big_k, big_v = torch.randn(2, 12, 32, generator=g).bfloat16().cuda(), torch.randn(2, 12, 32, generator=g).bfloat16().cuda()
    kn = torch.randn(2, 1, 32, generator=g).bfloat16().cuda()
    k, v = ops.kv_append(big_k[:, -7:], big_v[:, -7:], kn, kn)
    assert torch.equal(k, torch.cat([big_k[:, -7:], kn], 1)) and torch.equal(v, torch.cat([big_v[:, -7:], kn], 1))


def test_errors_surface_as_exceptions():
    from perceiver_io_b200 import ops
    from perceiver_io_b200._lib import PcvError

    q, k, v = _qkv(1, 8, 16, 2, 16, 16)
    with pytest.raises(ValueError):
        ops.attention(q, k[:, :, :16], v, 2, 1.0)
    with pytest.raises(PcvError, match="m_total"):
        ops.attention_partial(q, k, v, 2, 1.0, m_total=8, m_offset=0)


def test_head_major_4d_operands_by_stride():
    """K/V stored (B, H, M, d) and passed as a permuted (B, M, H, d) view: same result, no copy."""
    from perceiver_io_b200 import ops

    B, N, M, H, d = 2, 96, 700, 4, 64
    q, k, v = _qkv(B, N, M, H, d, d, seed=21)
    k_hm = k.view(B, M, H, d).permute(0, 2, 1, 3).contiguous()   # (B, H, M, d) storage
    v_hm = v.view(B, M, H, d).permute(0, 2, 1, 3).contiguous()
    out = ops.attention(q, k_hm.permute(0, 2, 1, 3), v_hm.permute(0, 2, 1, 3), H, d ** -0.5)
    assert_close(out, oracle_core(q, k, v, H, d ** -0.5), REL_TC, "head-major")
    assert torch.equal(out, ops.attention(q, k, v, H, d ** -0.5))


@pytest.mark.parametrize("shape", [(1, 256, 3000, 2, 192, 320), (2, 130, 1500, 1, 322, 322), (1, 300, 2000, 1, 512, 512)],
                         ids=lambda s: "x".join(map(str, s)))
def test_big_head_kernel_multi_tile_with_masks(shape):
    """qk head dims > 128 / v head dims > 256 (optical-flow geometry): Q K^T over up to eight 64-channel boxes (serial
    schedule), two V passes; several key tiles per CTA, padding + causal masks, partial-state output."""
    from perceiver_io_b200 import ops

    B, N, M, H, dqk, dv = shape
    q, k, v = _qkv(B, N, M, H, dqk, dv, seed=23, q_gain=2.0)
    assert ops.tcgen05_supported(q, k, v, H)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, 100:900] = True
    for causal in (False, True):
        out = ops.attention(q, k, v, H, dqk ** -0.5, pad_mask=pad.cuda(), causal=causal, impl="tcgen05")
        assert_parity(out, q, k, v, H, dqk ** -0.5, pad, causal, what=f"big-head causal={causal}")
    if dqk % 8 == 0 and dv % 8 == 0:
        part = ops.attention_partial(q, k, v, H, dqk ** -0.5, pad_mask=pad.cuda(), impl="tcgen05")
        merged = ops.combine_partials(part[0][None], part[1][None], part[2][None])
        assert_close(merged, oracle_core(q, k, v, H, dqk ** -0.5, pad, False), REL_TC, "big-head partial state")


def _ramp_qk(B, N, M, H, dqk, step_log2, dtype, seed=5):
    """Scores that RISE with the key index by `step_log2` (log2 units of the softmax exponent) per 64 keys: the running
    row max moves at every key tile, so the O accumulators (registers) and the denominator are rescaled again and
    again by alpha = 2^(m_old - m_new)."""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(H, dqk, generator=g)
    uq = (u / (u * u).sum(-1, keepdim=True) * dqk ** 0.5).reshape(1, 1, H * dqk)
    q = uq + torch.randn(B, N, H * dqk, generator=g) * 0.05
    ramp = torch.arange(M, dtype=torch.float32)[None, :, None] * (step_log2 * 0.6931 / 64.0)
    k = ramp * u.reshape(1, 1, H * dqk) + torch.randn(B, M, H * dqk, generator=g) * 0.05
    return q.to(dtype).cuda(), k.to(dtype).cuda()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("step", [12.0, 1.5, -3.0], ids=["steep", "gentle", "falling"])
def test_moving_reference_rescale_paths(dtype, step):
    """steep: the max rises by 24 (log2 units) per key tile, so at every tile alpha = 2^-24 all but clears the old
    accumulators; gentle: it rises by 3 per tile (alpha = 1/8), so the roundings of many rescales add up; falling: the
    first tile holds the maximum for good and alpha stays 1."""
    from perceiver_io_b200 import ops

    B, N, M, H, d = 2, 300, 2304, 2, 128
    q, k = _ramp_qk(B, N, M, H, d, step, dtype)
    v = torch.randn(B, M, H * d, generator=torch.Generator().manual_seed(9)).to(dtype).cuda()
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[1, 1000:1100] = True
    for causal, pm in ((False, None), (True, pad)):
        out = ops.attention(q, k, v, H, d ** -0.5, pad_mask=None if pm is None else pm.cuda(), causal=causal, impl="tcgen05")
        assert_parity(out, q, k, v, H, d ** -0.5, pm, causal, what=f"ramp {step} {dtype} causal={causal}")


def test_kv_arena_decode_loop_in_place_append_on_device():
    """Decode-style loop: every step feeds the returned cache back in.  The appended cache must equal torch.cat
    bit for bit, earlier results must stay intact (functional contract), and attention over the arena's strided
    row range must equal attention over a contiguous copy."""
    from perceiver_io_b200 import ops

    B, H, d = 2, 4, 64
    g = torch.Generator().manual_seed(21)
    k = torch.zeros(B, 0, H * d, dtype=torch.bfloat16, device="cuda")
    v = torch.zeros(B, 0, H * d, dtype=torch.bfloat16, device="cuda")
    ks, vs, held = [], [], []
    for step in range(70):
        n = 130 if step == 0 else 1           # prompt, then one token per step
        kn = torch.randn(B, n, H * d, generator=g).bfloat16().cuda()
        vn = torch.randn(B, n, H * d, generator=g).bfloat16().cuda()
        ks.append(kn)
        vs.append(vn)
        k, v = ops.kv_append(k, v, kn, vn)
        assert torch.equal(k, torch.cat(ks, 1)) and torch.equal(v, torch.cat(vs, 1))
        if step % 16 == 0:
            held.append((k, k.clone()))
    assert k._base is not None and not k.is_contiguous()          # a row range of an arena with head-room
    for view, snap in held:                                         # nothing handed out earlier has changed
        assert torch.equal(view, snap)
    q = torch.randn(B, 1, H * d, generator=g).bfloat16().cuda()
    for impl in ("auto", "simt"):
        a = ops.attention(q, k, v, H, d ** -0.5, impl=impl)
        b = ops.attention(q, k.contiguous(), v.contiguous(), H, d ** -0.5, impl=impl)
        assert torch.equal(a, b), impl
    assert_close(a, oracle_core(q, k, v, H, d ** -0.5), REL_SIMT, "arena attention")
    # a second continuation of an older cache must not disturb the newest one
    old_k, old_snap = held[1]
    branch, _ = ops.kv_append(old_k, old_k, torch.ones_like(kn), torch.ones_like(kn))
    assert torch.equal(k, torch.cat(ks, 1)) and torch.equal(branch[:, :-1], old_snap)


def test_rotary_is_differentiable_and_matches_the_torch_rotation():
    """ops.rotary keeps its input in the autograd graph (ADVICE r1): gradient = transpose of the pairwise rotation."""
    from perceiver_io_b200 import ops

    g = torch.Generator().manual_seed(2)
    B, n, H, d, f = 2, 19, 3, 16, 8
    x = torch.randn(B, n, H * d, generator=g).cuda().requires_grad_(True)
    pos = O.positions(B, n + 4, torch.tensor([[0], [3]]))
    angles = O.frequency_angles(pos, f).cuda()
    wgt = torch.randn(B, n, H * d, generator=g).cuda()
    for right in (True, False):
        y = ops.rotary(x, H, angles, right)
        assert y.requires_grad
        (gx,) = torch.autograd.grad((y * wgt).sum(), x)
        xr = x.detach().double().cpu().requires_grad_(True)
        ref = O.merge_heads(O.rotate(O.split_heads(xr, H), angles.double().cpu(), right))
        (gref,) = torch.autograd.grad((ref * wgt.double().cpu()).sum(), xr)
        assert_close(gx, gref, 1e-5, f"rotary grad right_align={right}")


DECODE_SHAPES = [
    # B, N, M, H, dqk, dv
    (8, 1, 16384, 8, 128, 128),   # the Perceiver-AR decode step of BASELINE.json configs[3] (d = 1024)
    (2, 1, 5000, 8, 96, 96),      # giantmidi head dim, ragged key count
    (3, 2, 2049, 4, 64, 64),      # two query rows
    (2, 4, 3000, 8, 32, 160),     # asymmetric head widths, four query rows
    (1, 3, 2500, 1, 256, 256),    # widest rows the streaming kernel takes
    (2, 1, 2048, 2, 8, 8),        # one 16-byte chunk per row
]


@pytest.mark.parametrize("shape", DECODE_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_decode_kernel_matches_oracle(shape, dtype):
    """The streaming kernel for N <= 4 query rows (pcv_attn_decode.cu): padding + right-aligned causal masks, batch-1
    queries broadcast, partial-state output, and `auto` must select it for these shapes."""
    from perceiver_io_b200 import ops

    B, N, M, H, dqk, dv = shape
    q, k, v = _qkv(B, N, M, H, dqk, dv, seed=31, q_gain=2.0, dtype=dtype)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, : M // 9] = True
    if B > 1:
        pad[1, :] = True              # fully padded batch row: uniform average of all values
    scale = dqk ** -0.5
    for causal in (False, True):
        out = ops.attention(q, k, v, H, scale, pad_mask=pad.cuda(), causal=causal, impl="decode")
        assert_parity(out, q, k, v, H, scale, pad, causal, what=f"decode {shape} causal={causal}")
        auto = ops.attention(q, k, v, H, scale, pad_mask=pad.cuda(), causal=causal)
        assert torch.equal(auto, out), "auto did not select the decode kernel"
    q1 = q[:1]
    out = ops.attention(q1, k, v, H, scale, impl="decode")
    assert_parity(out, q1, k, v, H, scale, what=f"decode {shape} broadcast q")
    part = ops.attention_partial(q, k[:, : M // 2], v[:, : M // 2], H, scale, pad_mask=pad.cuda()[:, : M // 2], m_total=M, m_offset=0, impl="decode")
    part2 = ops.attention_partial(q, k[:, M // 2:], v[:, M // 2:], H, scale, pad_mask=pad.cuda()[:, M // 2:], m_total=M, m_offset=M // 2)
    merged = ops.combine_partials(torch.stack([part[0], part2[0]]), torch.stack([part[1], part2[1]]), torch.stack([part[2], part2[2]]), dtype)
    assert_parity(merged, q, k, v, H, scale, pad, False, what=f"decode {shape} two key shards merged")


@pytest.mark.parametrize("shape", [(2, 300, 700, 2, 128, 128), (1, 512, 2048, 4, 64, 128), (3, 400, 900, 2, 96, 96),
                                   (2, 1024, 4096, 2, 128, 128)], ids=lambda s: "x".join(map(str, s)))
def test_cta_pair_kernel_matches_oracle(shape):
    """CTA-pair kernel (a 2-CTA cluster takes two adjacent 128-row query tiles; each CTA loads one 64-key half of
    every K / V box and multicasts it to both, and a ring slot is refilled only after both CTAs released it; split
    units merged by the combine kernel), incl. padding + causal masks, ragged N / M, batch-1 queries and the
    partial-state output."""
    from perceiver_io_b200 import ops

    B, N, M, H, dqk, dv = shape
    q, k, v = _qkv(B, N, M, H, dqk, dv, Bq=1 if B == 3 else None, seed=17, q_gain=2.0)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, : M // 5] = True
    if B > 2:
        pad[2, :] = True
    for causal in (False, True):
        out = ops.attention(q, k, v, H, dqk ** -0.5, pad_mask=pad.cuda(), causal=causal, impl="tcgen05_pair")
        assert_parity(out, q, k, v, H, dqk ** -0.5, pad, causal, what=f"pair {shape} causal={causal}")
    part = ops.attention_partial(q, k, v, H, dqk ** -0.5, pad_mask=pad.cuda(), impl="tcgen05_pair")
    merged = ops.combine_partials(part[0][None], part[1][None], part[2][None])
    assert_parity(merged, q, k, v, H, dqk ** -0.5, pad, False, what=f"pair {shape} partial state")
