"""The FP8 (e4m3) attention forward (ops.attention_fp8, pcv_attn_fwd_fp8) on the GPU against the fp64 emulation of
tests/fp8_emulation.py, which rounds the probabilities where the kernel does.  Each output element is gated at
2^-6 * sum_j p_j |v_j| (the exact probabilities), a quarter of the worst case of rounding every probability to e4m3.
The gate catches layout, fragment-permutation, mask and descale errors; a kernel that rounded P against a slightly
different reference maximum could still stay inside it."""
import math

import pytest
import torch

from fp8_emulation import F8, emulate, make_vt, per_head_descale, quantize
from perceiver_io_b200 import ops

pytestmark = pytest.mark.gpu

GATE = 2.0 ** -6


def _operands(B, Bq, N, M, H, dqk, dv, peaked=False, seed=0):
    """e4m3 operands whose scores the tensor cores compute exactly.

    Hopper's FP8 wgmma does not accumulate in full fp32 (on real-valued codes S differs from fp64 by about 1e-4
    relative), and at large scores that moves probabilities across e4m3 rounding boundaries.  q / k codes here are
    small integers in [-4, 4], so every partial sum of q8 . k8 is an integer below 2^13 and exact; the regime comes
    from the descales: scores (log2 domain) with a spread of about 1.5 (flat) or 16 (peaked).  V codes are full range."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    q8 = torch.randint(-4, 5, (Bq, N, H * dqk), generator=g).float().to(F8).cuda()
    k8 = torch.randint(-4, 5, (B, M, H * dqk), generator=g).float().to(F8).cuda()
    v = torch.randn(B, M, H * dv, generator=g).cuda()
    spread = 16.0 if peaked else 1.5
    sl2 = spread / math.sqrt(dqk * 80.0 / 12.0 * 80.0 / 12.0)  # std of q8 . k8 = sqrt(dqk) * var(code)
    d = math.sqrt(sl2 / (dqk ** -0.5 / math.log(2.0)))
    qd = torch.full((H,), d, device="cuda") * torch.linspace(0.8, 1.2, H, device="cuda")
    kd = torch.full((H,), d, device="cuda")
    vd = per_head_descale(v, H, per_channel=True).cuda()
    vt8 = make_vt(quantize(v, vd, H), H)
    return q8, k8, vt8, qd, kd, vd


def _check(out, ref, what):
    """out (B, N, H*dv) against the emulation dict's out / pv_abs (B, H, N, dv)."""
    B, H, N, dv = ref["out"].shape
    got = out.double().reshape(B, N, H, dv).permute(0, 2, 1, 3)
    err = (got - ref["out"]).abs()
    bound = GATE * ref["pv_abs"]
    assert torch.isfinite(got).all(), what
    worst = (err / bound.clamp_min(1e-300)).max().item()
    assert (err <= bound).all(), f"{what}: max error / gate = {worst:.3f}"


CASES = [
    # B, Bq, N, M, H, dqk, dv, pad, causal, peaked
    pytest.param(2, 1, 200, 1000, 2, 128, 128, False, False, False, id="north-star-dims-bcast-q"),
    pytest.param(3, 3, 130, 900, 2, 32, 160, True, False, False, id="mlm-enc-pad-full-row"),
    pytest.param(2, 2, 200, 700, 2, 64, 96, False, True, False, id="causal-64-96"),
    pytest.param(1, 1, 130, 520, 2, 256, 512, False, False, False, id="256-512"),
    pytest.param(2, 1, 64, 1500, 2, 128, 64, True, True, True, id="peaked-pad-causal"),
    pytest.param(2, 2, 100, 300, 4, 32, 96, False, False, True, id="mlm-dec-peaked"),
]


@pytest.mark.parametrize("B,Bq,N,M,H,dqk,dv,pad,causal,peaked", CASES)
def test_fp8_forward_matches_emulation(B, Bq, N, M, H, dqk, dv, pad, causal, peaked):
    q8, k8, vt8, qd, kd, vd = _operands(B, Bq, N, M, H, dqk, dv, peaked)
    pad_mask = None
    if pad:
        pad_mask = torch.zeros(B, M, dtype=torch.bool, device="cuda")
        pad_mask[0, M - 333:] = True
        pad_mask[-1, :] = True  # a fully padded batch row: the uniform average of its values
    scale = dqk ** -0.5
    assert ops.attention_fp8_supported(q8, k8, vt8, qd, kd, vd, H, scale, pad_mask, causal)
    with torch.no_grad():
        out = ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, scale, pad_mask=pad_mask, causal=causal)
    assert out.dtype == torch.bfloat16 and out.shape == (B, N, H * dv)
    sms = ops.device_info()["num_sms"]
    ref = emulate(q8, k8, vt8, qd, kd, vd, H, scale, pad_mask, causal, workers=sms)
    _check(out, ref, "out")


def test_fp8_key_shards_partial_states_combine():
    """Two key shards (m_offset even and odd) with causal masking, partial=True, merged by combine_partials."""
    B, Bq, N, M, H, dqk, dv = 2, 1, 150, 1100, 2, 64, 160
    q8, k8, vt8, qd, kd, vd = _operands(B, Bq, N, M, H, dqk, dv)
    scale = dqk ** -0.5
    cut = 517
    parts = []
    k_sh = [k8[:, :cut], k8[:, cut:]]
    v8 = vt8[..., :M].permute(0, 3, 1, 2).reshape(B, M, H * dv)  # back to (B, M, H*dv) e4m3
    v_sh = [make_vt(v8[:, :cut].contiguous(), H), make_vt(v8[:, cut:].contiguous(), H)]
    with torch.no_grad():
        for off, kk, vv in ((0, k_sh[0], v_sh[0]), (cut, k_sh[1], v_sh[1])):
            parts.append(ops.attention_fp8(q8, kk.contiguous(), vv, qd, kd, vd, H, scale, causal=True, m_total=M,
                                           m_offset=off, partial=True))
        po, pm, pl = (torch.stack(x) for x in zip(*parts))
        out = ops.combine_partials(po, pm, pl, torch.float16)
        whole = ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, scale, causal=True, out_dtype=torch.float16)
    sms = ops.device_info()["num_sms"]
    refs = [emulate(q8, kk.contiguous(), vv, qd, kd, vd, H, scale, None, True, M, off, workers=sms)
            for off, kk, vv in ((0, k_sh[0], v_sh[0]), (cut, k_sh[1], v_sh[1]))]
    # each shard's state against its own emulation (part_o relative to part_m, and the denominators)
    for (o, m_, l_), r in zip(parts, refs):
        assert ((m_.double() - r["m"]).abs() <= 1e-4 * r["m"].abs().clamp_min(1.0)).all()
        assert ((l_.double() - r["l"]).abs() <= 1e-4 * r["l"]).all()
        err = (o.double() / l_.double()[..., None] - r["out"]).abs()
        assert (err <= GATE * r["pv_abs"]).all()
    m = torch.maximum(refs[0]["m"], refs[1]["m"])
    w0, w1 = torch.exp2(refs[0]["m"] - m), torch.exp2(refs[1]["m"] - m)
    merged_out = (refs[0]["o"] * w0[..., None] + refs[1]["o"] * w1[..., None]) / (refs[0]["l"] * w0 + refs[1]["l"] * w1)[..., None]
    full = emulate(q8, k8, vt8, qd, kd, vd, H, scale, None, True, workers=sms)
    assert out.dtype == torch.float16
    _check(out, {"out": merged_out, "pv_abs": full["pv_abs"]}, "combined shards")
    _check(whole, full, "whole")


def test_fp8_error_against_exact_attention_is_reported():
    """The FP8 result on real-valued operands quantised with amax scales, against exact fp64 attention on the
    unquantised operands, flat and peaked (printed).  Quantising q and k to e4m3 moves each score by a few percent of
    its spread, which at peaked scores changes which keys dominate, so only the flat regime is gated (loosely, against
    gross errors)."""
    from oracle import mha_oracle as O

    B, N, M, H, d = 2, 256, 2048, 2, 128
    for peaked in (False, True):
        g = torch.Generator(device="cpu").manual_seed(1)
        q = torch.randn(1, N, H * d, generator=g) * (4.0 if peaked else 1.0)
        k = torch.randn(B, M, H * d, generator=g) * (4.0 if peaked else 1.0)
        v = torch.randn(B, M, H * d, generator=g)
        q, k, v = (t.cuda().bfloat16() for t in (q, k, v))
        qd, kd, vd = per_head_descale(q, H), per_head_descale(k, H), per_head_descale(v, H, per_channel=True)
        q8, k8 = quantize(q, qd, H), quantize(k, kd, H)
        vt8 = make_vt(quantize(v, vd, H), H)
        with torch.no_grad():
            out8 = ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, d ** -0.5)
            out16 = ops.attention(q, k, v, H, d ** -0.5)
        split = lambda t: O.split_heads(t.cpu().double(), H)
        ref = O.merge_heads(O.core_attention(split(q.expand(B, -1, -1)), split(k), split(v), d ** -0.5, None))
        e8 = (out8.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
        e16 = (out16.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
        print(f"{'peaked' if peaked else 'flat'}: max |err| / max |ref|  fp8 {e8:.3e}  bf16 {e16:.3e}")
        assert math.isfinite(e8) and (peaked or e8 < 0.25)


def test_fp8_rejects_what_it_does_not_cover():
    q8, k8, vt8, qd, kd, vd = _operands(1, 1, 64, 256, 1, 64, 64)
    assert ops.attention_fp8_supported(q8, k8, vt8, qd, kd, vd, 1, 0.125)
    with pytest.raises(Exception, match="FP8"):
        ops.attention_fp8(q8, k8, vt8, qd, kd, vd, 1, 0.0)  # scale must be positive
