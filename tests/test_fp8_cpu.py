"""CPU checks of the FP8 forward: the weight-derived scales (ops.fp8_descales) are never exceeded, the ctypes mirror
of pcv_fp8_attn matches the header, the e4m3 entry points refuse what they do not cover before any CUDA call, and the
fp64 emulation used as the GPU tests' oracle follows the kernel's rounding steps."""
import ctypes
import math
import subprocess

import pytest
import torch

from conftest import ROOT
from fp8_emulation import FLT_MAX, LOG2E, emulate, make_vt, per_head_descale, quantize, round_p, score_scale
from perceiver_io_b200 import _lib, ops


def _ln_linear(C, n, seed):
    g = torch.Generator().manual_seed(seed)
    ln = torch.nn.LayerNorm(C)
    lin = torch.nn.Linear(C, n)
    with torch.no_grad():
        ln.weight.copy_(1.0 + 0.5 * torch.randn(C, generator=g))
        ln.bias.copy_(0.3 * torch.randn(C, generator=g))
        lin.weight.copy_(torch.randn(n, C, generator=g) / math.sqrt(C))
        lin.bias.copy_(0.2 * torch.randn(n, generator=g))
    return ln, lin


@pytest.mark.parametrize("C,H,d", [(1024, 8, 128), (512, 8, 32), (256, 4, 40)])
def test_descales_are_never_exceeded_on_random_inputs(C, H, d):
    ln, lin = _ln_linear(C, H * d, seed=C + d)
    head = ops.fp8_descales(ln.weight, ln.bias, lin.weight, lin.bias, H)
    chan = ops.fp8_descales(ln.weight, ln.bias, lin.weight, lin.bias, H, per_channel=True)
    assert head.shape == (H,) and chan.shape == (H, d) and head.dtype == torch.float32
    assert torch.equal(chan.amax(dim=1), head)
    g = torch.Generator().manual_seed(7)
    x = torch.cat([torch.randn(2000, C, generator=g), 50.0 * torch.randn(10, C, generator=g) + 3.0,
                   torch.randn(10, C, generator=g).pow(9)])  # heavy-tailed rows too
    with torch.no_grad():
        y = lin(ln(x)).double().view(-1, H, d)
    assert (y.abs() <= chan.double() * 448.0).all()
    assert (y.abs().amax(dim=2) <= head.double() * 448.0).all()
    # quantising y / descale never saturates, and a typical value sits a few binades below 448
    assert torch.isfinite((y.float() / chan).to(torch.float8_e4m3fn).float()).all()
    assert (y.abs() / (chan.double() * 448.0)).max() > 2.0 ** -6


def test_descale_bound_is_reached_by_the_adversarial_row():
    """x_hat = sqrt(C) u0 / |u0| (u = gamma * W_n, u0 its zero-mean part, signed as t_n) attains the bound up to the
    mean of u, which LayerNorm removes."""
    C, H, d = 1024, 8, 128
    ln, lin = _ln_linear(C, H * d, seed=3)
    chan = ops.fp8_descales(ln.weight, ln.bias, lin.weight, lin.bias, H, per_channel=True).double().view(-1)
    w, col_st = ops.fold_ln_linear(ln.weight, ln.bias, [lin.weight], [lin.bias], torch.float32)
    for n in (0, 77, 1023):
        u = w[n].double()
        u0 = u - u.mean()
        sign = 1.0 if col_st[n, 1] >= 0 else -1.0
        x = sign * math.sqrt(C) * u0 / u0.norm()
        with torch.no_grad():
            y = lin.double()(ln.double()(x[None]))[0, n].item()
        bound = chan[n].item() * 448.0
        assert abs(y) <= bound
        assert abs(y) >= 0.97 * bound, (n, y, bound)


def test_descales_need_the_layernorm():
    lin = torch.nn.Linear(64, 64)
    with pytest.raises(ValueError, match="LayerNorm"):
        ops.fp8_descales(None, None, lin.weight, lin.bias, 4)


def test_ctypes_mirror_matches_the_header(tmp_path):
    header = f"{ROOT}/include/pcv_attn.h"
    cls = _lib.Fp8Attn
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void){",
             'printf("size %zu\\n", sizeof(pcv_fp8_attn));', 'printf("e4m3 %d\\n", (int)PCV_E4M3);']
    lines += [f'printf("{f} %zu\\n", offsetof(pcv_fp8_attn, {f}));' for f, _ in cls._fields_]
    lines.append("return 0;}")
    src = tmp_path / "fp8_layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "fp8_layout"
    subprocess.check_call(["gcc", "-o", str(exe), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines() if l)
    assert int(got["size"]) == ctypes.sizeof(cls)
    assert int(got["e4m3"]) == _lib.PCV_E4M3 == 3
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def _fp8_params(dqk=64, dv=64, impl=_lib.PCV_IMPL_AUTO):
    p = _lib.AttnParams()
    p.q, p.k, p.v, p.out = 1 << 20, 2 << 20, 3 << 20, 4 << 20  # never dereferenced: the checks run first
    p.B, p.H, p.N, p.M, p.dqk, p.dv = 2, 2, 128, 256, dqk, dv
    p.q_stride_b, p.q_stride_n, p.q_stride_h = 128 * 2 * dqk, 2 * dqk, dqk
    p.k_stride_b, p.k_stride_m, p.k_stride_h = 256 * 2 * dqk, 2 * dqk, dqk
    p.o_stride_b, p.o_stride_n, p.o_stride_h = 128 * 2 * dv, 2 * dv, dv
    p.scale, p.dtype, p.m_total, p.impl = 0.125, _lib.PCV_E4M3, 256, impl
    f = _lib.Fp8Attn()
    f.q_descale, f.k_descale, f.v_descale = 5 << 20, 6 << 20, 7 << 20
    f.vt_stride_c, f.vt_stride_h, f.vt_stride_b = 256, 256 * dv, 256 * dv * 2
    f.out_dtype = _lib.PCV_BF16
    return p, f


@pytest.mark.parametrize("kw,reason", [
    ({"dqk": 40}, b"multiples of 16"),
    ({"dqk": 272}, b"qk head dim > 256"),
    ({"dv": 520}, b"v head dim > 512"),
    ({"impl": _lib.PCV_IMPL_TCGEN05_PAIR}, b"single-CTA tensor-core kernel only"),
    ({"impl": _lib.PCV_IMPL_DECODE}, b"single-CTA tensor-core kernel only"),
])
def test_fp8_supported_reasons_without_gpu(kw, reason):
    lib = _lib.lib()
    p, f = _fp8_params(**kw)
    assert lib.pcv_attn_fwd_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert reason in lib.pcv_last_error()
    assert lib.pcv_attn_fwd_fp8(ctypes.byref(p), ctypes.byref(f), None) == 2
    assert reason in lib.pcv_last_error()


def test_e4m3_is_refused_by_the_16_bit_forward_entries():
    lib = _lib.lib()
    p, f = _fp8_params()
    assert lib.pcv_attn_fwd(ctypes.byref(p), None) == 2 and b"pcv_attn_fwd_fp8" in lib.pcv_last_error()
    p.write_partial = 1
    p.part_o = p.part_m = p.part_l = 8 << 20
    assert lib.pcv_attn_fwd_sharded_supported(ctypes.byref(p)) == 0 and b"pcv_attn_fwd_fp8" in lib.pcv_last_error()
    assert lib.pcv_attn_fwd_partial_dropout_supported(ctypes.byref(p), ctypes.c_float(0.1)) == 0
    assert b"pcv_attn_fwd_fp8" in lib.pcv_last_error()
    f.out_dtype = _lib.PCV_F32
    assert lib.pcv_attn_fwd_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert b"out_dtype" in lib.pcv_last_error()
    assert lib.pcv_attn_fwd_fp8_supported(ctypes.byref(p), None) == 0


def test_probability_rounding_step():
    p = torch.tensor([1.0, 0.5, 2.0 ** -14, 2.0 ** -20, 0.0, 0.3, 0.999], dtype=torch.float64)
    r = round_p(p)
    assert r[0] == 1.0 and r[1] == 0.5 and r[2] == 2.0 ** -14 and r[4] == 0.0
    assert (r <= 1.0).all() and ((r - p).abs() <= p * 2.0 ** -4 + 2.0 ** -17).all()
    assert r[3] == 0.0  # below half the smallest e4m3 subnormal after the 2^8 scale: flushed


def _operands(B, N, M, H, dqk, dv, seed=0):
    g = torch.Generator().manual_seed(seed)
    q, k = torch.randn(1, N, H * dqk, generator=g) * 2, torch.randn(B, M, H * dqk, generator=g) * 2
    v = torch.randn(B, M, H * dv, generator=g)
    qd, kd, vd = per_head_descale(q, H), per_head_descale(k, H), per_head_descale(v, H, per_channel=True)
    return quantize(q, qd, H), quantize(k, kd, H), make_vt(quantize(v, vd, H), H), qd, kd, vd


def test_emulation_of_one_tile_is_the_direct_formula():
    """M <= 128: one tile, one segment; P relative to the row max, rounded, over the unrounded sum."""
    B, N, M, H, dqk, dv = 1, 20, 100, 2, 32, 48
    q8, k8, vt8, qd, kd, vd = _operands(B, N, M, H, dqk, dv)
    scale = dqk ** -0.5
    ref = emulate(q8, k8, vt8, qd, kd, vd, H, scale)
    q = q8.double().view(1, N, H, dqk).permute(0, 2, 1, 3)
    k = k8.double().view(B, M, H, dqk).permute(0, 2, 1, 3)
    t = (q @ k.transpose(-1, -2)) * score_scale(scale, qd, kd)[None, :, None, None]
    p = torch.exp2(t - t.amax(dim=-1, keepdim=True))
    v = vt8[..., :M].double().transpose(-1, -2) * vd.double()[None, :, None, :]
    want = (round_p(p) @ v) / p.sum(dim=-1, keepdim=True)
    assert torch.allclose(ref["out"], want, rtol=1e-10, atol=1e-12)
    assert ((ref["out"] - torch.softmax(t / LOG2E, -1) @ v).abs() <= 2.0 ** -4 * ref["pv_abs"] + 1e-12).all()


def test_emulation_rounds_relative_to_the_running_maximum():
    """Several tiles in one segment: each tile's probabilities are rounded relative to the running maximum at that
    tile (then rescaled), as the kernel's online softmax does, which differs from rounding relative to the final max."""
    B, N, M, H, dqk, dv = 1, 8, 512, 1, 32, 32
    q8, k8, vt8, qd, kd, vd = _operands(B, N, M, H, dqk, dv, seed=4)
    scale = dqk ** -0.5
    ref = emulate(q8, k8, vt8, qd, kd, vd, H, scale, workers=1)  # one CTA: one segment over all 4 tiles
    q = q8.double().view(1, N, H, dqk).permute(0, 2, 1, 3)
    k = k8.double().view(B, M, H, dqk).permute(0, 2, 1, 3)
    t = ((q @ k.transpose(-1, -2)) * score_scale(scale, qd, kd)[None, :, None, None])[0, 0]
    v = vt8[0, 0].double().t() * vd.double()[0][None, :]
    o = torch.zeros(N, dv, dtype=torch.float64)
    l = torch.zeros(N, dtype=torch.float64)
    m = torch.full((N,), -math.inf, dtype=torch.float64)
    for j0 in range(0, M, 128):
        x = t[:, j0:j0 + 128]
        mn = torch.maximum(m, x.amax(dim=1))
        a = torch.exp2(m - mn)
        pt = torch.exp2(x - mn[:, None])
        o = o * a[:, None] + round_p(pt) @ v[j0:j0 + 128]
        l = l * a + pt.sum(dim=1)
        m = mn
    assert torch.allclose(ref["out"][0, 0], o / l[:, None], rtol=1e-10, atol=1e-12)
    final = torch.exp2(t - t.amax(dim=1, keepdim=True))
    assert not torch.allclose(ref["out"][0, 0], (round_p(final) @ v) / final.sum(dim=1, keepdim=True), rtol=1e-9)


def test_emulation_masks_like_the_kernel():
    """Pad and causal keys take the finite fill, so a fully padded row is the uniform average of its M values."""
    B, N, M, H, dqk, dv = 2, 16, 200, 1, 32, 32
    q8, k8, vt8, qd, kd, vd = _operands(B, N, M, H, dqk, dv, seed=5)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[1] = True
    ref = emulate(q8, k8, vt8, qd, kd, vd, H, 0.2, pad_mask=pad, causal=True, m_total=M + 40, m_offset=40)
    v = vt8[1, 0, :, :M].double().t() * vd.double()[0][None, :]
    assert torch.allclose(ref["out"][1, 0], v.mean(dim=0).expand(N, dv), rtol=1e-10, atol=1e-12)
    assert torch.isfinite(ref["out"]).all() and (ref["m"][1] == -FLT_MAX).all()


def test_producer_ctypes_mirror_matches_the_header(tmp_path):
    header = f"{ROOT}/include/pcv_attn.h"
    cls = _lib.KvProjFp8
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void){",
             'printf("size %zu\\n", sizeof(pcv_kvproj_fp8));']
    lines += [f'printf("{f} %zu\\n", offsetof(pcv_kvproj_fp8, {f}));' for f, _ in cls._fields_]
    lines.append("return 0;}")
    src = tmp_path / "kv8_layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "kv8_layout"
    subprocess.check_call(["gcc", "-o", str(exe), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines() if l)
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def test_zero_key_batch_stride_is_refused():
    lib = _lib.lib()
    p, f = _fp8_params()
    f.vt_stride_b = 0
    assert lib.pcv_attn_fwd_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert b"non-zero batch stride" in lib.pcv_last_error()
    p, f = _fp8_params()
    p.k_stride_b = 0
    assert lib.pcv_attn_fwd_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0


def test_producer_fp8_refusals_without_gpu():
    lib = _lib.lib()
    p = _lib.KvProjParams()
    p.x, p.w, p.col_st, p.k_out = 1 << 20, 2 << 20, 3 << 20, 4 << 20
    p.x_stride_row, p.k_stride_row, p.rows, p.C, p.n_k, p.n_v, p.dtype = 512, 512, 2000, 512, 512, 512, _lib.PCV_BF16
    f = _lib.KvProjFp8()
    f.inv_scale, f.vt_out = 5 << 20, 6 << 20
    f.keys_per_batch, f.v_head_dim = 1000, 128
    f.vt_stride_c, f.vt_stride_h, f.vt_stride_b = 1008, 1008 * 128, 1008 * 512
    p.cta_group = 2
    assert lib.pcv_kv_project_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert b"one CTA per tile" in lib.pcv_last_error()
    p.cta_group = 0
    f.keys_per_batch = 999
    assert lib.pcv_kv_project_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert b"keys_per_batch" in lib.pcv_last_error()
    assert lib.pcv_kv_project_fp8(None, None, None) == 1
