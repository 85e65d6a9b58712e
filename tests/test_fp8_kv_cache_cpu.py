"""CPU checks of the FP8 (e4m3) KV cache: the ctypes mirrors of its side structs match the header, its entry points
refuse what they do not cover before any CUDA call (and the bf16 ones refuse e4m3), the weight-derived K / V bounds are
never exceeded (also under rotary and for Perceiver AR's two-norm keys) and are reached, and the arena bookkeeping
works on float8 roots."""
import ctypes
import math
import subprocess

import pytest
import torch

from conftest import ROOT
from perceiver_io_b200 import _lib, ops

F8 = torch.float8_e4m3fn


@pytest.mark.parametrize("struct,cls", [("pcv_decode_fp8", "DecodeFp8"), ("pcv_kv_fp8_scales", "KvFp8Scales"),
                                        ("pcv_rotary_fp8", "RotaryFp8")])
def test_ctypes_mirrors_match_the_header(tmp_path, struct, cls):
    cls = getattr(_lib, cls)
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{ROOT}/include/pcv_attn.h"', "int main(void){",
             f'printf("size %zu\\n", sizeof({struct}));']
    lines += [f'printf("{f} %zu\\n", offsetof({struct}, {f}));' for f, _ in cls._fields_]
    lines.append("return 0;}")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-o", str(exe), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().splitlines() if l)
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def _decode_params(N=1, dqk=64, dv=64, impl=_lib.PCV_IMPL_AUTO):
    H, B, M = 2, 2, 300
    p = _lib.AttnParams()
    p.q, p.k, p.v, p.out = 1 << 20, 2 << 20, 3 << 20, 4 << 20  # never dereferenced: the checks run first
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.q_stride_b, p.q_stride_n, p.q_stride_h = N * H * dqk, H * dqk, dqk
    p.k_stride_b, p.k_stride_m, p.k_stride_h = M * H * dqk, H * dqk, dqk
    p.v_stride_b, p.v_stride_m, p.v_stride_h = M * H * dv, H * dv, dv
    p.o_stride_b, p.o_stride_n, p.o_stride_h = N * H * dv, H * dv, dv
    p.scale, p.dtype, p.m_total, p.impl = 0.125, _lib.PCV_BF16, M, impl
    f = _lib.DecodeFp8()
    f.k_descale, f.v_descale = 5 << 20, 6 << 20
    return p, f


def _refine(p, f, what):
    if what == "partial":
        p.write_partial = 1
        p.part_o = p.part_m = p.part_l = 8 << 20
    elif what == "shard":
        p.m_total, p.m_offset = p.M + 100, 100
    elif what == "stride":
        p.k_stride_m = p.H * p.dqk + 8
    elif what == "descale":
        f.v_descale = None
    elif what == "q_dtype":
        p.dtype = _lib.PCV_E4M3
    return p, f


@pytest.mark.parametrize("kw,what,reason", [
    ({"N": 5}, None, b"more than 4 query rows"),
    ({"dqk": 40}, None, b"multiples of 16"),
    ({"dv": 272}, None, b"head dim > 256"),
    ({"impl": _lib.PCV_IMPL_TCGEN05}, None, b"impl must be AUTO or DECODE"),
    ({}, "partial", b"no write_partial"),
    ({}, "shard", b"no key shard"),
    ({}, "stride", b"multiples of 16 elements"),
    ({}, "descale", b"NULL"),
    ({}, "q_dtype", b"e4m3 operands"),
])
def test_decode_fp8_refusals_without_gpu(kw, what, reason):
    lib = _lib.lib()
    p, f = _refine(*_decode_params(**kw), what)
    assert lib.pcv_attn_decode_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert reason in lib.pcv_last_error()
    assert lib.pcv_attn_decode_fp8(ctypes.byref(p), ctypes.byref(f), None) != 0
    assert reason in lib.pcv_last_error()
    assert lib.pcv_attn_decode_fp8_supported(ctypes.byref(p), None) == 0


def _append_params(dtype=_lib.PCV_BF16, Ck=64, Cv=64):
    B, L, n = 2, 10, 1
    p = _lib.KvAppendParams()
    p.k_cache, p.v_cache, p.k_new, p.v_new, p.k_dst, p.v_dst = (i << 20 for i in range(1, 7))
    p.kc_stride_b, p.kc_stride_l, p.vc_stride_b, p.vc_stride_l = 64 * Ck, Ck, 64 * Cv, Cv
    p.kn_stride_b, p.kn_stride_l, p.vn_stride_b, p.vn_stride_l = n * Ck, Ck, n * Cv, Cv
    p.kd_stride_b, p.kd_stride_l, p.vd_stride_b, p.vd_stride_l = 64 * Ck, Ck, 64 * Cv, Cv
    p.B, p.L_old, p.n, p.Ck, p.Cv, p.dtype = B, L, n, Ck, Cv, dtype
    f = _lib.KvFp8Scales()
    f.k_inv_scale, f.v_inv_scale = 7 << 20, 8 << 20
    return p, f


@pytest.mark.parametrize("kw,change,reason", [
    ({"dtype": _lib.PCV_F32}, None, b"bf16 or fp16"),
    ({"dtype": _lib.PCV_E4M3}, None, b"bf16 or fp16"),
    ({"Ck": 24}, None, b"multiples of 16"),
    ({}, ("kd_stride_l", 72), b"multiples of 16 bytes"),
    ({}, ("kn_stride_l", 68), b"multiples of 8 elements"),
    ({}, ("k_inv_scale", None), b"NULL"),
    ({}, ("k_dst", (1 << 20) + 8), b"16-byte aligned"),
])
def test_kv_append_fp8_refusals_without_gpu(kw, change, reason):
    lib = _lib.lib()
    p, f = _append_params(**kw)
    if change is not None:
        setattr(f if change[0].endswith("inv_scale") else p, *change)
    assert lib.pcv_kv_append_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert reason in lib.pcv_last_error()
    assert lib.pcv_kv_append_fp8(ctypes.byref(p), ctypes.byref(f), None) != 0
    assert reason in lib.pcv_last_error()


def _rotary_params(dtype=_lib.PCV_BF16, d=32):
    p = _lib.RotaryParams()
    p.x, p.y, p.angles = 1 << 20, 2 << 20, 3 << 20
    p.x_stride_b, p.x_stride_n, p.x_stride_h = 4 * 2 * d, 2 * d, d
    p.y_stride_b, p.y_stride_n, p.y_stride_h = 4 * 2 * d, 2 * d, d
    p.a_stride_n = d
    p.B, p.n, p.H, p.d, p.rotate_dim, p.dtype = 1, 4, 2, d, d, dtype
    f = _lib.RotaryFp8()
    f.y_inv_scale = 4 << 20
    return p, f


@pytest.mark.parametrize("kw,change,reason", [
    ({"d": 33}, ("rotate_dim", 32), b"d must be even"),
    ({"dtype": _lib.PCV_E4M3}, None, b"needs x_descale"),
    ({"dtype": _lib.PCV_F32}, None, b"bf16, fp16 or e4m3"),
    ({}, ("y_stride_n", 63), b"strides must be even"),
])
def test_rotary_fp8_refusals_without_gpu(kw, change, reason):
    lib = _lib.lib()
    p, f = _rotary_params(**kw)
    if change is not None:
        setattr(p, *change)
    assert lib.pcv_rotary_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert reason in lib.pcv_last_error()
    assert lib.pcv_rotary_apply_fp8(ctypes.byref(p), ctypes.byref(f), None) != 0


def test_bf16_entry_points_refuse_e4m3():
    lib = _lib.lib()
    p, _ = _append_params(dtype=_lib.PCV_E4M3)
    assert lib.pcv_kv_append(ctypes.byref(p), None) == 1 and b"unknown dtype" in lib.pcv_last_error()
    r, _ = _rotary_params(dtype=_lib.PCV_E4M3)
    assert lib.pcv_rotary_apply(ctypes.byref(r), None) == 1 and b"unknown dtype" in lib.pcv_last_error()
    a, _ = _decode_params(impl=_lib.PCV_IMPL_DECODE)
    a.dtype = _lib.PCV_E4M3
    assert lib.pcv_attn_fwd(ctypes.byref(a), None) == 2 and b"pcv_attn_fwd_fp8" in lib.pcv_last_error()


# ---- the K / V bounds -----------------------------------------------------------------------------------------------
def _ln_linear(C, n, seed, beta_scale=0.3):
    g = torch.Generator().manual_seed(seed)
    ln = torch.nn.LayerNorm(C).double()
    lin = torch.nn.Linear(C, n).double()
    with torch.no_grad():
        ln.weight.copy_(1.0 + 0.5 * torch.randn(C, generator=g))
        ln.bias.copy_(beta_scale * torch.randn(C, generator=g))
        lin.weight.copy_(torch.randn(n, C, generator=g) / math.sqrt(C))
        lin.bias.copy_(0.2 * torch.randn(n, generator=g))
    return ln, lin


def _rows(C, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.cat([torch.randn(1500, C, generator=g), 50.0 * torch.randn(10, C, generator=g) + 3.0,
                      torch.randn(10, C, generator=g).pow(9)]).double()


def _rotate(y, H, angles, rotate_dim):
    """fp64 rotation of (R, H*d) rows by per-row angles (R, rotate_dim), the kernels' pairwise formula."""
    R = y.shape[0]
    y = y.view(R, H, -1).clone()
    a = angles[:, None, :]
    e, o = y[..., 0:rotate_dim:2].clone(), y[..., 1:rotate_dim:2].clone()
    y[..., 0:rotate_dim:2] = e * torch.cos(a[..., 0::2]) - o * torch.sin(a[..., 0::2])
    y[..., 1:rotate_dim:2] = o * torch.cos(a[..., 1::2]) + e * torch.sin(a[..., 1::2])
    return y.view(R, -1)


def _k_descale(norms, lin, H, rotate_dim):
    chan = torch.stack([ops.fp8_descales(n.weight, n.bias, lin.weight, lin.bias, H, per_channel=True)
                        for n in norms]).amax(dim=0)
    return ops.fp8_pair_descale(chan, rotate_dim)


@pytest.mark.parametrize("C,H,d,rotate_dim,beta", [(512, 8, 64, 64, 0.3), (512, 8, 64, 64, 30.0),
                                                   (256, 4, 32, 16, 30.0), (384, 2, 96, 0, 30.0)])
def test_k_bound_holds_before_and_after_rotation(C, H, d, rotate_dim, beta):
    ln, lin = _ln_linear(C, H * d, seed=C + d, beta_scale=beta)
    kd = _k_descale([ln], lin, H, rotate_dim).double()
    with torch.no_grad():
        y = lin(ln(_rows(C, 1)))
    g = torch.Generator().manual_seed(2)
    angles = (1000.0 * torch.rand(y.shape[0], rotate_dim, generator=g, dtype=torch.float64)).repeat_interleave(1, 1)
    angles[:, 1::2] = angles[:, 0::2]                      # rotary repeats every frequency twice
    for rows in (y, _rotate(y, H, angles, rotate_dim)):
        ratio = rows.view(-1, H, d).abs().amax(dim=2) / (kd * 448.0)
        assert (ratio <= 1.0).all(), ratio.max().item()
        assert torch.isfinite((rows.view(-1, H, d).float() / kd.float()[:, None]).to(F8).float()).all()


def test_v_bound_holds_per_channel():
    C, H, d = 512, 8, 64
    ln, lin = _ln_linear(C, H * d, seed=9, beta_scale=30.0)
    vd = ops.fp8_descales(ln.weight, ln.bias, lin.weight, lin.bias, H, per_channel=True).double()
    with torch.no_grad():
        y = lin(ln(_rows(C, 3))).view(-1, H, d)
    assert (y.abs() <= vd * 448.0).all()


def test_two_norm_cross_attention_keys_stay_under_the_max_bound():
    """Perceiver AR: keys of kv_norm(prefix) and of q_norm(latents) go through one k_proj; one bound covers both."""
    C, H, d, rd = 256, 4, 64, 32
    ln_kv, lin = _ln_linear(C, H * d, seed=5, beta_scale=30.0)
    ln_q, _ = _ln_linear(C, H * d, seed=6, beta_scale=0.1)
    kd = _k_descale([ln_kv, ln_q], lin, H, rd).double()
    kd_kv_only = _k_descale([ln_kv], lin, H, rd).double()
    with torch.no_grad():
        keys = torch.cat([lin(ln_kv(_rows(C, 7))), lin(ln_q(_rows(C, 8)))])
    angles = torch.linspace(0, 300, keys.shape[0], dtype=torch.float64)[:, None].expand(-1, rd).contiguous()
    for rows in (keys, _rotate(keys, H, angles, rd)):
        assert (rows.view(-1, H, d).abs().amax(dim=2) <= kd * 448.0).all()
    assert (kd >= kd_kv_only).all()


def test_pair_norm_bound_is_reached_by_the_adversarial_row():
    """With parallel weight rows in a rotary pair (W_2p+1 = lam W_2p, no bias), x_hat = sqrt(C) u0 / |u0| and the angle
    atan2(-y_2p+1, y_2p) rotate channel 2p onto the pair norm of the two single-channel bounds."""
    C, H, d = 1024, 2, 64
    ln, lin = _ln_linear(C, H * d, seed=11, beta_scale=0.0)
    with torch.no_grad():
        lin.bias.zero_()
        lin.weight[1::2] = 0.6 * lin.weight[0::2]
    kd = _k_descale([ln], lin, H, d).double()
    chan = ops.fp8_descales(ln.weight, ln.bias, lin.weight, lin.bias, H, per_channel=True).double().view(-1) * 448.0
    pair = (chan[0::2] ** 2 + chan[1::2] ** 2).sqrt()
    w, _ = ops.fold_ln_linear(ln.weight, ln.bias, [lin.weight], [lin.bias], torch.float64)
    top = int(pair[: d // 2].argmax()) * 2                    # the pair that sets head 0's bound
    for n in (top, 10, 70):
        u0 = w[n].double() - w[n].double().mean()
        x = math.sqrt(C) * u0 / u0.norm()
        with torch.no_grad():
            y = lin(ln(x[None]))[0]
        ya, yb = y[n].item(), y[n + 1].item()
        theta = math.atan2(-yb, ya)
        rotated = ya * math.cos(theta) - yb * math.sin(theta)
        assert abs(rotated) <= kd[n // d].item() * 448.0
        assert abs(rotated) >= 0.97 * pair[n // 2].item(), (n, rotated, pair[n // 2].item())
        assert abs(rotated) > chan[n].item()                  # the single-channel bound alone would be exceeded
    assert abs(rotated) <= kd[1].item() * 448.0
    u0 = w[top].double() - w[top].double().mean()
    with torch.no_grad():
        y = lin(ln((math.sqrt(C) * u0 / u0.norm())[None]))[0]
    assert math.hypot(y[top].item(), y[top + 1].item()) >= 0.97 * kd[0].item() * 448.0


# ---- arena bookkeeping on float8 roots -------------------------------------------------------------------------------
@pytest.fixture
def cpu_launch(monkeypatch):
    calls = {"in_place": 0, "copied": 0}

    def fake_launch(kc, vc, kn, vn, kd, vd, k_in_place, v_in_place, scales=None):
        assert scales is not None and kd.dtype == F8 and vd.dtype == F8
        L = kc.shape[1]
        for cache, new, dst, in_place, inv in ((kc, kn, kd, k_in_place, scales[0]), (vc, vn, vd, v_in_place, scales[1])):
            if in_place:
                calls["in_place"] += 1
            elif L:
                dst[:, :L] = cache
                calls["copied"] += L
            dst[:, L:] = (new.float() * inv).clamp(-448.0, 448.0).to(F8)

    monkeypatch.setattr(ops, "_launch_kv_append", fake_launch)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    return calls


def _codes(x, inv):
    return (x.float() * inv).clamp(-448.0, 448.0).to(F8)


def test_fp8_arena_appends_in_place_at_the_frontier(cpu_launch):
    B, C = 2, 16
    inv = torch.full((C,), 4.0)
    empty = torch.zeros(B, 0, C, dtype=torch.bfloat16)
    rows = [torch.randn(B, 3, C, dtype=torch.bfloat16)]
    k, v = ops.kv_append_fp8(empty, empty, rows[0], rows[0], inv, inv)
    assert k.dtype == F8 and v.dtype == F8 and k.shape == (B, 3, C)
    for _ in range(100):
        rows.append(torch.randn(B, 1, C, dtype=torch.bfloat16))
        k, v = ops.kv_append_fp8(k, v, rows[-1], rows[-1], inv, inv)
        want = _codes(torch.cat(rows, 1), inv)
        assert torch.equal(k.view(torch.uint8), want.view(torch.uint8))
    assert cpu_launch["in_place"] > 2 * 90


def test_fp8_continuations_stay_independent(cpu_launch):
    B, C = 2, 16
    inv = torch.ones(C)
    base = torch.randn(B, 5, C, dtype=torch.bfloat16)
    k, v = ops.kv_append_fp8(torch.empty(B, 0, C, dtype=F8), torch.empty(B, 0, C, dtype=F8), base, base, inv, inv)
    snap = k.view(torch.uint8).clone()
    a, _ = ops.kv_append_fp8(k, v, torch.full((B, 1, C), 1.0, dtype=torch.bfloat16),
                             torch.full((B, 1, C), 1.0, dtype=torch.bfloat16), inv, inv)
    b, _ = ops.kv_append_fp8(k, v, torch.full((B, 1, C), 2.0, dtype=torch.bfloat16),
                             torch.full((B, 1, C), 2.0, dtype=torch.bfloat16), inv, inv)
    assert torch.equal(k.view(torch.uint8), snap)
    assert (a[:, 5].float() == 1).all() and (b[:, 5].float() == 2).all()
    assert torch.equal(a[:, :5].view(torch.uint8), snap) and torch.equal(b[:, :5].view(torch.uint8), snap)


def test_fp8_truncated_view_is_recognised_and_index_select_is_fresh(cpu_launch):
    B, C, W = 3, 16, 12
    inv = torch.full((C,), 2.0)
    full = torch.randn(B, W, C, dtype=torch.bfloat16)
    k, v = ops.kv_append_fp8(torch.empty(B, 0, C, dtype=F8), torch.empty(B, 0, C, dtype=F8), full, full, inv, inv)
    kt, vt = k[:, -(W - 2):], v[:, -(W - 2):]                 # what the sliding-window truncation does
    hit = ops._arena_of(kt)
    assert hit is not None and hit[1] == 2
    new = torch.randn(B, 1, C, dtype=torch.bfloat16)
    before = cpu_launch["in_place"]
    k2, _ = ops.kv_append_fp8(kt, vt, new, new, inv, inv)
    assert cpu_launch["in_place"] == before + 2                # still at the frontier: appended in place
    assert torch.equal(k2.view(torch.uint8), _codes(torch.cat([full[:, 2:], new], 1), inv).view(torch.uint8))
    idx = torch.tensor([2, 0, 1])
    kr, vr = k2.index_select(0, idx), k2.index_select(0, idx)   # what the beam reorder does
    assert kr.dtype == F8 and ops._arena_of(kr) is None
    copied = cpu_launch["copied"]
    k3, _ = ops.kv_append_fp8(kr, vr, new, new, inv, inv)
    assert cpu_launch["copied"] == copied + 2 * kr.shape[1]    # a fresh arena: the old rows were copied once
    assert ops._arena_of(k3) is not None and ops._arena_of(k3)[0] is not ops._arena_of(k2)[0]
    assert torch.equal(k3[:, :-1].view(torch.uint8), kr.view(torch.uint8))


def test_fp8_append_refuses_a_bf16_cache_with_rows(cpu_launch):
    B, C = 1, 16
    inv = torch.ones(C)
    with pytest.raises(ValueError, match="float8_e4m3fn or empty"):
        ops.kv_append_fp8(torch.zeros(B, 2, C, dtype=torch.bfloat16), torch.zeros(B, 2, C, dtype=torch.bfloat16),
                          torch.zeros(B, 1, C, dtype=torch.bfloat16), torch.zeros(B, 1, C, dtype=torch.bfloat16), inv, inv)
