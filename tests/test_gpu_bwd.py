"""-m gpu: the tensor-core backward kernels (pcv_attn_bwd) against autograd through the reference algorithm.

Reference gradients come from torch autograd through `gpu_util.torch_core` (the reference's own op sequence,
modules.py:123-167) in float64 on the SAME rounded operands; every gradient goes through `gpu_util.assert_grads`: the
derived whole-tensor gate of the forward tests, max|kernel - ref64| <= max(2 * max|eager_16bit_autograd - ref64| +
1e-3 * max|ref64|, 6e-3 * max|ref64|), and an element-wise gate scaled by the fp64 gradient on magnitudes."""
import pytest
import torch

from gpu_util import GradMagnitude, assert_grad_set, assert_grads, grad_magnitudes, torch_core
from perceiver_io_b200 import _lib, ops

pytestmark = pytest.mark.gpu


def _ref_grads(q, k, v, go, H, scale, pad, causal, dtype):
    qq, kk, vv = (t.detach().to(dtype).requires_grad_() for t in (q, k, v))
    o = torch_core(qq, kk, vv, H, scale, pad, causal, dtype)
    o.backward(go.to(dtype))
    return qq.grad, kk.grad, vv.grad


def _case(B, N, M, H, dqk, dv, pad_kind=None, causal=False, bcast=False, dtype=torch.bfloat16, seed=0, peaked=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sc = 3.0 if peaked else 1.0
    q = (torch.randn(1 if bcast else B, N, H * dqk, device="cuda", generator=g) * sc).to(dtype)
    k = (torch.randn(B, M, H * dqk, device="cuda", generator=g) * sc).to(dtype)
    v = torch.randn(B, M, H * dv, device="cuda", generator=g).to(dtype)
    go = torch.randn(B, N, H * dv, device="cuda", generator=g).to(dtype)
    pad = None
    if pad_kind == "ragged":
        lens = torch.randint(1, M + 1, (B,), device="cuda", generator=g)
        pad = torch.arange(M, device="cuda")[None, :] >= lens[:, None]
    elif pad_kind == "row_full":  # one batch row entirely padding: uniform attention, gradient only into V
        pad = torch.zeros(B, M, dtype=torch.bool, device="cuda")
        pad[0] = True
        if B > 1:
            pad[1, M // 3:] = True
    elif pad_kind == "random":
        pad = torch.rand(B, M, device="cuda", generator=g) < 0.3
        pad[:, 0] = False
    return q, k, v, go, pad


def _check(q, k, v, go, H, pad, causal, what):
    scale = (q.shape[-1] // H) ** -0.5
    po, pm, pl = ops.attention_partial(q, k, v, H, scale, pad_mask=pad, causal=causal)
    out = ops.combine_partials(po[None], pm[None], pl[None], q.dtype)
    got = ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, pad_mask=pad, causal=causal)
    ref = _ref_grads(q, k, v, go, H, scale, pad, causal, torch.float64)
    eag = _ref_grads(q, k, v, go, H, scale, pad, causal, q.dtype)
    mags = grad_magnitudes(q, k, v, go, H, scale, pad, causal)
    return max(assert_grad_set(got, ref, eag, mags, q.dtype, what).values())


CASES = [
    # B, N, M, H, dqk, dv, pad, causal, bcast
    (2, 256, 1024, 2, 128, 128, None, False, False),
    (1, 128, 128, 1, 64, 64, None, False, False),
    (2, 200, 1000, 4, 64, 64, "ragged", False, False),
    (1, 100, 40, 2, 32, 96, None, False, False),
    (2, 96, 352, 2, 64, 64, None, True, False),
    (3, 300, 900, 2, 64, 128, "random", True, True),
    (2, 130, 700, 2, 128, 64, "row_full", False, False),
    (2, 512, 4096, 8, 128, 128, None, False, True),
    (2, 384, 2048, 4, 96, 96, "ragged", True, False),
]


@pytest.mark.parametrize("case", CASES, ids=[f"B{c[0]}N{c[1]}M{c[2]}H{c[3]}d{c[4]}x{c[5]}{c[6] or ''}{'c' if c[7] else ''}{'b' if c[8] else ''}" for c in CASES])
def test_bwd_kernels_match_autograd(case):
    B, N, M, H, dqk, dv, pad_kind, causal, bcast = case
    q, k, v, go, pad = _case(B, N, M, H, dqk, dv, pad_kind, causal, bcast)
    _check(q, k, v, go, H, pad, causal, f"{case}")


def test_bwd_fp16_and_peaked():
    q, k, v, go, pad = _case(2, 256, 1536, 2, 64, 64, "ragged", False, False, dtype=torch.float16, seed=3)
    _check(q, k, v, go, 2, pad, False, "fp16")
    q, k, v, go, pad = _case(1, 256, 2048, 2, 128, 128, None, False, False, seed=4, peaked=True)
    _check(q, k, v, go, 2, pad, False, "peaked")


def test_autograd_routes_through_the_kernels():
    """ops.attention under autograd: backward = pcv_attn_bwd (impl 'kernel' raises if it were not), and it agrees with
    the torch shim on the same call."""
    q, k, v, go, pad = _case(2, 256, 1024, 4, 64, 64, "ragged", False, False, seed=7)
    scale = 64 ** -0.5
    grads = {}
    for mode in ("kernel", "shim"):
        ops.backward_config["impl"] = mode
        try:
            qq, kk, vv = (t.detach().clone().requires_grad_() for t in (q, k, v))
            before = _lib.launch_count()
            o = ops.attention(qq, kk, vv, 4, scale, pad_mask=pad)
            o.backward(go)
            grads[mode] = (qq.grad, kk.grad, vv.grad, _lib.launch_count() - before)
        finally:
            ops.backward_config["impl"] = "auto"
    assert grads["kernel"][3] > grads["shim"][3]  # the shim launches nothing of ours in backward
    for a, b_, name in zip(grads["kernel"][:3], grads["shim"][:3], ("dq", "dk", "dv")):
        ref_max = b_.float().abs().max().item()
        err = (a.float() - b_.float()).abs().max().item()
        print(f"[bwd kernel vs shim] {name}: {err:.3e} (max {ref_max:.3e})")
        assert err <= 1.5e-2 * ref_max, name


def test_bwd_full_size_slices():
    """The benchmarked shape (B=8, N=512, M=65536, H=8, d=128): gradients of whole (b, h) slices against float64
    autograd of the reference algorithm on that slice (512 x 65536 scores fit in float64 on the device)."""
    B, N, M, H, d = 8, 512, 65536, 8, 128
    g = torch.Generator(device="cuda").manual_seed(11)
    q = torch.randn(1, N, H * d, device="cuda", generator=g).to(torch.bfloat16)
    k = torch.randn(B, M, H * d, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn(B, M, H * d, device="cuda", generator=g).to(torch.bfloat16)
    go = torch.randn(B, N, H * d, device="cuda", generator=g).to(torch.bfloat16)
    pad = torch.zeros(B, M, dtype=torch.bool, device="cuda")
    pad[5, 40000:] = True
    scale = d ** -0.5
    po, pm, pl = ops.attention_partial(q, k, v, H, scale, pad_mask=pad)
    out = ops.combine_partials(po[None], pm[None], pl[None], q.dtype)
    gq, gk, gv = ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, pad_mask=pad)
    assert torch.isfinite(gq).all() and torch.isfinite(gk).all() and torch.isfinite(gv).all()
    dq_sum = torch.zeros(N, d, dtype=torch.float64, device="cuda")
    for b, h in ((0, 0), (5, 3), (7, 7)):
        sl = slice(h * d, (h + 1) * d)
        refs = _ref_grads(q[:, :, sl], k[b:b + 1, :, sl], v[b:b + 1, :, sl], go[b:b + 1, :, sl], 1, scale,
                          pad[b:b + 1], False, torch.float64)
        eag = _ref_grads(q[:, :, sl], k[b:b + 1, :, sl], v[b:b + 1, :, sl], go[b:b + 1, :, sl], 1, scale,
                         pad[b:b + 1], False, torch.bfloat16)
        mags = grad_magnitudes(q[:, :, sl], k[b:b + 1, :, sl], v[b:b + 1, :, sl], go[b:b + 1, :, sl], 1, scale,
                               pad[b:b + 1], False)
        for name, got, r_, e_, m_ in (("dk", gk[b:b + 1, :, sl], refs[1], eag[1], mags[1]),
                                      ("dv", gv[b:b + 1, :, sl], refs[2], eag[2], mags[2])):
            assert_grads(got, r_, e_, m_, q.dtype, f"full size (b={b},h={h}) {name}")
        del refs, eag, mags
    # dq of the shared latents sums over the batch: check one head against the float64 sum over all 8 batch rows
    h = 2
    sl = slice(h * d, (h + 1) * d)
    eag_sum = torch.zeros(N, d, dtype=torch.float64, device="cuda")
    abs_sum, sub_sum = (torch.zeros(N, d, dtype=torch.float64, device="cuda") for _ in range(2))
    for b in range(B):
        r = _ref_grads(q[:, :, sl], k[b:b + 1, :, sl], v[b:b + 1, :, sl], go[b:b + 1, :, sl], 1, scale, pad[b:b + 1], False,
                       torch.float64)[0]
        e = _ref_grads(q[:, :, sl], k[b:b + 1, :, sl], v[b:b + 1, :, sl], go[b:b + 1, :, sl], 1, scale, pad[b:b + 1], False,
                       torch.bfloat16)[0]
        m_ = grad_magnitudes(q[:, :, sl], k[b:b + 1, :, sl], v[b:b + 1, :, sl], go[b:b + 1, :, sl], 1, scale,
                             pad[b:b + 1], False)[0]
        dq_sum += r[0]
        eag_sum += e[0].double()
        abs_sum += m_.abs[0]
        sub_sum += m_.sub[0] - 1.0  # one output spacing in all, added below
    assert_grads(gq[0, :, sl], dq_sum, eag_sum, GradMagnitude(abs_sum, sub_sum + 1.0), q.dtype, f"full size dq head {h}")
