"""-m gpu: attention-probability dropout (reference modules.py:161) in the training kernels.

The mask is counter-based (a pure function of seed, b, h, query, key), so the tests export it with
`ops.dropout_keep_mask` and evaluate the reference algorithm — softmax, mask * 1/(1-p), P V — with exactly that mask in
float64; the forward is then held to the derived gate of the other parity tests, the gradients to gpu_util.assert_grads
(the derived gate and the element-wise one)."""
import pytest
import torch

from gpu_util import GRAD_FLOOR, assert_grad_set, derived_bound, grad_magnitudes
from perceiver_io_b200 import modules, ops

pytestmark = pytest.mark.gpu

FLOOR = GRAD_FLOOR


def _rp(p):
    t = min(255, max(1, round(p * 256)))
    return t, 256.0 / (256.0 - t)


def _core_drop(q, k, v, H, scale, pad, causal, dtype, keep, rp):
    """gpu_util.torch_core with the dropout step of the reference (:161) on a given keep mask."""
    B, M = k.shape[0], k.shape[1]
    N = q.shape[1]
    qh = q.to(dtype).expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2) * scale
    kh = k.to(dtype).reshape(B, M, H, -1).transpose(1, 2)
    vh = v.to(dtype).reshape(B, M, H, -1).transpose(1, 2)
    attn = torch.einsum("bhic,bhjc->bhij", qh, kh)
    neg = -torch.finfo(attn.dtype).max
    if pad is not None:
        attn = attn.masked_fill(pad.bool()[:, None, None, :], neg)
    if causal:
        attn = attn.masked_fill(torch.ones(N, M, device=q.device, dtype=torch.bool).triu(M - N + 1), neg)
    attn = attn.softmax(dim=-1)
    attn = attn * keep.to(dtype) * rp                                   # nn.Dropout in training mode
    o = torch.einsum("bhij,bhjc->bhic", attn, vh)
    return o.transpose(1, 2).reshape(B, N, -1)


def _drop_ref(q, k, v, go, H, scale, pad, causal, dtype, keep, rp):
    """Autograd of _core_drop in `dtype` on the given keep mask -> (out, grad_q, grad_k, grad_v)."""
    a, b_, c = (t.detach().to(dtype).requires_grad_() for t in (q, k, v))
    o = _core_drop(a, b_, c, H, scale, pad, causal, dtype, keep, rp)
    o.backward(go.to(dtype))
    return o.detach(), a.grad, b_.grad, c.grad


def _inputs(B, N, M, H, dqk, dv, pad_kind, bcast, seed, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(1 if bcast else B, N, H * dqk, device="cuda", generator=g).to(dtype)
    k = torch.randn(B, M, H * dqk, device="cuda", generator=g).to(dtype)
    v = torch.randn(B, M, H * dv, device="cuda", generator=g).to(dtype)
    go = torch.randn(B, N, H * dv, device="cuda", generator=g).to(dtype)
    pad = None
    if pad_kind == "ragged":
        lens = torch.randint(1, M + 1, (B,), device="cuda", generator=g)
        pad = torch.arange(M, device="cuda")[None, :] >= lens[:, None]
    elif pad_kind == "row_full":
        pad = torch.zeros(B, M, dtype=torch.bool, device="cuda")
        pad[0] = True
    return q, k, v, go, pad


def test_keep_mask_statistics_and_determinism():
    p, seed = 0.1, 1234567
    t, _ = _rp(p)
    keep = ops.dropout_keep_mask(2, 4, 256, 2048, p, seed)
    rate = keep.float().mean().item()
    n = keep.numel()
    sigma = ((t / 256) * (1 - t / 256) / n) ** 0.5
    assert abs(rate - (1 - t / 256)) < 5 * sigma, (rate, 1 - t / 256)
    # every row and every column sees the same rate; neighbours (in the 2x2 blocks that share a hash) are independent
    assert (keep.float().mean(-1) - (1 - t / 256)).abs().max().item() < 0.05
    assert (keep.float().mean(-2) - (1 - t / 256)).abs().max().item() < 0.12
    kf = keep.float() - (1 - t / 256)
    var = (t / 256) * (1 - t / 256)
    assert abs((kf[..., :, 0::2] * kf[..., :, 1::2]).mean().item()) < 0.02 * var + 5e-4
    assert abs((kf[..., 0::2, :] * kf[..., 1::2, :]).mean().item()) < 0.02 * var + 5e-4
    assert torch.equal(keep, ops.dropout_keep_mask(2, 4, 256, 2048, p, seed))
    other = ops.dropout_keep_mask(2, 4, 256, 2048, p, seed + 1)
    assert (keep != other).float().mean().item() > 0.1
    assert ops.dropout_keep_mask(1, 1, 8, 64, 0.5, 7).float().mean().item() == pytest.approx(0.5, abs=0.15)


CASES = [
    # B, N, M, H, dqk, dv, pad, causal, bcast, p
    (2, 256, 1024, 2, 128, 128, None, False, False, 0.1),
    (2, 200, 1000, 4, 64, 64, "ragged", False, True, 0.1),
    (1, 100, 300, 2, 32, 96, None, False, False, 0.25),
    (2, 96, 352, 2, 64, 64, "ragged", True, False, 0.1),
    (2, 130, 700, 2, 128, 64, "row_full", False, False, 0.5),
    (2, 512, 4096, 8, 128, 128, None, False, True, 0.1),
]


@pytest.mark.parametrize("case", CASES, ids=[f"B{c[0]}N{c[1]}M{c[2]}H{c[3]}d{c[4]}x{c[5]}{c[6] or ''}{'c' if c[7] else ''}{'b' if c[8] else ''}p{c[9]}" for c in CASES])
def test_dropout_forward_and_backward_match_reference_on_the_exported_mask(case):
    _check_against_reference(case, "auto")


@pytest.mark.parametrize("impl", ["auto", "tcgen05", "tcgen05_pair", "simt"])
def test_every_impl_takes_dropout(impl):
    """The dropout forward runs on the single-CTA tensor-core kernel whichever forward kernel ``impl`` names."""
    _check_against_reference(CASES[1], impl)


def _check_against_reference(case, impl):
    B, N, M, H, dqk, dv, pad_kind, causal, bcast, p = case
    q, k, v, go, pad = _inputs(B, N, M, H, dqk, dv, pad_kind, bcast, seed=5)
    scale = dqk ** -0.5
    seed = 424242
    _, rp = _rp(p)
    keep = ops.dropout_keep_mask(B, H, N, M, p, seed)

    qq, kk, vv = (t.detach().clone().requires_grad_() for t in (q, k, v))
    ops.backward_config["impl"] = "kernel"
    try:
        out = ops.attention(qq, kk, vv, H, scale, pad_mask=pad, causal=causal, impl=impl, dropout_p=p,
                            dropout_seed=seed)
        out.backward(go)
    finally:
        ops.backward_config["impl"] = "auto"

    r64, e16 = (_drop_ref(q, k, v, go, H, scale, pad, causal, dt, keep, rp) for dt in (torch.float64, torch.bfloat16))
    assert out.shape == r64[0].shape and torch.isfinite(out).all()
    bound, eager_err, ref_max = derived_bound(r64[0], e16[0])
    bound = max(bound, FLOOR * ref_max)
    err = (out.double() - r64[0]).abs().max().item()
    print(f"[dropout parity] {case} {impl} out: err {err:.3e} bound {bound:.3e} (eager {eager_err:.3e}, "
          f"max|ref| {ref_max:.3e})")
    assert err <= bound, f"out: err {err:.3e} > bound {bound:.3e}"
    mags = grad_magnitudes(q, k, v, go, H, scale, pad, causal, keep, rp)
    assert_grad_set((qq.grad, kk.grad, vv.grad), r64[1:], e16[1:], mags, q.dtype, f"dropout {case} {impl}")


def test_module_dropout_train_and_eval():
    """MultiHeadAttention with dropout=0.1: eval == no dropout; train is reproducible under torch.manual_seed, differs from
    eval, is unbiased on average, and backpropagates through the kernels."""
    torch.manual_seed(0)
    mha = modules.MultiHeadAttention(num_heads=4, num_q_input_channels=256, num_kv_input_channels=256, dropout=0.1)
    mha = mha.cuda().to(torch.bfloat16)
    x_q = torch.randn(2, 128, 256, device="cuda", dtype=torch.bfloat16)
    x_kv = torch.randn(2, 640, 256, device="cuda", dtype=torch.bfloat16)
    mha.eval()
    with torch.no_grad():
        ref = mha(x_q, x_kv).last_hidden_state
    mha.train()
    torch.manual_seed(11)
    a = mha(x_q, x_kv).last_hidden_state
    torch.manual_seed(11)
    b = mha(x_q, x_kv).last_hidden_state
    assert torch.equal(a, b)
    assert (a.float() - ref.float()).abs().max().item() > 1e-3
    acc = torch.zeros_like(ref, dtype=torch.float32)
    n = 24
    with torch.no_grad():
        for i in range(n):
            torch.manual_seed(100 + i)
            acc += mha(x_q, x_kv).last_hidden_state.float()
    bias = (acc / n - ref.float()).abs().mean().item()
    spread = (a.float() - ref.float()).abs().mean().item()
    print(f"[dropout module] mean |E[train] - eval| {bias:.3e} vs single-sample spread {spread:.3e}")
    assert bias < 0.45 * spread  # averaging 24 masks shrinks the deviation ~ 1/sqrt(24)
    ops.backward_config["impl"] = "kernel"
    try:
        xq = x_q.clone().requires_grad_()
        out = mha(xq, x_kv).last_hidden_state
        out.float().square().mean().backward()
    finally:
        ops.backward_config["impl"] = "auto"
    assert torch.isfinite(xq.grad).all() and xq.grad.abs().max().item() > 0
    assert all(torch.isfinite(p_.grad).all() for p_ in mha.parameters() if p_.grad is not None)


def test_device_mask_equals_the_numpy_oracle_bit_for_bit():
    """Integer path: the device generator (drop_bits / drop_keep in csrc/pcv_attn_bwd.cu, exported by
    pcv_attn_dropout_mask) against its numpy restatement oracle/dropout_oracle.py — exact equality."""
    import numpy as np

    from oracle import dropout_oracle as D

    for (B, H, N, M, p, seed) in [(2, 3, 70, 130, 0.1, 1), (1, 2, 33, 257, 0.5, 0xFFFFFFFFFFFF), (1, 1, 128, 512, 0.25, 424242),
                                  (2, 1, 5, 7, 0.9, (1 << 62) - 3)]:
        dev = ops.dropout_keep_mask(B, H, N, M, p, seed).cpu().numpy()
        ref = D.keep_mask(B, H, N, M, p, seed)
        assert np.array_equal(dev, ref), (B, H, N, M, p, seed, int((dev != ref).sum()))
