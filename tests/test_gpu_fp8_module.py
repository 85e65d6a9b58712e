"""The e4m3 producer (ops.kv_project_fp8, pcv_kv_project_fp8) and the FP8 route of CrossAttention.forward
(modules.fp8_config) on the GPU."""
import pytest
import torch
from torch import nn

import perceiver_io_b200 as P
from fp8_emulation import emulate
from perceiver_io_b200 import modules, ops
from perceiver_io_b200.patch import patch

pytestmark = pytest.mark.gpu


def _e4m3_ulp(x):
    """Spacing of e4m3 values at |x| (normal range; 2^-9 below it)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -6)))
    return torch.exp2(e - 3)


@pytest.mark.parametrize("B,M,C,H,dqk,dv", [(3, 1000, 512, 4, 64, 96), (2, 300, 256, 8, 32, 160)])
def test_producer_matches_torch_quantisation(B, M, C, H, dqk, dv):
    """k8 / V^T against torch quantisation of the 16-bit producer output with the same scales: at most one e4m3 ulp
    apart, on a small fraction of elements (the 16-bit output is itself rounded); M % 128 != 0, so 128-row tiles cross
    batch boundaries and V^T must land at the right (batch, key)."""
    torch.manual_seed(B + M)
    norm = nn.LayerNorm(C).cuda()
    kp, vp = nn.Linear(C, H * dqk).cuda(), nn.Linear(C, H * dv).cuda()
    with torch.no_grad():
        norm.weight.add_(0.3 * torch.randn(C, device="cuda"))
        norm.bias.add_(0.2 * torch.randn(C, device="cuda"))
    x = (torch.randn(B, M, C, device="cuda") * 3 + 1).bfloat16()
    kd = ops.fp8_descales(norm.weight, norm.bias, kp.weight, kp.bias, H)
    vd = ops.fp8_descales(norm.weight, norm.bias, vp.weight, vp.bias, H, per_channel=True)
    w_cat, col_st = ops.fold_ln_linear(norm.weight, norm.bias, [kp.weight, vp.weight], [kp.bias, vp.bias], torch.bfloat16)
    inv = torch.cat([(1.0 / kd).repeat_interleave(dqk), (1.0 / vd).reshape(-1)])
    with torch.no_grad():
        k8, vt8 = ops.kv_project_fp8(x, w_cat, col_st, inv, H * dqk, H * dv, H, eps=norm.eps)
        k16, v16 = ops.kv_project(x, w_cat, col_st, H * dqk, H * dv, eps=norm.eps)
    assert k8.shape == (B, M, H * dqk) and vt8.shape == (B, H, dv, (M + 15) // 16 * 16)
    for got, want in ((k8.float(), ops.fp8_quantize(k16, kd, H).float()),
                      (vt8[..., :M].float(), ops.fp8_transpose_v(ops.fp8_quantize(v16, vd, H), H)[..., :M].float())):
        diff = (got - want).abs()
        assert (diff <= _e4m3_ulp(torch.maximum(got.abs(), want.abs())) * 1.0001).all()
        assert (diff > 0).float().mean().item() < 0.05
        assert got.abs().max() <= 448.0


def _layer(D=512, H=4, seed=0):
    torch.manual_seed(seed)
    return P.CrossAttention(num_heads=H, num_q_input_channels=D, num_kv_input_channels=D).cuda().bfloat16().eval()


def _inputs(B=2, N=192, M=1000, D=512):
    g = torch.Generator(device="cuda").manual_seed(1)
    x_q = torch.randn(1, N, D, device="cuda", generator=g).bfloat16()
    x_kv = torch.randn(B, M, D, device="cuda", generator=g).bfloat16()
    pad = torch.zeros(B, M, dtype=torch.bool, device="cuda")
    pad[1, 700:] = True
    return x_q, x_kv, pad


def _run(layer, *args, fp8):
    modules.fp8_config["enabled"] = fp8
    try:
        with torch.no_grad():
            return layer(*args).last_hidden_state
    finally:
        modules.fp8_config["enabled"] = False


def test_module_fp8_route_is_the_fp8_pipeline_and_matches_the_emulation():
    layer = _layer()
    x_q, x_kv, pad = _inputs()
    out = _run(layer, x_q, x_kv, None, pad, fp8=True)
    attn, H = layer.attention, layer.attention.num_heads
    qd, kd, vd, inv_q, inv_kv = modules._fp8_scales(layer, torch.bfloat16)
    with torch.no_grad():
        wq, stq = ops.fold_ln_linear(layer.q_norm.weight, layer.q_norm.bias, [attn.q_proj.weight], [attn.q_proj.bias],
                                     torch.bfloat16)
        wkv, stkv = ops.fold_ln_linear(layer.kv_norm.weight, layer.kv_norm.bias, [attn.k_proj.weight, attn.v_proj.weight],
                                       [attn.k_proj.bias, attn.v_proj.bias], torch.bfloat16)
        q8, _ = ops.kv_project_fp8(x_q, wq, stq, inv_q, 512, 0, H)
        k8, vt8 = ops.kv_project_fp8(x_kv, wkv, stkv, inv_kv, 512, 512, H)
        o = ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, attn.dp_scale, pad_mask=pad)
        manual = attn.o_proj(o)
    assert torch.equal(out, manual)
    ref = emulate(q8, k8, vt8, qd, kd, vd, H, attn.dp_scale, pad, workers=ops.device_info()["num_sms"])
    got = o.double().view(2, 192, H, -1).permute(0, 2, 1, 3)
    assert ((got - ref["out"]).abs() <= 2.0 ** -6 * ref["pv_abs"]).all()
    # error of the whole FP8 module (weight-derived scales) against the bf16 route, printed for the record
    bf = _run(layer, x_q, x_kv, None, pad, fp8=False)
    print(f"module FP8 vs bf16: max |diff| / max |bf16| = {((out.float() - bf.float()).abs().max() / bf.float().abs().max()).item():.3e}")


def test_option_off_is_bitwise_unchanged():
    layer = _layer()
    x_q, x_kv, pad = _inputs()
    before = _run(layer, x_q, x_kv, None, pad, fp8=False)
    _run(layer, x_q, x_kv, None, pad, fp8=True)
    after = _run(layer, x_q, x_kv, None, pad, fp8=False)
    assert torch.equal(before, after)


def test_training_and_grad_calls_take_the_bf16_path():
    layer = _layer()
    x_q, x_kv, pad = _inputs()
    bf = _run(layer, x_q, x_kv, None, pad, fp8=False)
    bf_grad = layer(x_q, x_kv, pad_mask=pad).last_hidden_state  # the bf16 route under autograd
    layer.train()
    modules.fp8_config["enabled"] = True
    try:
        with torch.no_grad():
            train_out = layer(x_q, x_kv, pad_mask=pad).last_hidden_state
        layer.eval()
        grad_out = layer(x_q, x_kv, pad_mask=pad).last_hidden_state  # parameters require grad, grad enabled
    finally:
        modules.fp8_config["enabled"] = False
    assert torch.equal(train_out, bf)
    assert grad_out.requires_grad and torch.equal(grad_out.detach(), bf_grad.detach())


class CrossAttention(nn.Module):
    """Stand-in for a reference CrossAttention (same class name and attributes), rebound by patch()."""

    def __init__(self, ours):
        super().__init__()
        self.q_norm, self.kv_norm, self.attention = ours.q_norm, ours.kv_norm, ours.attention

    def forward(self, *args, **kwargs):
        raise AssertionError("patch() did not rebind forward")


def test_patched_reference_module_takes_the_fp8_route():
    ours = _layer()
    ref = CrossAttention(ours).eval()
    assert patch(nn.Sequential(ref)) == 0  # no MultiHeadAttention of the reference's own; CrossAttention rebound
    x_q, x_kv, pad = _inputs()
    assert torch.equal(_run(ref, x_q, x_kv, None, pad, fp8=True), _run(ours, x_q, x_kv, None, pad, fp8=True))
    assert not torch.equal(_run(ref, x_q, x_kv, None, pad, fp8=True), _run(ref, x_q, x_kv, None, pad, fp8=False))
