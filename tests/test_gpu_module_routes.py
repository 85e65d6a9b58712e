"""GPU checks of the modules' autograd rule (``modules._needs_grad``): a call in which only biases require grad — BitFit-
style fine-tuning, weights frozen, inputs without grad — is differentiable on every route.  The inference kernels
(fused producer, FP8 cross-attention) must decline it, and every bias must receive its gradient."""
import copy

import pytest
import torch

import perceiver_io_b200 as P
from perceiver_io_b200 import modules
from test_gpu_ln_linear_bwd import _gate, _randomize_layer_norms, route  # noqa: F401 (route: fixture)

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _bias_only(module):
    for name, p in module.named_parameters():
        p.requires_grad_(name.endswith("bias"))
    return module


def _grads(module, inputs, go, seed=0):
    module.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    out = module(*inputs).last_hidden_state
    out.backward(go)
    return out.detach(), {n: p.grad.clone() for n, p in module.named_parameters() if p.grad is not None}


def _same_as_library(module, inputs, go, monkeypatch, bitwise):
    """Gradients with the fused producer enabled (training route off) against the run with it disabled: the names in
    ``bitwise`` bit for bit, the rest (downstream of grad_q's fp32 atomics) within one rounding step."""
    biases = {n for n, p in module.named_parameters() if p.requires_grad}
    _, fused = _grads(module, inputs, go)
    assert fused.keys() == biases, sorted(biases - fused.keys())
    monkeypatch.setitem(modules.kv_producer_config, "enabled", False)
    _, lib = _grads(module, inputs, go)
    monkeypatch.setitem(modules.kv_producer_config, "enabled", True)
    for name in biases:
        a, b = fused[name], lib[name]
        if name in bitwise:
            assert torch.equal(a, b), name
        else:
            step = torch.finfo(b.dtype).eps * b.abs().max().item()
            assert (a.double() - b.double()).abs().max().item() <= step, name


def _cross_attention():
    torch.manual_seed(0)
    B, N, M, D, C, H = 2, 512, 1024, 256, 512, 4
    layer = P.CrossAttention(num_heads=H, num_q_input_channels=D, num_kv_input_channels=C).to(DEV).bfloat16()
    _randomize_layer_norms(layer)
    x_q = torch.randn(1, N, D, device=DEV).bfloat16()
    x_kv = torch.randn(B, M, C, device=DEV).bfloat16()
    go = torch.randn(B, N, D, device=DEV).bfloat16()
    return _bias_only(layer), [x_q, x_kv], go


def test_cross_attention_bias_only_training(monkeypatch):
    layer, inputs, go = _cross_attention()
    monkeypatch.setitem(modules.kv_producer_config, "training", False)
    assert inputs[1].shape[0] * inputs[1].shape[1] >= modules.kv_producer_config["min_rows"]
    _same_as_library(layer.train(), inputs, go, monkeypatch,
                     bitwise={"kv_norm.bias", "attention.k_proj.bias", "attention.v_proj.bias", "attention.o_proj.bias"})


def test_cross_attention_bias_only_training_route(route):  # noqa: F811
    layer, inputs, go = _cross_attention()
    layer.train()
    route.set(True)
    _, on = _grads(layer, inputs, go)
    assert route.taken == ["_pcv_q_fold", "_pcv_kv_fold"], route.taken
    route.set(False)
    _, off = _grads(layer, inputs, go)
    assert route.taken == []
    _, ref = _grads(copy.deepcopy(layer).double(), [t.double() for t in inputs], go.double())
    assert on.keys() == off.keys() == ref.keys() == {n for n, p in layer.named_parameters() if p.requires_grad}
    for name in on:
        _gate(on[name], ref[name], off[name], f"bias-only CrossAttention {name}")


def test_fp8_cross_attention_declines_bias_only_grad(monkeypatch):
    layer, inputs, go = _cross_attention()
    layer.eval()
    out_bf16, want = _grads(layer, inputs, go)
    monkeypatch.setitem(modules.fp8_config, "enabled", True)
    out, got = _grads(layer, inputs, go)
    assert "_pcv_fp8_scales" not in layer.__dict__
    assert torch.equal(out, out_bf16)
    assert got.keys() == want.keys() == {n for n, p in layer.named_parameters() if p.requires_grad}


def test_self_attention_bias_only_training(monkeypatch):
    torch.manual_seed(1)
    B, N, D, H = 2, 2048, 256, 4
    layer = _bias_only(P.SelfAttention(num_heads=H, num_channels=D).to(DEV).bfloat16().train())
    _randomize_layer_norms(layer)
    x = torch.randn(B, N, D, device=DEV).bfloat16()
    go = torch.randn(B, N, D, device=DEV).bfloat16()
    monkeypatch.setitem(modules.kv_producer_config, "training", False)
    assert B * N >= modules.kv_producer_config["min_rows_latent"]
    _same_as_library(layer, [x], go, monkeypatch,
                     bitwise={"attention.k_proj.bias", "attention.v_proj.bias", "attention.o_proj.bias"})
