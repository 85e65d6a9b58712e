"""-m gpu: the one-pass dropout forward (attn_fwd_drop_kernel, ops.attention_partial with dropout_p) and the backward
shim with dropout, at head dims above 128 or not multiples of 8.

- The kernel leaves the softmax statistics alone: part_m / part_l equal the dropout-free kernel's bit for bit.
- The mask it applies is the exported one: with q = 0 every score is 0, so with v = e_(j mod dv) part_o counts the kept
  keys per channel.
- Forward and gradients through ops.attention meet the gates of test_gpu_dropout.py on the exported mask."""
import pytest
import torch

from fwd_variants import BF16, SCHEDULE_SHAPES, VARIANT_CASES, case_id, check_schedule, workers_for
from gpu_util import assert_grad_set, derived_bound, grad_magnitudes
from perceiver_io_b200 import adapter, modules, ops
from test_gpu_dropout import FLOOR, _drop_ref, _inputs, _rp

pytestmark = pytest.mark.gpu

SEED = 0x5EED0F1A2B
NONPAIR = [c for c in VARIANT_CASES if not c[3]]


def _dtype(dt):
    return torch.bfloat16 if dt == BF16 else torch.float16


def _operands(B, H, N, M, dqk, dv, dt, seed=1, pad=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, N, H * dqk, device="cuda", generator=g).to(_dtype(dt))
    k = torch.randn(B, M, H * dqk, device="cuda", generator=g).to(_dtype(dt))
    v = torch.randn(B, M, H * dv, device="cuda", generator=g).to(_dtype(dt))
    pad_mask = None
    if pad:
        pad_mask = torch.zeros(B, M, dtype=torch.bool, device="cuda")
        pad_mask[0, M - M // 3:] = True
    return q, k, v, pad_mask


def _stats_equal(q, k, v, H, pad, causal=False, p=0.1):
    scale = (q.shape[-1] // H) ** -0.5
    _, m0, l0 = ops.attention_partial(q, k, v, H, scale, pad_mask=pad, causal=causal, impl="tcgen05")
    _, m1, l1 = ops.attention_partial(q, k, v, H, scale, pad_mask=pad, causal=causal, dropout_p=p, dropout_seed=SEED)
    assert torch.equal(m0, m1), (m0 - m1).abs().max().item()
    assert torch.equal(l0, l1), (l0 - l1).abs().max().item()


@pytest.mark.parametrize("case", NONPAIR, ids=case_id)
def test_statistics_are_those_of_the_dropout_free_kernel(case):
    dqk, dv, dt, _ = case
    q, k, v, pad = _operands(2, 2, 200, 700, dqk, dv, dt)
    _stats_equal(q, k, v, 2, pad)
    _stats_equal(q, k, v, 2, None, causal=True, p=0.5)


@pytest.mark.parametrize("shape_name", ["ring", "whole"])
@pytest.mark.parametrize("case", [(40, 120, BF16, False), (136, 120, BF16, False), (392, 56, BF16, False)], ids=case_id)
def test_statistics_untouched_in_the_split_and_whole_unit_plans(case, shape_name):
    dqk, dv, dt, _ = case
    print(check_schedule(shape_name, case, workers_for(torch.cuda.get_device_properties(0).multi_processor_count, False)))
    B, H, N, M = SCHEDULE_SHAPES[shape_name]
    q, k, v, pad = _operands(B, H, N, M, dqk, dv, dt)
    _stats_equal(q, k, v, H, pad)


def _count_check(B, H, N, M, dqk, dv, dt, p):
    """q = 0: every score is 0, so m = 0 and l = M exactly.  v = e_(j mod dv): part_o[b, h, n, c] = r * (number of kept
    keys j = c mod dv), one fp32 rounding of an exact count (the split plan adds its slots: a few roundings)."""
    dtype = _dtype(dt)
    q = torch.zeros(1, N, H * dqk, device="cuda", dtype=dtype)
    k = torch.randn(B, M, H * dqk, device="cuda", dtype=dtype)
    j = torch.arange(M, device="cuda")
    vh = torch.nn.functional.one_hot(j % dv, dv).to(dtype)                       # (M, dv)
    v = vh[None, :, None, :].expand(B, M, H, dv).reshape(B, M, H * dv).contiguous()
    po, pm, pl = ops.attention_partial(q, k, v, H, dqk ** -0.5, dropout_p=p, dropout_seed=SEED)
    assert (pm == 0).all() and (pl == M).all()
    keep = ops.dropout_keep_mask(B, H, N, M, p, SEED).float()
    Mp = (M + dv - 1) // dv * dv
    counts = torch.nn.functional.pad(keep, (0, Mp - M)).reshape(B, H, N, Mp // dv, dv).sum(-2)
    want = counts * torch.tensor(_rp(p)[1], dtype=torch.float32)
    zero = counts == 0
    assert (po[zero] == 0).all()
    rel = ((po - want).abs() / want.clamp_min(1)).max().item()
    print(f"[mask count] B{B} H{H} N{N} M{M} qk{dqk} v{dv} {dt}: {int(zero.sum())} zero counts, max rel err {rel:.2e}")
    assert rel <= 1e-6


@pytest.mark.parametrize("case", NONPAIR + [(72, 512, BF16, False), (456, 320, "fp16", False)], ids=case_id)
def test_applied_mask_is_the_exported_mask(case):
    dqk, dv, dt, _ = case
    _count_check(2, 2, 130, 1000, dqk, dv, dt, 0.25)


def test_applied_mask_is_the_exported_mask_in_the_split_plan():
    B, H, N, M = SCHEDULE_SHAPES["ring"]
    _count_check(B, H, N, M, 264, 184, BF16, 0.1)


PARITY = [
    # B, N, M, H, dqk, dv, pad, causal, bcast, p, dtype
    (2, 256, 600, 8, 32, 160, "ragged", False, True, 0.1, torch.bfloat16),      # masked-LM encoder cross-attention
    (2, 64, 784, 1, 131, 131, "ragged", False, True, 0.1, torch.bfloat16),      # image classifier: odd dims, padded
    (2, 200, 456, 2, 256, 256, "ragged", True, False, 0.1, torch.bfloat16),
    (1, 128, 500, 1, 322, 322, None, False, False, 0.1, torch.bfloat16),
    (1, 100, 400, 2, 512, 512, "row_full", False, False, 0.5, torch.bfloat16),
    (2, 150, 333, 2, 200, 200, "ragged", False, False, 0.1, torch.float16),
    (1, 120, 40000, 1, 192, 192, None, False, False, 0.1, torch.bfloat16),      # split (stream-K) plan
]


def _pid(c):
    return f"B{c[0]}N{c[1]}M{c[2]}H{c[3]}d{c[4]}x{c[5]}{c[6] or ''}{'c' if c[7] else ''}{'b' if c[8] else ''}p{c[9]}" + (
        "fp16" if c[10] == torch.float16 else "")


@pytest.mark.parametrize("case", PARITY, ids=_pid)
def test_one_pass_forward_and_gradients_match_the_reference_on_the_exported_mask(case, monkeypatch):
    B, N, M, H, dqk, dv, pad_kind, causal, bcast, p, dtype = case
    q, k, v, go, pad = _inputs(B, N, M, H, dqk, dv, pad_kind, bcast, seed=7, dtype=dtype)
    scale = dqk ** -0.5
    keep = ops.dropout_keep_mask(B, H, N, M, p, SEED)
    _, rp = _rp(p)
    partial, drops = ops.attention_partial, []

    def recording_partial(*args, **kwargs):
        drops.append(kwargs.get("dropout_p", 0.0))
        return partial(*args, **kwargs)

    monkeypatch.setattr(ops, "attention_partial", recording_partial)
    qq, kk, vv = (t.detach().clone().requires_grad_() for t in (q, k, v))
    out = ops.attention(qq, kk, vv, H, scale, pad_mask=pad, causal=causal, dropout_p=p, dropout_seed=SEED)
    assert drops == [p]  # the one-pass route: one partial forward, with the mask applied
    out.backward(go)

    r64, eager = (_drop_ref(q, k, v, go, H, scale, pad, causal, dt, keep, rp) for dt in (torch.float64, dtype))
    assert out.shape == r64[0].shape and torch.isfinite(out).all()
    bound, eager_err, ref_max = derived_bound(r64[0], eager[0])
    bound = max(bound, FLOOR * ref_max)
    err = (out.double() - r64[0]).abs().max().item()
    print(f"[bighead dropout parity] {_pid(case)} out: err {err:.3e} bound {bound:.3e} "
          f"(eager {eager_err:.3e}, max|ref| {ref_max:.3e})")
    assert err <= bound, f"out: err {err:.3e} > bound {bound:.3e}"
    mags = grad_magnitudes(q, k, v, go, H, scale, pad, causal, keep, rp)
    assert_grad_set((qq.grad, kk.grad, vv.grad), r64[1:], eager[1:], mags, dtype, f"bighead dropout {_pid(case)}")


def test_head_dims_beyond_the_forward_kernel_stay_unsupported():
    q, k, v, _ = _operands(2, 1, 64, 256, 768, 768, BF16, pad=False)
    with pytest.raises(NotImplementedError, match="dropout"):
        ops.attention(q, k, v, 1, 768 ** -0.5, dropout_p=0.1, dropout_seed=1)


@pytest.mark.parametrize("B, H, N, M, p, seed", [(2, 3, 70, 1000, 0.1, 1), (1, 8, 256, 2048, 0.5, SEED)])
def test_range_export_is_a_slice_of_the_full_mask_and_of_the_oracle(B, H, N, M, p, seed):
    import numpy as np

    from oracle import dropout_oracle as D

    full = ops.dropout_keep_mask(B, H, N, M, p, seed)
    ref = D.keep_mask(B, H, N, M, p, seed)
    for k0, k1 in [(0, M), (0, 1), (1, 2), (127, 385), (M - 3, M), (333, 334), (512, M)]:
        part = ops.dropout_keep_mask(B, H, N, M, p, seed, key_begin=k0, key_end=k1)
        assert part.shape == (B, H, N, k1 - k0)
        assert torch.equal(part, full[..., k0:k1]), (k0, k1)
        assert np.array_equal(part.cpu().numpy(), ref[..., k0:k1]), (k0, k1)


class _Identity(adapter.InputAdapter):
    def forward(self, x):
        return x


def _mlm_encoder():
    """The masked-LM encoder (8 heads, qk 256 / v 1280 channels: head dims 32 / 160), one self-attention layer."""
    ad = adapter.TokenInputAdapter(vocab_size=262, max_seq_len=512, num_input_channels=768)
    return modules.PerceiverEncoder(ad, num_latents=256, num_latent_channels=1280, num_cross_attention_heads=8,
                                    num_cross_attention_qk_channels=256, num_cross_attention_v_channels=1280,
                                    num_self_attention_heads=8, num_self_attention_qk_channels=256,
                                    num_self_attention_v_channels=1280, num_self_attention_layers_per_block=1,
                                    dropout=0.1)


def _mnist_encoder():
    """The image classifier's encoder (one cross-attention head of 131 channels), one self-attention layer."""
    return modules.PerceiverEncoder(_Identity(131), num_latents=32, num_latent_channels=128, num_cross_attention_heads=1,
                                    num_cross_attention_qk_channels=131, num_cross_attention_v_channels=131,
                                    num_self_attention_heads=4, num_self_attention_layers_per_block=1, dropout=0.1)


def _set_dropout(module, p):
    for m in module.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = p


@pytest.mark.parametrize("name", ["mlm", "mnist"])
def test_encoder_trains_with_dropout(name, monkeypatch):
    """One training step with dropout 0.1 through the one-pass forward and the backward shim: finite gradients,
    reproducible under torch.manual_seed; eval equals the dropout-free output; the core output of the encoder
    cross-attention (the first ops.attention call of a forward; linear in the mask) averaged over 24 masks is unbiased."""
    torch.manual_seed(0)
    if name == "mlm":
        enc = _mlm_encoder()
        x = torch.randint(0, 262, (2, 512), device="cuda")
        pad = torch.zeros(2, 512, dtype=torch.bool, device="cuda")
        pad[1, 300:] = True
    else:
        enc = _mnist_encoder()
        x = torch.randn(2, 784, 131, device="cuda", dtype=torch.bfloat16)
        pad = None
    enc = enc.cuda().to(torch.bfloat16)
    seen = []
    attention = ops.attention

    def recording_attention(*args, **kwargs):
        out = attention(*args, **kwargs)
        seen.append(out.detach().float())
        return out

    monkeypatch.setattr(ops, "attention", recording_attention)

    enc.eval()
    with torch.no_grad():
        seen.clear()
        ref = enc(x, pad_mask=pad).float()
        ref_mha = seen[0]
        enc.train()
        _set_dropout(enc, 0.0)
        assert torch.equal(ref, enc(x, pad_mask=pad).float())  # eval == the dropout-free training forward
        _set_dropout(enc, 0.1)

    def step(seed):
        enc.zero_grad(set_to_none=True)
        torch.manual_seed(seed)
        out = enc(x, pad_mask=pad)
        out.float().square().mean().backward()
        return out.detach(), [p_.grad.clone() for p_ in enc.parameters() if p_.grad is not None]

    a, ga = step(11)
    seen.clear()
    b, gb = step(11)
    train_mha = seen[0]
    assert ga and all(torch.isfinite(g).all() for g in ga)
    assert torch.equal(a, b) and all(torch.equal(g, h) for g, h in zip(ga, gb))
    assert (a.float() - ref).abs().max().item() > 1e-3
    spread = (train_mha - ref_mha).abs().mean().item()
    acc = torch.zeros_like(ref_mha)
    n = 24
    with torch.no_grad():
        for i in range(n):
            torch.manual_seed(100 + i)
            seen.clear()
            enc(x, pad_mask=pad)
            acc += seen[0]
    bias = (acc / n - ref_mha).abs().mean().item()
    print(f"[bighead dropout module] {name}: mean |E[train] - eval| {bias:.3e} vs single-sample spread {spread:.3e}")
    assert bias < 0.45 * spread
