"""-m gpu: the attention backward for head dims above 128 (up to 192): the dK/dV kernel's dV and dK passes and
bwd_dq_kernel on 64-key stages (ordered dQ partials), against float64 autograd of the reference algorithm with the
gates of test_gpu_bwd.py (gpu_util.assert_grads)."""
import pytest
import torch

from gpu_util import assert_grad_set, grad_magnitudes
from perceiver_io_b200 import _lib, ops
from test_gpu_bwd import _case, _check
from test_gpu_dropout import _drop_ref, _rp
from test_gpu_dropout_bighead import _mlm_encoder, _mnist_encoder

pytestmark = pytest.mark.gpu

# one head-dim pair per (NQB, NVB) with a third box, none a multiple of 64 where the box allows it
VARIANTS = [(32, 160), (72, 184), (160, 32), (184, 120), (136, 192)]
DTYPES = [torch.bfloat16, torch.float16]
MASKS = [  # pad kind, causal, batch-1 q
    (None, False, False),
    ("ragged", False, False),
    ("row_full", False, False),   # one batch row wholly padded, one padded from M/3 on
    (None, True, False),
    ("ragged", True, False),
    ("random", False, True),
]


def _dt(dtype):
    return "bf16" if dtype == torch.bfloat16 else "fp16"


@pytest.mark.parametrize("mask", MASKS, ids=lambda m: f"{m[0] or 'nopad'}{'-causal' if m[1] else ''}{'-bcast' if m[2] else ''}")
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("dims", VARIANTS, ids=lambda d: f"d{d[0]}x{d[1]}")
def test_wide_variants_match_autograd(dims, dtype, mask):
    dqk, dv = dims
    pad_kind, causal, bcast = mask
    q, k, v, go, pad = _case(2, 130, 300, 2, dqk, dv, pad_kind, causal, bcast, dtype=dtype, seed=dqk + dv)
    _check(q, k, v, go, 2, pad, causal, f"{dims} {_dt(dtype)} {mask}")


SHAPES = [  # B, N, M, H, dqk, dv, pad, causal, bcast
    (2, 1, 300, 2, 136, 136, "ragged", False, False),       # one query
    (2, 200, 300, 2, 136, 136, None, True, False),          # N not a multiple of 64
    (2, 130, 100, 2, 192, 192, "ragged", False, False),     # M < 128, not a multiple of 64
    (1, 100, 100, 1, 136, 192, None, True, False),          # causal self-attention, M < 128
    (2, 64, 190, 2, 32, 160, None, True, True),             # M = 2 x 64 + 62
    (1, 64, 20000, 1, 192, 192, None, False, False),        # many dQ splits
    (2, 64, 20000, 2, 136, 136, "ragged", False, True),     # 2 x 2 x 157 dK/dV tiles: the persistent loops wrap
    (3, 96, 5000, 1, 160, 32, "row_full", True, True),
]


@pytest.mark.parametrize("case", SHAPES, ids=[f"B{c[0]}N{c[1]}M{c[2]}H{c[3]}d{c[4]}x{c[5]}{c[6] or ''}{'c' if c[7] else ''}{'b' if c[8] else ''}" for c in SHAPES])
def test_wide_schedule_edges_match_autograd(case):
    B, N, M, H, dqk, dv, pad_kind, causal, bcast = case
    q, k, v, go, pad = _case(B, N, M, H, dqk, dv, pad_kind, causal, bcast, seed=N + M)
    _check(q, k, v, go, H, pad, causal, f"{case}")


SEED = 0x5EED0F1A2B


@pytest.mark.parametrize("case", [
    (2, 256, 600, 8, 32, 160, "ragged", False, True, torch.bfloat16),
    (2, 64, 784, 1, 136, 136, None, False, True, torch.bfloat16),
    (2, 100, 333, 2, 136, 136, "row_full", True, False, torch.float16),
], ids=["mlm32x160", "img136", "causal136fp16"])
def test_wide_dropout_gradients_match_the_reference_on_the_exported_mask(case):
    B, N, M, H, dqk, dv, pad_kind, causal, bcast, dtype = case
    p = 0.1
    q, k, v, go, pad = _case(B, N, M, H, dqk, dv, pad_kind, causal, bcast, dtype=dtype, seed=9)
    scale = dqk ** -0.5
    keep = ops.dropout_keep_mask(B, H, N, M, p, SEED)
    _, rp = _rp(p)
    po, pm, pl = ops.attention_partial(q, k, v, H, scale, pad_mask=pad, causal=causal, dropout_p=p, dropout_seed=SEED)
    out = ops.combine_partials(po[None], pm[None], pl[None], q.dtype)
    got = ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, pad_mask=pad, causal=causal, dropout_p=p,
                                 dropout_seed=SEED)

    r64, eager = (_drop_ref(q, k, v, go, H, scale, pad, causal, dt, keep, rp)[1:] for dt in (torch.float64, dtype))
    mags = grad_magnitudes(q, k, v, go, H, scale, pad, causal, keep, rp)
    assert_grad_set(got, r64, eager, mags, dtype, f"wide bwd dropout {case[4]}x{case[5]}")


def test_wide_dq_is_bitwise_reproducible():
    """Batch-1 q, B = 4 and several key splits: each dQ element sums 4 x splits partials, always in the same order."""
    q, k, v, go, pad = _case(4, 128, 12000, 2, 136, 136, "ragged", False, True, seed=21)
    scale = 136 ** -0.5
    po, pm, pl = ops.attention_partial(q, k, v, 2, scale, pad_mask=pad)
    out = ops.combine_partials(po[None], pm[None], pl[None], q.dtype)
    a = ops.attention_backward(q, k, v, out, go, pm, pl, 2, scale, pad_mask=pad)
    b = ops.attention_backward(q, k, v, out, go, pm, pl, 2, scale, pad_mask=pad)
    for x, y, name in zip(a, b, ("dq", "dk", "dv")):
        assert torch.equal(x, y), name


def _train_step(enc, x, pad, mode):
    ops.backward_config["impl"] = mode
    try:
        enc.zero_grad(set_to_none=True)
        torch.manual_seed(11)
        before = _lib.launch_count()
        out = enc(x, pad_mask=pad)
        out.float().square().mean().backward()
        torch.cuda.synchronize()
        return _lib.launch_count() - before, [(n, p_.grad.clone()) for n, p_ in enc.named_parameters() if p_.grad is not None]
    finally:
        ops.backward_config["impl"] = "auto"


@pytest.mark.parametrize("name", ["mlm", "mnist"])
def test_recipe_encoders_train_on_the_kernels(name):
    """backward_config['impl'] = 'kernel' succeeds for the masked-LM encoder (32 / 160) and the image classifier's
    encoder (131, padded to 136), launches more of our kernels than the shim, and every parameter gradient agrees with
    the shim's (the same dropout masks: same seed)."""
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
    enc = enc.cuda().to(torch.bfloat16).train()
    n_kernel, g_kernel = _train_step(enc, x, pad, "kernel")
    n_shim, g_shim = _train_step(enc, x, pad, "shim")
    assert n_kernel > n_shim
    worst = 0.0
    for (pname, a), (_, b) in zip(g_kernel, g_shim):
        assert torch.isfinite(a).all(), pname
        ref_max = b.float().abs().max().item()
        err = (a.float() - b.float()).abs().max().item()
        bound = 3e-2 * ref_max + 1e-6
        worst = max(worst, err / bound)
        assert err <= bound, (pname, err, ref_max)
    print(f"[wide bwd recipe] {name}: {len(g_kernel)} parameter gradients, worst kernel-vs-shim err/bound {worst:.3f}")


@pytest.mark.parametrize("d", [200, 322])
def test_kernel_mode_still_raises_above_192(d):
    q, k, v, go, _ = _case(2, 64, 256, 1, d, d, seed=3)
    qq, kk, vv = (t.detach().clone().requires_grad_() for t in (q, k, v))
    ops.backward_config["impl"] = "kernel"
    try:
        out = ops.attention(qq, kk, vv, 1, d ** -0.5)
        with pytest.raises(RuntimeError, match="does not cover"):
            out.backward(go)
    finally:
        ops.backward_config["impl"] = "auto"


def test_zz_watchdog_record_is_clear():
    """No barrier wait of any kernel timed out during this module (runs last in it)."""
    torch.cuda.synchronize()
    assert _lib.debug_read()[0] == 0, _lib.debug_read()
