"""-m gpu: the CTA-pair kernel (impl "tcgen05_pair") and the single-CTA kernel at the headline head geometry (dh 128,
N 512, M 65536, several hundred key tiles per CTA), gated per row against fp64 with the derived bound and against each
other; and the pair plan never has more pairs than the device can hold at once.  With M >> N the causal mask hides no
key of this shape: the causal cases check that the causal path gives the unmasked result."""
import pytest
import torch

from gpu_util import assert_parity

pytestmark = pytest.mark.gpu

DTYPE = {"bf16": torch.bfloat16, "fp16": torch.float16}
EPS = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}  # unit roundoff of the 16-bit output
B, N, M, H, DH = 2, 512, 65536, 8, 128


def test_pair_plan_fits_on_the_device():
    """Both CTAs of a 2-CTA cluster sit in one GPC: the plan's pair count is SMs / 2 capped at the clusters that fit, so
    no pair waits for another to finish (a second wave)."""
    from perceiver_io_b200 import _lib, ops

    workers, fit = _lib.debug_pair_workers()
    sms = ops.device_info()["num_sms"]
    print(f"{sms} SMs, {fit} 2-CTA clusters fit, {workers} CTA pairs in the plan")
    assert fit >= 1 and workers == min(sms // 2, fit)


@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("masked", [False, True], ids=["nopad", "pad"])
@pytest.mark.parametrize("dt", list(DTYPE))
def test_pair_and_single_cta_kernels_match_fp64_and_each_other(dt, masked, causal):
    from perceiver_io_b200 import ops

    dtype, scale = DTYPE[dt], DH ** -0.5
    g = torch.Generator(device="cuda").manual_seed(5)
    q = torch.randn(B, N, H * DH, generator=g, device="cuda").to(dtype)
    k = torch.randn(B, M, H * DH, generator=g, device="cuda").to(dtype)
    v = torch.randn(B, M, H * DH, generator=g, device="cuda").to(dtype)
    pad = None
    if masked:
        pad = torch.rand(B, M, generator=torch.Generator().manual_seed(6)) < 0.3
        pad[1, M // 2:] = True
    padc = None if pad is None else pad.cuda()
    name = f"{dt} {'pad' if masked else 'nopad'} {'causal' if causal else 'full'}"
    out = {}
    for impl in ("tcgen05", "tcgen05_pair"):
        out[impl] = ops.attention(q, k, v, H, scale, pad_mask=padc, causal=causal, impl=impl)
        assert_parity(out[impl], q, k, v, H, scale, pad, causal, what=f"{impl} {name}", per_row=True)

    # The two plans split the key range at other tiles, so their fp32 merges run in another order and each rounds the
    # same row to 16 bits on its own: at most one rounding step apart (2u |x|).
    a, s = out["tcgen05_pair"].double(), out["tcgen05"].double()
    diff = (a - s).abs()
    lim = 2.0 * EPS[dt] * torch.maximum(a.abs(), s.abs())
    print(f"[pair vs single] {name}: max diff {diff.max().item():.3e}, {(diff > 0).double().mean().item():.2e} of the "
          f"elements differ, worst diff / one rounding step {(diff / lim.clamp_min(1e-30)).max().item():.3f}")
    assert (diff <= lim).all(), f"{name}: the pair and single-CTA kernels differ by more than one 16-bit rounding step"
