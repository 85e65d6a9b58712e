"""-m gpu: the ORIGINAL project (krasserm/perceiver-io) as the yardstick of whole models built from this package.

oracle/gen_live_golden.py ran the original modules on the CPU with the seeded weights and inputs of tests/live_cases.py
and stored, per case, a fixed sample of its fp64 output, the error of its own eager bf16 run over the whole output and
max|ref64| (tests/golden/live_cases.pt).  Here the package's modules, whose parameter names and shapes are those of the
original, get the same seeded weights and run on the GPU kernels; the stated gate
    max|ours - ref64| <= 2 * max|eager - ref64| + 1e-3 * max|ref64|        (BASELINE.md §3)
is applied on the stored sample.  The cross-attention case is also gated against the original's CPU fp32 forward."""
import copy

import pytest
import torch

import perceiver_io_b200 as core
from conftest import load_golden
from live_cases import cross_attention_case, csm_config, encoder_kwargs, grad_case, randomize
from perceiver_io_b200.adapter import InputAdapter

pytestmark = pytest.mark.gpu

GOLD = load_golden("live_cases.pt")


def _gate(ours, case, what):
    g = GOLD[case]
    got = ours.detach().double().cpu().reshape(-1)[g["idx"]]
    bound = 2.0 * g["eager_err"] + 1e-3 * g["ref_max"]
    err = (got - g["ref"]).abs().max().item()
    print(f"[parity] {what}: err {err:.3e} bound {bound:.3e} (eager {g['eager_err']:.3e}, max|ref| {g['ref_max']:.3e})")
    assert torch.isfinite(ours).all(), what
    assert err <= bound, f"{what}: err {err:.3e} > derived bound {bound:.3e}"
    return err, bound


def _bf16(model):
    import perceiver_io_b200 as P

    m = copy.deepcopy(model).bfloat16().cuda().eval()
    P.patch(m)  # no-op on the package's own modules (kept: the call must accept them)
    return m


def test_patch_on_reference_cross_attention_north_star_geometry():
    a = cross_attention_case()
    ref = core.CrossAttention(num_heads=a["H"], num_q_input_channels=a["D"], num_kv_input_channels=a["D"]).eval()
    randomize(ref, 1)
    with torch.no_grad():
        ref.attention.q_proj.weight.mul_(3.0)   # peaked rows as well
        mine = _bf16(ref)
        ours = mine(a["xq"].cuda(), a["xkv"].cuda(), pad_mask=a["pad"].cuda()).last_hidden_state
    assert "_pcv_kv_fold" in mine.__dict__, "CrossAttention did not take the fused K/V producer"
    _gate(ours, "cross", "CrossAttention vs the original fp64")
    _gate(ours, "cross_cpu32", "CrossAttention vs the original CPU fp32 forward")


class _PassThroughInput(InputAdapter):
    def forward(self, x):
        return x


def test_patch_on_reference_perceiver_encoder():
    kw, (x, pad) = encoder_kwargs()
    enc = core.PerceiverEncoder(_PassThroughInput(kw.pop("C")), **kw).eval()
    randomize(enc, 5)
    from perceiver_io_b200 import modules

    with torch.no_grad():
        mine = _bf16(enc)
        modules.kv_producer_config["min_rows_latent"] = 512   # exercise the one-GEMM QKV projection on the 640 latent rows
        try:
            ours = mine(x.cuda(), pad_mask=pad.cuda())
        finally:
            modules.kv_producer_config["min_rows_latent"] = 4096
    folded = [k for m in mine.modules() for k in m.__dict__ if k.startswith("_pcv_") and k.endswith("_fold")]
    assert "_pcv_qkv_fold" in folded and "_pcv_kv_fold" in folded and "_pcv_o_fold" in folded, folded
    _gate(ours, "encoder", "PerceiverEncoder (2 cross-attention + 4 self-attention layers) vs the original fp64")


def _csm(seed=7):
    m = core.CausalSequenceModel(core.CausalSequenceModelConfig(**csm_config()[0])).eval()
    randomize(m, seed, scale=0.04)
    return m


def test_patch_on_reference_causal_sequence_model_logits_and_cache():
    """Perceiver AR: left padding, right-aligned rotary over all head channels, causal prefix cross-attention,
    causal latent stack; then 3 cached decode steps must agree with the original's uncached fp64 logits (the original's
    own tests/kv_cache_test.py:191-234 pattern).  The model runs in fp32 under torch.autocast (Lightning's
    precision="bf16"), as the original's eager yardstick did."""
    _, (tokens, pad, n0, prefix) = csm_config()
    mine = _csm().cuda()
    t, p = tokens.cuda(), pad.cuda()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        full = mine(t[:, :n0], prefix_len=prefix, pad_mask=p[:, :n0], kv_cache=[])
        _gate(full.logits, "csm_full", "CausalSequenceModel: full forward logits")
        cache = full.kv_cache
        for s in range(3):
            step = mine(t[:, n0 + s: n0 + s + 1], prefix_len=prefix, pad_mask=p[:, : n0 + s + 1], kv_cache=cache)
            cache = step.kv_cache
            _gate(step.logits[:, 0], f"csm_step{s}", f"cached decode step {s}")
        assert cache[0][0].shape[1] == n0 + 3 and len(cache) == 1 + 3


def test_training_gradients_reach_q_and_k_projections_through_rotary():
    """Rotated q / k must stay in the autograd graph: CausalSequenceModel (fp32 weights, training mode, no dropout) on
    the GPU kernels against the original's own fp32 autograd: gradients of the cross-attention and first self-attention
    layer's q_proj / k_proj weights."""
    cfg, (tokens, pad, target, names) = grad_case()
    mine = core.CausalSequenceModel(core.CausalSequenceModelConfig(**cfg))
    randomize(mine, 11, scale=0.06)
    mine = mine.cuda().train()
    mine.zero_grad()
    logits = mine(tokens.cuda(), prefix_len=96, pad_mask=pad.cuda()).logits
    torch.nn.functional.cross_entropy(logits.reshape(-1, 64), target.cuda().reshape(-1)).backward()
    prm = dict(mine.named_parameters())
    for n in names:
        gm, gr = prm[n].grad, GOLD["grads"][n].double()
        assert gm is not None and gm.abs().max().item() > 0, f"no gradient reached {n}"
        err = (gm.double().cpu() - gr).abs().max().item()
        scale = gr.abs().max().item()
        # forward and backward run the bf16 tensor-core kernels: bf16 rounding of q/k/v/P (2^-8 each) is the only
        # difference to the original's fp32 autograd
        assert err <= 3e-2 * scale, f"{n}: grad err {err:.3e} vs max {scale:.3e}"


def test_cached_generation_under_autocast_promotes_like_torch_cat():
    """ADVICE r1 (medium): under torch.autocast the first cached step meets an fp32 empty cache and bf16 k/v; the
    reference's torch.cat promotes, kv_append must not raise."""
    import perceiver_io_b200 as P

    m = _csm(3).cuda()
    P.patch(m)
    t = torch.randint(0, 262, (1, 300)).cuda()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        full = m(t[:, :299], prefix_len=100, kv_cache=[])
        step = m(t[:, 299:], prefix_len=100, kv_cache=full.kv_cache)
    assert torch.isfinite(step.logits).all() and step.kv_cache[0][0].shape[1] == 300


def test_patched_reference_encoder_trains_with_attention_dropout():
    """A PerceiverEncoder built with dropout=0.1 in TRAINING mode: the attention-probability
    dropout of modules.py:161 runs inside the kernels (round 1 raised here).  Checks: reproducible under
    torch.manual_seed, differs from the eval forward, mean over seeds approaches it, loss.backward() reaches the input
    and every parameter through the backward kernels (impl='kernel' raises otherwise), eval is untouched."""
    from perceiver_io_b200 import ops

    torch.manual_seed(0)
    B, M, C, N, D = 2, 1500, 256, 192, 256
    enc = core.PerceiverEncoder(
        _PassThroughInput(C), num_latents=N, num_latent_channels=D, num_cross_attention_heads=4,
        num_cross_attention_layers=1, num_self_attention_heads=4, num_self_attention_layers_per_block=2,
        num_self_attention_blocks=1, dropout=0.1)
    randomize(enc, 21)
    mine = _bf16(enc)
    x = (torch.randn(B, M, C, generator=torch.Generator().manual_seed(22)) + 0.1).bfloat16().cuda()
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[1, 1200:] = True
    pad = pad.cuda()
    mine.eval()
    with torch.no_grad():
        ev = mine(x, pad_mask=pad).float()
    mine.train()
    with torch.no_grad():
        torch.manual_seed(5)
        a = mine(x, pad_mask=pad).float()
        torch.manual_seed(5)
        b = mine(x, pad_mask=pad).float()
        assert torch.equal(a, b)
        spread = (a - ev).abs().mean().item()
        assert spread > 1e-4
        acc = torch.zeros_like(ev)
        n = 16
        for i in range(n):
            torch.manual_seed(50 + i)
            acc += mine(x, pad_mask=pad).float()
        bias = (acc / n - ev).abs().mean().item()
        print(f"[dropout encoder] mean |E[train] - eval| {bias:.3e} vs single-sample spread {spread:.3e}")
        assert bias < 0.6 * spread
    ops.backward_config["impl"] = "kernel"
    try:
        xg = x.clone().requires_grad_()
        torch.manual_seed(7)
        out = mine(xg, pad_mask=pad)
        out.float().square().mean().backward()
    finally:
        ops.backward_config["impl"] = "auto"
    assert torch.isfinite(xg.grad).all() and xg.grad.abs().max().item() > 0
    missing = [n_ for n_, p_ in mine.named_parameters() if p_.requires_grad and (p_.grad is None or not torch.isfinite(p_.grad).all())]
    assert not missing, missing
    mine.eval()
    with torch.no_grad():
        assert torch.equal(mine(x, pad_mask=pad).float(), ev)
