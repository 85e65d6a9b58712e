"""-m gpu: the tensor-core attention on an FP8 KV cache (attn_cached_kernel<BF16, true, false, NVB>,
csrc/pcv_attn_cached.cu) at its row, tile, split and mask edges, and the cached steps of 5 to 64 new tokens that reach
it through the model.
The matrix, the restated plan and the CPU emulation live in cached_fp8_variants.py (test_cached_fp8_cpu.py checks that
the matrix covers every instantiation and that the emulated arithmetic stays within half of the gate used here).

  - random operands: fp64 attention on the dequantised codes, gated row by row (assert_parity(per_row=True)) and per
    element (cached_fp8_variants.element_bound: gpu_util.decode_element_bound plus the P-rounding term);
  - exact probes (decode_variants.py's operands): the count probe (q = 0: RN16(S / L) of the integer sum and count of a
    row's live keys) and the needle probe (one key ~185 log2 units above the rest: RN16(v[needle]) when it is live);
  - two launches are bit-identical; at N = 4 the kernel and the streaming decode kernel agree within both gates."""
import copy
import math

import pytest
import torch

import cached_fp8_variants as CV
import decode_variants as DV
from gpu_util import UNIT_ROUNDOFF, assert_decode_elements, assert_parity, decode_element_bound

pytestmark = pytest.mark.gpu

CUDA = "cuda"
F8 = torch.float8_e4m3fn


def _ops():
    from perceiver_io_b200 import ops
    return ops


def _cached(q, k8, v8, kd, vd, H, scale, pad, causal):
    """pcv_attn_cached_fp8 for any N (ops.attention_decode_fp8 takes it from 5 rows on)."""
    import ctypes

    from perceiver_io_b200 import _lib

    ops = _ops()
    with torch.cuda.device(k8.device):
        p, f, keep = ops._fill_decode(q, k8, v8, H, scale, pad, causal, kd, vd)
        p.impl = _lib.PCV_IMPL_AUTO
        out = ops._new_output(p, q.dtype, k8.device)
        ws = ops._workspace(p, k8.device, "pcv_attn_cached_fp8", ctypes.byref(p))
        ops.check(_lib.lib().pcv_attn_cached_fp8(ctypes.byref(p), ctypes.byref(f), ops._stream()), "pcv_attn_cached_fp8")
        del ws, keep
    return out


def _assert_gates(got, q, kq, vq, H, scale, pad, causal, dtype, depth, what):
    """The derived gate row by row and the element-wise gate with the P-rounding term; returns the worst element's
    err / bound.  The row gate's floor is two 16-bit roundings of the row's scale: the kernel rounds P (relative to the
    running maximum, where eager rounds the normalised softmax) and the output, so on a row of few keys eager's error
    can be the smaller by chance."""
    u = UNIT_ROUNDOFF[dtype]
    assert_parity(got, q, kq, vq, H, scale, pad, causal, what=what, eager_dtype=dtype, per_row=True, floor=2 * u)
    bound, ref = CV.element_bound(q, kq, vq, H, scale, pad, causal, dtype, depth)
    ratio = (got.double() - ref).abs() / bound
    worst = ratio.max().item()
    print(f"[cached elems] {what}: worst err/bound {worst:.3f}")
    assert int((ratio > 1).sum().item()) == 0, f"{what}: {int((ratio > 1).sum().item())} elements over their bound"
    return worst


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _assert_bits(got, want, what):
    eq = (got.view(torch.int16) == want.view(torch.int16)) | ((got == 0) & (want == 0))
    if not bool(eq.all()):
        bad = (~eq).nonzero()
        b, n, c = (int(x) for x in bad[0])
        raise AssertionError(f"{what}: {bad.shape[0]} of {eq.numel()} outputs differ; first at (b={b}, n={n}, "
                             f"channel {c}): got {got[b, n, c].item()!r} want {want[b, n, c].item()!r}")


@pytest.mark.parametrize("case", CV.VARIANT_CASES, ids=CV.case_id)
def test_random_operands_at_the_edges(case):
    """N in {1, 5, 8, 63, 64} x M in {1, 63, 64, 65, N, SPLIT_M} x causal (where M >= N) / not, left padding on batch row 1 and a
    wholly padded batch row 2, against fp64 on the dequantised codes; every call twice, bit-identical."""
    dt, dqk, dv = case
    dtype = CV.DTYPE[dt]
    B, H, scale = CV.EDGE_B, CV.EDGE_H, 0.3
    worst = 0.0
    for N in CV.EDGE_N:
        for M in CV.edge_ms(N):
            q, k8, v8, kd, vd = CV.random_operands(B, B, N, M, H, dqk, dv, dt, seed=7 * N + M, device=CUDA)
            pad = CV.left_pad(B, M, CUDA)
            kq, vq = (_ops().fp8_dequantize(x, d, H, torch.float64) for x, d in ((k8, kd), (v8, vd)))
            depth = CV.serial_depth(CV.plan(B, H, M, dqk, dv, CV.device_sms()))
            for causal in ((False, True) if M >= N else (False,)):   # a causal step holds its own N rows: M >= N
                what = f"{CV.case_id(case)} N={N} M={M} causal={causal}"
                out = _cached(q, k8, v8, kd, vd, H, scale, pad, causal)
                assert _bits_equal(out, _cached(q, k8, v8, kd, vd, H, scale, pad, causal)), f"{what}: two calls differ"
                worst = max(worst, _assert_gates(out, q, kq, vq, H, scale, pad, causal, dtype, depth, what))
    print(f"[cached fp8] {CV.case_id(case)}: worst element err / gate {worst:.3f}")


def _probe_keys(B, H, N, M, dqk, dv):
    pl = CV.plan(B, H, M, dqk, dv, CV.device_sms())
    return CV.split_ranges(M, pl), CV.edge_keys(M, pl, N)


@pytest.mark.parametrize("case", CV.VARIANT_CASES, ids=CV.case_id)
@pytest.mark.parametrize("N,M", [(8, CV.SPLIT_M), (64, 65), (5, 64), (63, 2 * CV.SPLIT_M)])
@pytest.mark.parametrize("causal", [False, True])
def test_count_probe(case, N, M, causal):
    """q = 0: every output is RN16(S / L) of the integer sum and count of the row's live keys (all its keys when none
    is live), with V nonzero only at split, tile and causal edges and at padded keys."""
    dt, dqk, dv = case
    dtype = CV.DTYPE[dt]
    B, H = CV.EDGE_B, CV.EDGE_H
    _ranges, marks = _probe_keys(B, H, N, M, dqk, dv)
    pad = CV.left_pad(B, M, CUDA)
    q, k8, v8 = DV.count_operands(B, B, N, M, H, dqk, dv, marks, pad, True, dtype, seed=N + M, device=CUDA)
    kd, vd = torch.ones(H, device=CUDA), DV.v_descale(H, dv, CUDA)
    out = _cached(q, k8, v8, kd, vd, H, 1.0, pad, causal)
    in_range, live = DV.key_sets(B, N, M, pad, causal, device=CUDA)
    _assert_bits(out, DV.count_expect(v8.float(), H, in_range, live, dtype, vd),
                 f"count {CV.case_id(case)} N={N} M={M} causal={causal}")


@pytest.mark.parametrize("case", CV.VARIANT_CASES, ids=CV.case_id)
@pytest.mark.parametrize("N,M", [(8, CV.SPLIT_M), (64, 130)])
@pytest.mark.parametrize("causal", [False, True])
def test_needle_probe(case, N, M, causal):
    """One needle key per (b, h, n) on the split and tile edges, the causal diagonals (and the key past them) and the
    first and last padded key, in rounds until every candidate held one: found, the output is RN16(v[needle]); masked,
    the row is the count probe's.  Each row sees its own q channel, so a case takes at most dqk rows."""
    dt, dqk, dv = case
    N = min(N, dqk)
    dtype = CV.DTYPE[dt]
    B, H = CV.EDGE_B, CV.EDGE_H
    _ranges, marks = _probe_keys(B, H, N, M, dqk, dv)
    pad = CV.left_pad(B, M, CUDA)
    in_range, live = DV.key_sets(B, N, M, pad, causal, device=CUDA)
    cands = []
    for b in range(B):
        c = set(marks) | {0, M - 1}
        if causal:
            c |= {M - N + n for n in range(N)} | {M - N + n + 1 for n in range(N - 1)}
        padded = pad[b].nonzero()
        if padded.numel():
            c |= {int(padded[0]), int(padded[-1])}
        cands.append(sorted(x for x in c if 0 <= x < M))
    kd, vd = torch.ones(H, device=CUDA), DV.v_descale(H, dv, CUDA)
    for r in range(DV.needle_rounds(cands, H, N)):
        nd = DV.needles(B, H, N, cands, r)
        q, k8, v8 = DV.needle_operands(B, B, N, M, H, dqk, dv, nd, True, dtype, seed=r + N, device=CUDA)
        out = _cached(q, k8, v8, kd, vd, H, DV.NEEDLE_SCALE, pad, causal)
        want = DV.needle_expect(v8.float(), H, in_range, live, nd, dtype, vd)
        _assert_bits(out, want, f"needle {CV.case_id(case)} N={N} M={M} causal={causal} round {r}")


@pytest.mark.parametrize("dt", CV.DTYPES)
@pytest.mark.parametrize("M", [4, 300, 5000])
def test_agrees_with_the_decode_kernel_at_four_rows(dt, M):
    """At N = 4 both kernels run on the same e4m3 cache: each within its own element-wise gate, and their difference
    within the sum of the two gates."""
    dqk = dv = 96
    B, H, N, scale, causal = 3, 2, 4, 0.3, True
    dtype = CV.DTYPE[dt]
    q, k8, v8, kd, vd = CV.random_operands(B, B, N, M, H, dqk, dv, dt, seed=M, device=CUDA)
    pad = CV.left_pad(B, M, CUDA)
    kq, vq = (_ops().fp8_dequantize(x, d, H, torch.float64) for x, d in ((k8, kd), (v8, vd)))
    a = _cached(q, k8, v8, kd, vd, H, scale, pad, causal)
    b = _ops().attention_decode_fp8(q, k8, v8, kd, vd, H, scale, pad_mask=pad, causal=causal)
    da = CV.serial_depth(CV.plan(B, H, M, dqk, dv, CV.device_sms()))
    nsplit, kps = DV.choose_split(B, H, M, DV.device_sms())
    lpk = DV.lanes_per_key(dqk, dv, True)
    db = DV.serial_depth(kps, nsplit, lpk, 4, True)
    _assert_gates(a, q, kq, vq, H, scale, pad, causal, dtype, da, f"cached N=4 M={M}")
    assert_decode_elements(b, q, kq, vq, H, scale, pad, causal, dtype, db, f"decode N=4 M={M}")
    ga, _ = CV.element_bound(q, kq, vq, H, scale, pad, causal, dtype, da)
    gb, _ = decode_element_bound(q, kq, vq, H, scale, pad, causal, dtype, db)
    assert bool(((a.double() - b.double()).abs() <= ga + gb).all())


@pytest.mark.parametrize("dt", CV.DTYPES)
def test_reference_rotary_keys_reach_the_kernel(dt):
    """Keys rotated e4m3 to e4m3 over the whole cache (ops.rotary_fp8, the reference-style rotary object's route) are
    plain e4m3 rows with the per-head k_descale: a 16-row step on them matches fp64 on the rotated codes."""
    ops = _ops()
    B, H, N, M, dqk, dv, scale = 2, 4, 16, 700, 64, 64, 0.125
    dtype = CV.DTYPE[dt]
    q, k8, v8, kd, vd = CV.random_operands(B, B, N, M, H, dqk, dv, dt, seed=11, device=CUDA)
    inv_freq = 1.0 / (10000 ** (torch.arange(0, 32, 2, device=CUDA).float() / 32))
    angles = (torch.arange(M, device=CUDA).float()[:, None] * inv_freq[None]).repeat_interleave(2, dim=-1)[None]
    kr8 = ops.rotary_fp8(k8, H, angles, False, kd)
    assert kr8.dtype == F8 and kr8.shape == k8.shape
    pad = CV.left_pad(B, M, CUDA)
    out = ops.attention_decode_fp8(q, kr8, v8, kd, vd, H, scale, pad_mask=pad, causal=True)
    kq, vq = ops.fp8_dequantize(kr8, kd, H, torch.float64), ops.fp8_dequantize(v8, vd, H, torch.float64)
    depth = CV.serial_depth(CV.plan(B, H, M, dqk, dv, CV.device_sms()))
    _assert_gates(out, q, kq, vq, H, scale, pad, True, dtype, depth, f"rotary_fp8 keys {dt}")


def test_generation_loop_with_multi_token_steps(monkeypatch):
    """A CausalSequenceModel with FP8 caches: left padding, cached steps of 1, 5, 16, 64 and 65 new tokens, both the
    token window and the latent window sliding, and a beam reorder; rotary keys from the e4m3 shadow.  Every step's
    logits are gated against an fp64 copy of the model on the route's codes (the gate of
    test_gpu_fp8_kv_cache.py's loop), and a spy checks the route: ops.fp8_dequantize is never called for steps of up
    to 64 tokens and is called for the 65-token step."""
    import perceiver_io_b200 as P
    from perceiver_io_b200 import modules, ops
    from test_gpu_fp8_kv_cache import _Fp64Attend, _owners

    torch.manual_seed(5)
    cfg = P.CausalSequenceModelConfig(vocab_size=97, max_seq_len=256, max_latents=96, num_channels=128, num_heads=4,
                                      num_self_attention_layers=2, num_self_attention_rotary_layers=1,
                                      cross_attention_dropout=0.0, output_norm=True, abs_pos_emb=False, init_scale=0.1)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.LayerNorm):
                m.weight.add_(0.3 * torch.randn_like(m.weight))
                m.bias.add_(0.3 * torch.randn_like(m.bias))
    model64 = copy.deepcopy(model).double()
    fp64 = _Fp64Attend(model64, _owners(model64))
    widths = [1, 5, 1, 16, 64, 1, 65, 1, 5, 1]
    reorder_step = 5
    B, n0, prefix = 2, 160, 120
    tokens0 = torch.randint(0, 97, (B, n0 + sum(widths))).cuda()
    pad0 = torch.zeros(B, tokens0.shape[1], dtype=torch.bool, device="cuda")
    pad0[1, :9] = True
    calls = {"n": 0}
    real = ops.fp8_dequantize

    def spy(*a, **k):
        calls["n"] += 1
        return real(*a, **k)

    monkeypatch.setattr(ops, "fp8_dequantize", spy)

    def run(arm):
        tokens, pad = tokens0.clone(), pad0.clone()
        out, ref, routes = [], [], []

        def call(x, plen, pm, kv):
            if arm == "fp64":
                with monkeypatch.context() as mp:
                    mp.setattr(modules, "attend", fp64)
                    mp.setattr(modules, "_kv8_route", lambda *a: None)
                    fp64.mode = "own"
                    return model64(x, prefix_len=plen, pad_mask=pm, kv_cache=kv)
            modules.fp8_config["kv_cache"] = arm == "fp8"
            calls["n"] = 0
            try:
                o = model(x, prefix_len=plen, pad_mask=pm, kv_cache=kv)
            finally:
                modules.fp8_config["kv_cache"] = False
            routes.append(calls["n"])
            if arm == "fp8":
                with monkeypatch.context() as mp:
                    mp.setattr(modules, "attend", fp64)
                    mp.setattr(modules, "_kv8_route", lambda *a: None)
                    if len(kv) == 0:
                        fp64.mode = "own"
                        r = model64(x, prefix_len=plen, pad_mask=pm)
                    else:
                        fp64.mode = "codes"
                        fp64.route_cache = o.kv_cache
                        fp64.route_scales = [ow.__dict__["_pcv_kv8_scales"][1] for ow in _owners(model)]
                        r = model64(x, prefix_len=plen, pad_mask=pm, kv_cache=kv)
                ref.append(r.logits[:, -1].double())
            return o

        with torch.no_grad():
            o = call(tokens[:, :n0], prefix, pad[:, :n0], [])
            out.append(o.logits[:, -1].double())
            cache, pos = o.kv_cache, n0
            for s, m in enumerate(widths):
                n = cache[0][0].shape[1] + m
                if n > cfg.max_seq_len:
                    d = n - cfg.max_seq_len
                    cache = [(cache[0][0][:, d:], cache[0][1][:, d:])] + cache[1:]
                    n -= d
                nlat = cache[1][0].shape[1] + m
                if nlat > cfg.max_latents:
                    d = nlat - cfg.max_latents
                    cache = cache[:1] + [(k[:, d:], v[:, d:]) for k, v in cache[1:]]
                    nlat -= d
                plen = n - nlat
                if s == reorder_step:
                    idx = torch.tensor([1, 0], device="cuda")
                    cache = [(k.index_select(0, idx), v.index_select(0, idx)) for k, v in cache]
                    tokens, pad = tokens[idx], pad[idx]
                o = call(tokens[:, pos:pos + m], plen, pad[:, pos + m - n:pos + m], cache)
                out.append(o.logits[:, -1].double())
                cache, pos = o.kv_cache, pos + m
        return torch.stack(out), (torch.stack(ref) if ref else None), routes

    a, a_ref, routes = run("fp8")
    b, _, _ = run("bf16")
    truth, _, _ = run("fp64")
    for s, m in enumerate(widths):
        if m <= 64:
            assert routes[s + 1] == 0, f"step {s} ({m} tokens) dequantised the cache"
        else:
            assert routes[s + 1] > 0, f"step {s} ({m} tokens) did not take the dequantising path"
    assert torch.isfinite(a).all()
    scale = truth.abs().max().item()
    err_a = (a - a_ref).abs().max().item()
    err_b = (b - truth).abs().max().item()
    print(f"[parity] multi-token fp8 steps: route vs fp64 on its codes {err_a:.3e}, bf16 route vs fp64 {err_b:.3e}, "
          f"max|logit| {scale:.3e}")
    assert math.isfinite(err_a) and err_a <= 2.0 * err_b + 1e-3 * scale, (err_a, err_b, scale)
