"""-m gpu: the FP8 (e4m3) KV cache of cached generation: the e4m3 decode kernel against fp64 attention on the
dequantised codes, the quantising append bit for bit, the e4m3 rotary shadow within half an e4m3 ulp, and a Perceiver AR
generation loop against an fp64 copy of the model that reads the codes the route produced."""
import copy
import math

import pytest
import torch

from gpu_util import assert_parity, torch_core

pytestmark = pytest.mark.gpu

F8 = torch.float8_e4m3fn


def _qkv(B, N, M, H, dqk, dv, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    q = (2.0 * torch.randn(B, N, H * dqk, generator=g)).to(dtype).cuda()
    k = torch.randn(B, M, H * dqk, generator=g).to(dtype).cuda()
    v = torch.randn(B, M, H * dv, generator=g).to(dtype).cuda()
    return q, k, v


def _amax_descale(x, H, per_channel=False):
    a = x.float().abs().reshape(-1, H, x.shape[-1] // H).amax(dim=0)
    return ((a if per_channel else a.amax(dim=1)) / 448.0).clamp_min(1e-12)


DECODE_SHAPES = [
    # B, N, M, H, dqk, dv: the bf16 decode test's shapes whose head dims are multiples of 16, then short key axes
    (8, 1, 16384, 8, 128, 128),
    (2, 1, 5000, 8, 96, 96),
    (3, 2, 2049, 4, 64, 64),
    (2, 4, 3000, 8, 32, 160),
    (1, 3, 2500, 1, 256, 256),
    (2, 1, 1, 4, 64, 64),
    (3, 4, 17, 2, 32, 32),
    (2, 2, 511, 4, 64, 256),
]


@pytest.mark.parametrize("shape", DECODE_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_decode_fp8_kernel_matches_fp64_on_the_codes(shape, dtype):
    """Dequantisation is exact, so fp64 attention on the dequantised codes isolates the kernel from the quantisation
    error; the gate is the bf16 decode test's derived gate."""
    from perceiver_io_b200 import ops

    B, N, M, H, dqk, dv = shape
    q, k, v = _qkv(B, N, M, H, dqk, dv, seed=41, dtype=dtype)
    kd, vd = _amax_descale(k, H), _amax_descale(v, H, per_channel=True)
    k8, v8 = ops.fp8_quantize(k, kd, H), ops.fp8_quantize(v, vd, H)
    kq, vq = ops.fp8_dequantize(k8, kd, H, torch.float64), ops.fp8_dequantize(v8, vd, H, torch.float64)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, : M // 9] = True
    if B > 1:
        pad[1, :] = True              # fully padded batch row: uniform average of all values
    scale = dqk ** -0.5
    assert ops.attention_decode_fp8_supported(q, k8, v8, kd, vd, H, scale)
    for causal in (False, True):
        out = ops.attention_decode_fp8(q, k8, v8, kd, vd, H, scale, pad_mask=pad.cuda(), causal=causal)
        assert out.dtype == dtype and out.shape == (B, N, H * dv)
        assert_parity(out, q, kq, vq, H, scale, pad, causal, eager_dtype=dtype, what=f"e4m3 decode {shape} causal={causal}")
    q1 = q[:1]
    out = ops.attention_decode_fp8(q1, k8, v8, kd, vd, H, scale)
    assert_parity(out, q1, kq, vq, H, scale, eager_dtype=dtype, what=f"e4m3 decode {shape} broadcast q")


def _ref_codes(x, inv):
    return (x.float() * inv).clamp(-448.0, 448.0).to(F8).view(torch.uint8)


def test_quantising_append_is_bit_exact():
    from perceiver_io_b200 import ops

    g = torch.Generator().manual_seed(5)
    B, Ck, Cv = 3, 128, 96
    k_inv = (torch.rand(Ck, generator=g) * 200 + 1).cuda()
    v_inv = (torch.rand(Cv, generator=g) * 200 + 1).cuda()
    k_inv[:4] = 1e5                                   # saturating channels
    rows_k, rows_v = [], []
    k = torch.empty(B, 0, Ck, dtype=torch.bfloat16, device="cuda")
    v = torch.empty(B, 0, Cv, dtype=torch.bfloat16, device="cuda")
    for step, n in enumerate((5, 1, 3, 1, 70, 1)):    # the 70-row append outgrows the arena: a copying append
        kn = torch.randn(B, n, Ck, generator=g).bfloat16().cuda()
        vn = (torch.randn(B, n, Cv, generator=g) * 3).bfloat16().cuda()
        rows_k.append(kn)
        rows_v.append(vn)
        k, v = ops.kv_append_fp8(k, v, kn, vn, k_inv, v_inv)
        assert k.dtype == F8 and v.dtype == F8
        assert torch.equal(k.view(torch.uint8), _ref_codes(torch.cat(rows_k, 1), k_inv)), step
        assert torch.equal(v.view(torch.uint8), _ref_codes(torch.cat(rows_v, 1), v_inv)), step
    # truncation keeps the arena, index_select makes a fresh one (a copying append of the old codes)
    idx = torch.tensor([2, 0, 1], device="cuda")
    kr, vr = k[:, 4:].index_select(0, idx), v[:, 4:].index_select(0, idx)
    kn = torch.randn(B, 2, Ck, generator=g).half().cuda()
    vn = torch.randn(B, 2, Cv, generator=g).half().cuda()
    k2, v2 = ops.kv_append_fp8(kr, vr, kn, vn, k_inv, v_inv)
    assert torch.equal(k2[:, :-2].view(torch.uint8), kr.view(torch.uint8))
    assert torch.equal(k2[:, -2:].view(torch.uint8), _ref_codes(kn, k_inv))
    assert torch.equal(v2[:, -2:].view(torch.uint8), _ref_codes(vn, v_inv))


def _e4m3_half_ulp(x):
    """Half the e4m3 spacing at |x| (normals: 2^(e-3); subnormals below 2^-6: 2^-9)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -6)))
    return 0.5 * torch.exp2(e - 3)


@pytest.mark.parametrize("rotate_frac", [1, 2], ids=["full", "half"])
def test_rotary_shadow_within_half_an_ulp(rotate_frac):
    from perceiver_io_b200 import ops

    g = torch.Generator().manual_seed(8)
    B, L, H, d = 2, 300, 4, 64
    f = d // rotate_frac
    inv_freq = (1.0 / 10000 ** (torch.arange(0, f, 2, dtype=torch.float32) / f)).cuda()
    x = (torch.randn(B, L, H * d, generator=g) * 2).bfloat16().cuda()
    kd = _amax_descale(x, H) * 1.5                      # room for the rotation (pair norm <= sqrt(2) amax)
    empty = torch.empty(B, 0, H * d, dtype=torch.bfloat16, device="cuda")
    k8, _ = ops.kv_append_fp8(empty, empty, x, x, 1.0 / kd.repeat_interleave(d), 1.0 / kd.repeat_interleave(d))
    q = x[:, -1:]
    ops.rotated_cache_keys(k8, q, H, inv_freq, k_new=x, k_descale=kd)
    angles = ops._abs_angles(inv_freq, 0, L).double()[0]            # (L, f)

    def rot64(t):
        t = t.double().reshape(B, L, H, d).clone()
        a = angles[None, :, None, :]
        e, o = t[..., 0:f:2].clone(), t[..., 1:f:2].clone()
        t[..., 0:f:2] = e * torch.cos(a[..., 0::2]) - o * torch.sin(a[..., 0::2])
        t[..., 1:f:2] = o * torch.cos(a[..., 1::2]) + e * torch.sin(a[..., 1::2])
        return t, (e.abs() + o.abs())

    for name, src in (("bf16 rows", x.double()), ("e4m3 codes", ops.fp8_dequantize(k8, kd, H, torch.float64))):
        if name == "e4m3 codes":                       # a fresh arena: the shadow is rebuilt from the codes
            k8 = k8.index_select(0, torch.arange(B, device="cuda"))
            k8, _ = ops.kv_append_fp8(k8, k8, x[:, :0], x[:, :0], 1.0 / kd.repeat_interleave(d),
                                      1.0 / kd.repeat_interleave(d))
            ops.rotated_cache_keys(k8, q, H, inv_freq, k_new=x[:, :0], k_descale=kd)
        shadow, p0 = ops.rotated_cache_shadow(k8)
        assert p0 == 0 and shadow.dtype == F8
        want, mag = rot64(src)
        want = want / kd.double()[None, None, :, None]
        got = shadow.double().reshape(B, L, H, d)
        slack = 2.0 ** -20 * want.abs()                 # fp32 products and scales
        slack[..., :f] += 2.0 ** -20 * torch.stack([mag, mag], -1).flatten(-2) / kd.double()[None, None, :, None]
        err = (got - want).abs() - _e4m3_half_ulp(want) - slack
        print(f"[rotary e4m3] {name}: max excess over half an ulp {err.max().item():.3e}")
        assert err.max().item() <= 0, name


# ---- the generation loop ------------------------------------------------------------------------------------------
def _rotate64(t, H, angles):
    """fp64 rotation of (B, n, H*d) rows by (Ba, n, f) angles (the kernels' pairwise formula)."""
    B, n, C = t.shape
    f = angles.shape[-1]
    x = t.reshape(B, n, H, C // H).clone()
    a = angles[:, :, None, :]
    e, o = x[..., 0:f:2].clone(), x[..., 1:f:2].clone()
    x[..., 0:f:2] = e * torch.cos(a[..., 0::2]) - o * torch.sin(a[..., 0::2])
    x[..., 1:f:2] = o * torch.cos(a[..., 1::2]) + e * torch.sin(a[..., 1::2])
    return x.reshape(B, n, C)


class _Fp64Attend:
    """``modules.attend`` of an fp64 copy of the model.  mode "own": its own fp64 cache and the reference's
    window-relative rotary; mode "codes": the dequantised codes of the caches the FP8 route produced in this step
    (``route_cache``) and of their rotated shadows, q rotated at the shadow's absolute positions."""

    def __init__(self, model64, owners):
        from perceiver_io_b200 import modules

        self.modules = modules
        self.mhas = {id(o.attention): i for i, o in enumerate(owners)}
        self.owners = owners
        self.mode, self.route_cache, self.route_scales = "own", None, None

    def __call__(self, mha, q, k, v, pad_mask=None, rot_pos_emb_q=None, rot_pos_emb_k=None, kv_cache=None,
                 min_rows_key=None, kv8=None):
        from perceiver_io_b200 import ops

        H = mha.num_heads
        if self.mode == "own":
            if kv_cache is not None:
                k, v = torch.cat([kv_cache[0], k], 1), torch.cat([kv_cache[1], v], 1)
                kv_cache = (k, v)
            frq = (lambda r: r.frq_pos_enc[:, 0].double())
            q_r = q if rot_pos_emb_q is None else _rotate64(q, H, frq(rot_pos_emb_q)[:, -q.shape[1]:])
            k_r = k if rot_pos_emb_k is None else _rotate64(k, H, frq(rot_pos_emb_k)[:, -k.shape[1]:])
            v_r = v
        else:
            i = self.mhas[id(mha)]
            k8, v8 = self.route_cache[i]
            s = self.route_scales[i]
            v_r = ops.fp8_dequantize(v8, s.v_descale, H, torch.float64)
            if rot_pos_emb_k is not None:
                shadow, p0 = ops.rotated_cache_shadow(k8)
                k_r = ops.fp8_dequantize(shadow, s.k_descale, H, torch.float64)
                L, N = k8.shape[1], q.shape[1]
                inv_freq = rot_pos_emb_k.inv_freq.double()
                pos = torch.arange(p0 + L - N, p0 + L, device=q.device, dtype=torch.float64)
                ang = (pos[None, :, None] * inv_freq[None, None, :]).repeat_interleave(2, dim=-1)
                q_r = _rotate64(q, H, ang)
            else:
                k_r, q_r = ops.fp8_dequantize(k8, s.k_descale, H, torch.float64), q
        o = torch_core(q_r, k_r, v_r, H, mha.dp_scale, pad_mask, mha.causal_attention, torch.float64)
        return self.modules.ModuleOutput(last_hidden_state=mha.o_proj(o), kv_cache=kv_cache)


def _owners(model):
    import perceiver_io_b200 as P

    return [m for m in model.modules() if isinstance(m, (P.CrossAttention, P.SelfAttention))]


def test_generation_loop_with_fp8_caches_matches_fp64_on_the_codes(monkeypatch):
    """Left padding, 40 cached steps (one of them with 5 new tokens, which takes the dequantising path), sliding-window
    truncation of both caches and one beam reorder.  Every step's logits of the FP8 route are gated against an fp64
    copy of the model that reads the route's codes; the gate is the bf16 rotated-key test's derived gate (twice the
    bf16 route's distance from the unquantised fp64 model, plus 1e-3 of the largest logit)."""
    import perceiver_io_b200 as P
    from perceiver_io_b200 import modules, ops

    torch.manual_seed(3)
    cfg = P.CausalSequenceModelConfig(vocab_size=97, max_seq_len=160, max_latents=48, num_channels=128, num_heads=4,
                                      num_self_attention_layers=2, num_self_attention_rotary_layers=1,
                                      cross_attention_dropout=0.0, output_norm=True, abs_pos_emb=False, init_scale=0.1)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    with torch.no_grad():   # LayerNorm affine parameters away from (1, 0): the scales must hold for trained weights
        for m in model.modules():
            if isinstance(m, torch.nn.LayerNorm):
                m.weight.add_(0.3 * torch.randn_like(m.weight))
                m.bias.add_(0.3 * torch.randn_like(m.bias))
    model64 = copy.deepcopy(model).double()
    fp64 = _Fp64Attend(model64, _owners(model64))
    B, n0, prefix, steps, wide_step, reorder_step = 2, 120, 90, 40, 30, 20
    tokens0 = torch.randint(0, 97, (B, n0 + steps + 4)).cuda()
    pad0 = torch.zeros(B, tokens0.shape[1], dtype=torch.bool, device="cuda")
    pad0[1, :7] = True

    def run(arm):
        tokens, pad = tokens0.clone(), pad0.clone()
        out, ref = [], []
        pos = n0

        def call(x, plen, pm, kv):
            if arm == "fp64":
                with monkeypatch.context() as mp:
                    mp.setattr(modules, "attend", fp64)
                    mp.setattr(modules, "_kv8_route", lambda *a: None)
                    fp64.mode = "own"
                    return model64(x, prefix_len=plen, pad_mask=pm, kv_cache=kv)
            modules.fp8_config["kv_cache"] = arm == "fp8"
            try:
                o = model(x, prefix_len=plen, pad_mask=pm, kv_cache=kv)
            finally:
                modules.fp8_config["kv_cache"] = False
            if arm == "fp8":
                for kc, vc in o.kv_cache:
                    assert kc.dtype == F8 and vc.dtype == F8 and kc.dim() == 3 and vc.dim() == 3
                with monkeypatch.context() as mp:
                    mp.setattr(modules, "attend", fp64)
                    mp.setattr(modules, "_kv8_route", lambda *a: None)
                    if len(kv) == 0:       # the prompt attended over its own rows
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
            cache = o.kv_cache
            for s in range(steps):
                m = 5 if s == wide_step else 1
                n = cache[0][0].shape[1] + m
                if n > cfg.max_seq_len:                      # sliding window: drop the oldest cached tokens
                    d = n - cfg.max_seq_len
                    cache = [(cache[0][0][:, d:], cache[0][1][:, d:])] + cache[1:]
                    n -= d
                nlat = cache[1][0].shape[1] + m
                if nlat > cfg.max_latents:                    # latents move into the prefix
                    d = nlat - cfg.max_latents
                    cache = cache[:1] + [(k[:, d:], v[:, d:]) for k, v in cache[1:]]
                    nlat -= d
                plen = n - nlat
                if s == reorder_step:                        # a beam reorder
                    idx = torch.tensor([1, 0], device="cuda")
                    cache = [(k.index_select(0, idx), v.index_select(0, idx)) for k, v in cache]
                    tokens, pad = tokens[idx], pad[idx]
                o = call(tokens[:, pos:pos + m], plen, pad[:, pos + m - n:pos + m], cache)
                out.append(o.logits[:, -1].double())
                cache = o.kv_cache
                pos += m
        return torch.stack(out), (torch.stack(ref) if ref else None), cache

    a, a_ref, cache8 = run("fp8")
    b, _, cache16 = run("bf16")
    truth, _, _ = run("fp64")
    assert torch.isfinite(a).all()
    scale = truth.abs().max().item()
    err_a = (a - a_ref).abs().max().item()
    err_b = (b - truth).abs().max().item()
    err_q = (a - truth).abs().max().item()
    print(f"[parity] fp8 KV cache: route vs fp64 on its codes {err_a:.3e}, bf16 route vs fp64 {err_b:.3e}, "
          f"fp8 route vs unquantised fp64 {err_q:.3e}, max|logit| {scale:.3e}")
    assert err_a <= 2.0 * err_b + 1e-3 * scale, (err_a, err_b, scale)
    # quantisation error: e4m3 rounds K and V by at most 2^-4 relative; three attention layers lie between the caches and
    # the logits, each moving its output by at most that fraction of its value scale
    assert math.isfinite(err_q) and err_q <= 3 * 2.0 ** -4 * scale, (err_q, scale)
    # memory: at the same lengths the e4m3 arenas hold half the bytes of the bf16 ones
    def nbytes(cache):
        return sum((t._base if t._base is not None else t).untyped_storage().nbytes() for kv in cache for t in kv)

    assert [t.shape for kv in cache8 for t in kv] == [t.shape for kv in cache16 for t in kv]
    assert 2 * nbytes(cache8) == nbytes(cache16), (nbytes(cache8), nbytes(cache16))


def test_switching_the_option_keeps_each_cache_dtype():
    import perceiver_io_b200 as P
    from perceiver_io_b200 import modules

    torch.manual_seed(1)
    layer = P.SelfAttention(num_heads=4, num_channels=128, causal_attention=True).cuda().bfloat16().eval()
    x = torch.randn(2, 6, 128, device="cuda").bfloat16()
    empty = (torch.empty(2, 0, 128, device="cuda").bfloat16(),) * 2
    with torch.no_grad():
        modules.fp8_config["kv_cache"] = True
        try:
            c8 = layer(x, kv_cache=empty).kv_cache
            c16 = None
            modules.fp8_config["kv_cache"] = False
            c16 = layer(x, kv_cache=empty).kv_cache
            modules.fp8_config["kv_cache"] = True
            o16 = layer(x[:, :1], kv_cache=c16)                 # a non-empty bf16 cache stays bf16
        finally:
            modules.fp8_config["kv_cache"] = False
        o8 = layer(x[:, :1], kv_cache=c8)                       # an e4m3 cache keeps working with the option off
    assert c8[0].dtype == F8 and o8.kv_cache[0].dtype == F8 and o8.kv_cache[0].shape == (2, 7, 128)
    assert c16[0].dtype == torch.bfloat16 and o16.kv_cache[0].dtype == torch.bfloat16
    h8, h16 = o8.last_hidden_state.float(), o16.last_hidden_state.float()
    assert torch.isfinite(h8).all() and (h8 - h16).abs().max() <= 0.1 * h16.abs().max()


class _RefRotary:
    """The reference's RotaryPositionEmbedding as the patched forwards see it: ``frq_pos_enc`` (B, 1, n, f) and
    ``right_align``, no frequency table."""

    def __init__(self, frq_pos_enc, right_align=True):
        self.frq_pos_enc, self.right_align = frq_pos_enc, right_align


def _window_angles(B, n, f, shift):
    """(B, 1, n, f) angles of positions 0..n-1 shifted per batch row (left padding), every frequency repeated twice."""
    inv_freq = 1.0 / 10000 ** (torch.arange(0, f, 2, dtype=torch.float32) / f)
    pos = torch.arange(n, dtype=torch.float32)[None, :] - torch.tensor(shift, dtype=torch.float32)[:, None]
    return (pos[..., None] * inv_freq).repeat_interleave(2, dim=-1)[:, None].cuda()


@pytest.mark.parametrize("rotary", [False, True], ids=["plain", "rotary"])
def test_patched_reference_modules_take_the_route(monkeypatch, rotary):
    """patch() finds reference modules by class name and attributes; the rebound forwards take the FP8 cache, and every
    cached step runs the e4m3 decode kernel.  With the reference's rotary objects (no frequency table) the cache is
    rotated at the window-relative angles e4m3 to e4m3 before the decode kernel."""
    import perceiver_io_b200 as P
    from perceiver_io_b200 import modules, ops

    class CrossAttention(torch.nn.Module):
        def __init__(self, C, H):
            super().__init__()
            self.q_norm, self.kv_norm = torch.nn.LayerNorm(C), torch.nn.LayerNorm(C)
            self.attention = P.MultiHeadAttention(H, C, C, causal_attention=True)

    class SelfAttention(torch.nn.Module):
        def __init__(self, C, H):
            super().__init__()
            self.norm = torch.nn.LayerNorm(C)
            self.attention = P.MultiHeadAttention(H, C, C, causal_attention=True)

    torch.manual_seed(2)
    C, H, B = 128, 4, 2
    net = torch.nn.ModuleDict({"ca": CrossAttention(C, H), "sa": SelfAttention(C, H)}).cuda().bfloat16().eval()
    P.patch(net)
    x = torch.randn(B, 9, C, device="cuda").bfloat16()
    prefix = torch.randn(B, 20, C, device="cuda").bfloat16()
    empty = (torch.empty(B, 0, C, device="cuda").bfloat16(),) * 2
    shift = [0, 3]
    rot = (lambda n: _RefRotary(_window_angles(B, n, C // H, shift))) if rotary else (lambda n: None)
    calls = {"decode": 0, "rotary_fp8": 0}
    for name in calls:
        fn = getattr(ops, {"decode": "attention_decode_fp8", "rotary_fp8": "rotary_fp8"}[name])

        def spy(*a, _fn=fn, _name=name, **kw):
            calls[_name] += 1
            return _fn(*a, **kw)

        monkeypatch.setattr(ops, fn.__name__, spy)

    def step(on):
        modules.fp8_config["kv_cache"] = on
        try:
            with torch.no_grad():
                ca = net["ca"](x[:, :8], x_kv_prefix=prefix, rot_pos_emb_q=rot(8), rot_pos_emb_k=rot(28), kv_cache=empty)
                sa = net["sa"](x[:, :8], rot_pos_emb=rot(8), kv_cache=empty)
                ca1 = net["ca"](x[:, 8:], x_kv_prefix=prefix[:, :0], rot_pos_emb_q=rot(29), rot_pos_emb_k=rot(29),
                                kv_cache=ca.kv_cache)
                sa1 = net["sa"](x[:, 8:], rot_pos_emb=rot(9), kv_cache=sa.kv_cache)
        finally:
            modules.fp8_config["kv_cache"] = False
        return ca1, sa1

    ca8, sa8 = step(True)
    assert calls == {"decode": 2, "rotary_fp8": 2 if rotary else 0}, calls
    ca16, sa16 = step(False)
    assert calls["decode"] == 2
    for o8, o16 in ((ca8, ca16), (sa8, sa16)):
        assert o8.kv_cache[0].dtype == F8 and o8.kv_cache[1].dtype == F8 and o16.kv_cache[0].dtype == torch.bfloat16
        h8, h16 = o8.last_hidden_state.float(), o16.last_hidden_state.float()
        assert torch.isfinite(h8).all() and (h8 - h16).abs().max() <= 0.1 * h16.abs().max()


def test_window_rotation_of_codes_within_half_an_ulp():
    """ops.rotary_fp8: e4m3 codes rotated at per-batch, right-aligned angles and requantised with the same descale are
    within half an e4m3 ulp (plus fp32 rounding) of the fp64 rotation of the dequantised codes."""
    from perceiver_io_b200 import ops

    g = torch.Generator().manual_seed(12)
    B, L, H, d, f = 2, 200, 4, 64, 32
    x = (torch.randn(B, L, H * d, generator=g) * 2).bfloat16().cuda()
    kd = _amax_descale(x, H) * 1.5
    x8 = ops.fp8_quantize(x, kd, H)
    angles = _window_angles(B, L + 7, f, [0, 5])              # more angle rows than keys: right-aligned
    y8 = ops.rotary_fp8(x8, H, angles, True, kd)
    src = ops.fp8_dequantize(x8, kd, H, torch.float64)
    want = _rotate64(src, H, angles[:, 0, -L:].double()).reshape(B, L, H, d) / kd.double()[None, None, :, None]
    xs = src.reshape(B, L, H, d) / kd.double()[None, None, :, None]
    mag = torch.cat([(xs[..., 0:f:2].abs() + xs[..., 1:f:2].abs()).repeat_interleave(2, -1), xs[..., f:].abs()], -1)
    err = (y8.double().reshape(B, L, H, d) - want).abs() - _e4m3_half_ulp(want) - 2.0 ** -20 * (mag + want.abs())
    print(f"[rotary e4m3] window angles: max excess over half an ulp {err.max().item():.3e}")
    assert err.max().item() <= 0


def test_training_mode_with_attention_dropout_keeps_the_bf16_cache():
    """Attention dropout runs on the bf16 path only: a module in training mode with dropout keeps a bf16 cache under
    the option, and an e4m3 cache fed to it is refused rather than run without its dropout."""
    import perceiver_io_b200 as P
    from perceiver_io_b200 import modules

    torch.manual_seed(4)
    layer = P.SelfAttention(num_heads=4, num_channels=128, causal_attention=True, dropout=0.1).cuda().bfloat16().eval()
    x = torch.randn(2, 6, 128, device="cuda").bfloat16()
    empty = (torch.empty(2, 0, 128, device="cuda").bfloat16(),) * 2
    modules.fp8_config["kv_cache"] = True
    try:
        with torch.no_grad():
            c8 = layer(x, kv_cache=empty).kv_cache
            layer.train()
            c16 = layer(x, kv_cache=empty).kv_cache
            with pytest.raises(RuntimeError, match="attention dropout"):
                layer(x[:, :1], kv_cache=c8)
    finally:
        modules.fp8_config["kv_cache"] = False
    assert c8[0].dtype == F8 and c16[0].dtype == torch.bfloat16
