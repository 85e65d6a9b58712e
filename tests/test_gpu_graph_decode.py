"""-m gpu: graph-replayed Perceiver AR decoding.  The window decode kernel recorded once and replayed over windows
rewritten in device memory, against fp64 attention on the window's rows; the append and rotary kernels at device rows
bit for bit against the eager ops; and a GraphedDecoder generation loop (left padding, both windows sliding, a beam
reorder) against an fp64 copy of the model, with every step under the CUDA sync-debug mode "error" and one capture."""
import copy

import pytest
import torch

from gpu_util import assert_parity
from test_gpu_fp8_kv_cache import _Fp64Attend, _amax_descale, _owners, _ref_codes

pytestmark = pytest.mark.gpu

F8 = torch.float8_e4m3fn
# (begin, end) windows of a 6000-row arena: lengths 1, 17, 1023, 1024, 5000 at non-zero begins, and an empty window
WINDOWS = [(7, 8), (100, 117), (500, 1523), (3000, 4024), (1000, 6000)]


def _record(fn):
    """(graph, static output) of fn() recorded once (after one eager warm-up on a side stream)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("kind", ["bf16", "fp16", "e4m3"])
def test_window_decode_replays_every_window(kind, N):
    from perceiver_io_b200 import ops

    dtype = torch.float16 if kind == "fp16" else torch.bfloat16
    g = torch.Generator().manual_seed(17)
    B, H, d, cap = 2, 4, 64, 6000
    q = (2.0 * torch.randn(B, N, H * d, generator=g)).to(dtype).cuda()
    k = torch.randn(B, cap, H * d, generator=g).to(dtype).cuda()
    v = torch.randn(B, cap, H * d, generator=g).to(dtype).cuda()
    pad = torch.zeros(B, cap, dtype=torch.uint8, device="cuda")
    pad[0, 500:700] = 1
    pad[0, 1000:1200] = 1
    pad[1, 3000:4024] = 1                 # the 1024-key window is fully masked on this row: the uniform average
    scale = d ** -0.5
    kd = vd = None
    if kind == "e4m3":
        kd, vd = _amax_descale(k, H), _amax_descale(v, H, per_channel=True)
        k, v = ops.fp8_quantize(k, kd, H), ops.fp8_quantize(v, vd, H)
        kq, vq = ops.fp8_dequantize(k, kd, H, torch.float64), ops.fp8_dequantize(v, vd, H, torch.float64)
    else:
        kq, vq = k, v
    bounds = torch.tensor([1, 2], dtype=torch.int32, device="cuda")
    graph, out = _record(lambda: ops.attention_decode_window(q, k, v, bounds, H, scale, pad_mask=pad, causal=True,
                                                             k_descale=kd, v_descale=vd))
    for b0, b1 in WINDOWS:
        bounds.copy_(torch.tensor([b0, b1], dtype=torch.int32))
        graph.replay()
        assert_parity(out, q, kq[:, b0:b1], vq[:, b0:b1], H, scale, pad[:, b0:b1].bool(), causal=True,
                      eager_dtype=dtype, what=f"{kind} window [{b0},{b1}) N={N}")
    bounds.copy_(torch.tensor([40, 40], dtype=torch.int32))
    graph.replay()
    assert (out == 0).all(), "an empty window writes zeros"


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "e4m3"])
def test_append_and_rotary_at_device_rows_are_bit_equal(fp8):
    from perceiver_io_b200 import ops

    g = torch.Generator().manual_seed(23)
    B, H, d, f, cap = 3, 4, 64, 32, 300
    inv_freq = (1.0 / 10000 ** (torch.arange(0, f, 2, dtype=torch.float32) / f)).bfloat16().cuda()
    table = ops.rotary_angle_table(inv_freq, cap)
    dt = F8 if fp8 else torch.bfloat16
    K = torch.zeros(B, cap, H * d, dtype=dt, device="cuda")
    V = torch.zeros_like(K)
    S = torch.zeros_like(K)
    k_inv = (torch.rand(H * d, generator=g) * 50 + 1).cuda()
    v_inv = (torch.rand(H * d, generator=g) * 50 + 1).cuda()
    kd = (1.0 / k_inv.view(H, d)[:, 0]).contiguous() * 2
    inv_h = 1.0 / kd
    kn = torch.randn(B, 1, H * d, generator=g).bfloat16().cuda()
    vn = torch.randn(B, 1, H * d, generator=g).bfloat16().cuda()
    qn = torch.randn(B, 1, H * d, generator=g).bfloat16().cuda()
    rows = torch.tensor([0, 1, 0, 0], dtype=torch.int32, device="cuda")   # [row, 1 (into S), row, 0 (q)]

    def fn():
        ops.kv_append_at(K, V, kn, vn, rows[0:1], *((k_inv, v_inv) if fp8 else ()))
        ops.rotary_apply_at(kn, H, table, rows[0:2], S, inv_h if fp8 else None)
        return ops.rotary_apply_at(qn, H, table, rows[2:4], torch.empty_like(qn))

    graph, q_rot = _record(fn)
    for r in (5, 6, 150, 299, cap, 10_000):            # the last two land past the arena: skipped
        kn.copy_(torch.randn(B, 1, H * d, generator=g).bfloat16())
        vn.copy_(torch.randn(B, 1, H * d, generator=g).bfloat16())
        qn.copy_(torch.randn(B, 1, H * d, generator=g).bfloat16())
        before = [t.clone() for t in (K, V, S)]
        rows.copy_(torch.tensor([r, 1, r, 0], dtype=torch.int32))
        graph.replay()
        if r >= cap:
            assert all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(before, (K, V, S)))
            continue
        if fp8:
            assert torch.equal(K[:, r].view(torch.uint8), _ref_codes(kn[:, 0], k_inv))
            assert torch.equal(V[:, r].view(torch.uint8), _ref_codes(vn[:, 0], v_inv))
            want = torch.empty(B, 1, H * d, dtype=F8, device="cuda")
            ops._rotary_fp8(kn, H, ops._abs_angles(inv_freq.float(), r, 1), want, inv_h)
            assert torch.equal(S[:, r].view(torch.uint8), want[:, 0].view(torch.uint8))
        else:
            assert torch.equal(K[:, r], kn[:, 0]) and torch.equal(V[:, r], vn[:, 0])
            assert torch.equal(S[:, r], ops.rotary_at(kn, H, inv_freq, r)[:, 0])
        assert torch.equal(q_rot, ops.rotary_at(qn, H, inv_freq, r))
        # rows other than r are untouched
        mask = torch.ones(cap, dtype=torch.bool, device="cuda")
        mask[r] = False
        assert all(torch.equal(a[:, mask].view(torch.uint8), b[:, mask].view(torch.uint8))
                   for a, b in zip(before, (K, V, S)))


def _model(abs_pos_emb):
    import perceiver_io_b200 as P

    torch.manual_seed(3)
    cfg = P.CausalSequenceModelConfig(vocab_size=97, max_seq_len=160, max_latents=48, num_channels=128, num_heads=4,
                                      num_self_attention_layers=2, num_self_attention_rotary_layers=1,
                                      cross_attention_dropout=0.0, output_norm=True, abs_pos_emb=abs_pos_emb,
                                      init_scale=0.1)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.LayerNorm):
                m.weight.add_(0.3 * torch.randn_like(m.weight))
                m.bias.add_(0.3 * torch.randn_like(m.bias))
    return cfg, model


@pytest.mark.parametrize("abs_pos_emb", [False, True], ids=["rotary", "abs_pos"])
def test_graphed_generation_matches_fp64(monkeypatch, abs_pos_emb):
    import perceiver_io_b200 as P
    from perceiver_io_b200 import modules

    cfg, model = _model(abs_pos_emb)
    model64 = copy.deepcopy(model).double()
    fp64 = _Fp64Attend(model64, _owners(model64))
    B, n0, prefix, steps, reorder_step = 2, 120, 90, 60, 20
    tokens0 = torch.randint(0, 97, (B, n0 + steps + 1)).cuda()
    pad0 = torch.zeros(B, tokens0.shape[1], dtype=torch.bool, device="cuda")
    pad0[1, :7] = True

    def eager(arm):
        """Per-step last-position logits of this package's eager cached loop ("bf16" / "fp8") or of the fp64 model."""
        tokens, pad, out = tokens0.clone(), pad0.clone(), []

        def call(x, plen, pm, kv):
            if arm == "fp64":
                with monkeypatch.context() as mp:
                    mp.setattr(modules, "attend", fp64)
                    mp.setattr(modules, "_kv8_route", lambda *a: None)
                    return model64(x, prefix_len=plen, pad_mask=pm, kv_cache=kv)
            modules.fp8_config["kv_cache"] = arm == "fp8"
            try:
                return model(x, prefix_len=plen, pad_mask=pm, kv_cache=kv)
            finally:
                modules.fp8_config["kv_cache"] = False

        with torch.no_grad():
            o = call(tokens[:, :n0], prefix, pad[:, :n0], [])
            out.append(o.logits[:, -1].double())
            cache = o.kv_cache
            for s, w in enumerate(P.decode_windows(n0, prefix, steps, cfg.max_seq_len, cfg.max_latents)):
                n, nlat = w.ca_end - w.ca_begin, w.sa_end - w.sa_begin
                cache = ([(cache[0][0][:, -(n - 1):], cache[0][1][:, -(n - 1):])]
                         + [(k[:, -(nlat - 1):], v[:, -(nlat - 1):]) for k, v in cache[1:]])
                if s == reorder_step:
                    idx = torch.tensor([1, 0], device="cuda")
                    cache = [(k.index_select(0, idx), v.index_select(0, idx)) for k, v in cache]
                    tokens, pad = tokens[idx], pad[idx]
                pos = n0 + s
                o = call(tokens[:, pos:pos + 1], w.prefix_len, pad[:, pos + 1 - n:pos + 1], cache)
                out.append(o.logits[:, -1].double())
                cache = o.kv_cache
        return torch.stack(out)

    def graphed(kind):
        tokens, out = tokens0.clone(), []
        dec = P.GraphedDecoder(model, batch=B, max_new_tokens=steps, kv_cache=kind)
        out.append(dec.prefill(tokens[:, :n0], prefix, pad0[:, :n0]).double())
        for s in range(steps):
            if s == reorder_step:
                idx = torch.tensor([1, 0], device="cuda")
                dec.reorder(idx)
                tokens = tokens[idx]
            torch.cuda.set_sync_debug_mode("error")
            try:
                logits = dec.step(tokens[:, n0 + s:n0 + s + 1])
            finally:
                torch.cuda.set_sync_debug_mode(0)
            out.append(logits.double().clone())
        assert dec.captures == 1
        with pytest.raises(RuntimeError, match="0 of max_new_tokens"):
            dec.step(tokens[:, :1])
        return torch.stack(out)

    truth = eager("fp64")
    scale = truth.abs().max().item()
    for kind in ("bf16", "fp8"):
        e = (eager(kind) - truth).abs().max().item()
        got = graphed(kind)
        assert torch.isfinite(got).all()
        err = (got - truth).abs().max().item()
        print(f"[parity] graphed {kind} generation: err {err:.3e}, eager {kind} err {e:.3e}, max|logit| {scale:.3e}")
        assert err <= 2.0 * e + 1e-3 * scale, (kind, err, e, scale)
