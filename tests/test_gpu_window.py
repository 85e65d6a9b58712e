"""-m gpu: the banded-window tensor-core attention (ops.attention_window: pcv_attn_cached_window / _fp8) and the k-token
steps of GraphedDecoder.

Kernel: every instantiation, recorded once per (rows, band) in a CUDA graph and replayed across windows by rewriting
only the device bounds, against fp64 attention on each row's keys with the element-wise gate of window_variants; an
empty window writes zeros; two launches are bit-identical; with the window [0, capacity) and no band the e4m3 entry is
bit-identical to pcv_attn_cached_fp8.  Exact probes (decode_variants.py's operands, the expected key sets from
window_variants.row_keys), every instantiation, recorded once per (rows, band) and replayed across the windows: the
count probe (q = 0: RN16(S / L) of the integer sum and count of a row's live keys, V nonzero only at the window, split,
tile and mask edges and at padded keys) and the needle probe (one key ~185 log2 units above the rest per (b, h, n), on
that row's band edge r_i + 1 - W and the key before it, its last key and the one after it, its causal diagonal, the
window, split and tile edges and the first and last padded key: RN16(v[needle]) when it is live, else the count probe's
row), both bit for bit.  Model loop: a GraphedDecoder fed through a mix of step, extend(3 / 5 / 16 / 64),
wrong draft tokens and rewind matches the fp64 one-token loop at every kept position, without a host synchronisation and
with one capture per distinct step length."""
import copy

import pytest
import torch

import decode_variants as DV
import window_variants as WV
from cached_fp8_variants import left_pad
from test_gpu_fp8_kv_cache import _Fp64Attend, _owners
from test_gpu_graph_decode import _model, _record

pytestmark = pytest.mark.gpu

B, H, CAP, SCALE = 3, 2, 1000, 0.3
# (begin, end): lengths 1, 63, 64 and 65 at unaligned begins, nine tiles (three of the four splits B*H = 6 plans at
# this capacity), and the full arena
WINDOWS = [(5, 6), (70, 133), (200, 264), (301, 366), (37, 613), (0, CAP)]
# (rows, band, causal): no band (full and causal), band 1, band 64, a band inside the window, a band wider than it
ROW_BANDS = [(1, 0, True), (5, 0, False), (64, 0, True), (2, 1, True), (5, 64, True), (63, 100, True),
             (64, 2000, True)]


def _operands(case, N, seed):
    dt, kind, dqk, dv = case
    q, k, v, kd, vd, k64, v64 = WV.random_operands(B, B, N, CAP, H, dqk, dv, dt, kind, seed=seed, device="cuda")
    return q, k, v, kd, vd, k64, v64


def _check(out, q, k64, v64, b0, b1, band, pad, causal, dt, pl, what):
    ref, bound = WV.reference_and_bound(q, k64, v64, H, SCALE, b0, b1, band, pad, causal, dt, pl)
    err = (out.double() - ref).abs()
    bad = err > bound
    assert not bad.any(), (f"{what}: {int(bad.sum())} elements over the gate, worst err {err.max().item():.3e}, "
                           f"worst err/gate {(err / bound.clamp_min(1e-300)).max().item():.3f}")


@pytest.mark.parametrize("case", WV.VARIANT_CASES, ids=[WV.case_id(c) for c in WV.VARIANT_CASES])
def test_every_variant_replays_every_window(case):
    from perceiver_io_b200 import ops

    dt, kind, dqk, dv = case
    pl = WV.plan(B, H, CAP, dqk, dv, torch.cuda.get_device_properties(0).multi_processor_count)
    assert [kb for kb, ke in WV.split_tiles(37, 613, CAP, pl["nsplit"]) if ke > kb] == [37, 229, 421]
    pad = left_pad(B, CAP, device="cuda")      # batch row 2 is wholly padded: every band of it is all padding
    for N, band, causal in ROW_BANDS:
        q, k, v, kd, vd, k64, v64 = _operands(case, N, seed=N + band + dqk)
        bounds = torch.tensor([1, 2], dtype=torch.int32, device="cuda")
        graph, out = _record(lambda: ops.attention_window(q, k, v, bounds, H, SCALE, band=band, pad_mask=pad,
                                                          causal=causal, k_descale=kd, v_descale=vd))
        for b0, b1 in WINDOWS:
            bounds.copy_(torch.tensor([b0, b1], dtype=torch.int32))
            graph.replay()
            first = out.clone()
            _check(out, q, k64, v64, b0, b1, band, pad, causal, dt, pl,
                   f"{WV.case_id(case)} N={N} band={band} causal={causal} window [{b0},{b1})")
            graph.replay()
            assert torch.equal(out.view(torch.int16), first.view(torch.int16)), "two launches differ"
        for b0, b1 in ((40, 40), (50, 12)):
            bounds.copy_(torch.tensor([b0, b1], dtype=torch.int32))
            graph.replay()
            assert (out == 0).all(), "an empty window writes zeros"


@pytest.mark.parametrize("case", [c for c in WV.VARIANT_CASES if c[1] == "e4m3"],
                         ids=[WV.case_id(c) for c in WV.VARIANT_CASES if c[1] == "e4m3"])
def test_full_window_without_band_is_the_cached_fp8_kernel(case):
    """Window [0, capacity), no band: bit for bit pcv_attn_cached_fp8 on the same arena (ops.attention_decode_fp8 of
    more than 4 rows), causal with left padding."""
    from perceiver_io_b200 import ops

    pad = left_pad(B, CAP, device="cuda")
    for N in (5, 64):
        q, k, v, kd, vd, _, _ = _operands(case, N, seed=3 * N)
        bounds = torch.tensor([0, CAP], dtype=torch.int32, device="cuda")
        got = ops.attention_window(q, k, v, bounds, H, SCALE, pad_mask=pad, causal=True, k_descale=kd, v_descale=vd)
        want = ops.attention_decode_fp8(q, k, v, kd, vd, H, SCALE, pad_mask=pad, causal=True)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (case, N)


def _assert_bits(got, want, what):
    eq = (got.view(torch.int16) == want.view(torch.int16)) | ((got == 0) & (want == 0))
    if not bool(eq.all()):
        bad = (~eq).nonzero()
        b, n, c = (int(x) for x in bad[0])
        raise AssertionError(f"{what}: {bad.shape[0]} of {eq.numel()} outputs differ; first at (b={b}, n={n}, "
                             f"channel {c}): got {got[b, n, c].item()!r} want {want[b, n, c].item()!r}")


def _probe_graph(case, N, band, causal, pad):
    """(q, k, v, kd, vd, bounds, graph, out): static probe operands and the window attention recorded on them
    (k_descale 1, power-of-two v_descale on e4m3 arenas; scale NEEDLE_SCALE, which the count probe's q = 0 does not
    see).  The graph reads every one of them, so the caller keeps them alive while it replays."""
    from perceiver_io_b200 import ops

    dt, kind, dqk, dv = case
    fp8 = kind == "e4m3"
    dtype = WV.DTYPE[dt]
    kvt = torch.float8_e4m3fn if fp8 else dtype
    q = torch.zeros(B, N, H * dqk, dtype=dtype, device="cuda")
    k = torch.zeros(B, CAP, H * dqk, dtype=kvt, device="cuda")
    v = torch.zeros(B, CAP, H * dv, dtype=kvt, device="cuda")
    kd = torch.ones(H, device="cuda") if fp8 else None
    vd = DV.v_descale(H, dv, "cuda") if fp8 else None
    bounds = torch.tensor([1, 2], dtype=torch.int32, device="cuda")
    graph, out = _record(lambda: ops.attention_window(q, k, v, bounds, H, DV.NEEDLE_SCALE, band=band, pad_mask=pad,
                                                      causal=causal, k_descale=kd, v_descale=vd))
    return q, k, v, kd, vd, bounds, graph, out


@pytest.mark.parametrize("case", WV.VARIANT_CASES, ids=[WV.case_id(c) for c in WV.VARIANT_CASES])
def test_count_probe(case):
    dt, kind, dqk, dv = case
    dtype = WV.DTYPE[dt]
    nsplit = WV.plan(B, H, CAP, dqk, dv, torch.cuda.get_device_properties(0).multi_processor_count)["nsplit"]
    pad = left_pad(B, CAP, device="cuda")
    for N, band, causal in ROW_BANDS:
        q, k, v, kd, vd, bounds, graph, out = _probe_graph(case, N, band, causal, pad)
        for b0, b1 in WINDOWS:
            marks = WV.probe_marks(N, b0, b1, CAP, band, causal, nsplit)
            q1, k1, v1 = DV.count_operands(B, B, N, CAP, H, dqk, dv, marks, pad, kind == "e4m3", dtype,
                                           seed=N + b0 + band, device="cuda")
            for dst, src in ((q, q1), (k, k1), (v, v1)):
                dst.copy_(src)
            bounds.copy_(torch.tensor([b0, b1], dtype=torch.int32))
            graph.replay()
            in_range, live = WV.key_sets(B, N, b0, b1, CAP, band, causal, pad, device="cuda")
            _assert_bits(out, DV.count_expect(v.float(), H, in_range, live, dtype, vd),
                         f"count {WV.case_id(case)} N={N} band={band} causal={causal} window [{b0},{b1})")


@pytest.mark.parametrize("case", WV.VARIANT_CASES, ids=[WV.case_id(c) for c in WV.VARIANT_CASES])
def test_needle_probe(case):
    """Each row sees its own q channel (decode_variants.needle_channels), so a case takes at most dqk rows."""
    dt, kind, dqk, dv = case
    dtype = WV.DTYPE[dt]
    nsplit = WV.plan(B, H, CAP, dqk, dv, torch.cuda.get_device_properties(0).multi_processor_count)["nsplit"]
    pad = left_pad(B, CAP, device="cuda")
    for N, band, causal in ROW_BANDS:
        N = min(N, dqk)
        q, k, v, kd, vd, bounds, graph, out = _probe_graph(case, N, band, causal, pad)
        for b0, b1 in WINDOWS:
            cands = WV.needle_candidates(N, b0, b1, CAP, band, causal, nsplit, pad.cpu())
            in_range, live = WV.key_sets(B, N, b0, b1, CAP, band, causal, pad, device="cuda")
            bounds.copy_(torch.tensor([b0, b1], dtype=torch.int32))
            for r in range(WV.needle_rounds(cands, H)):
                nd = WV.needles(B, H, N, cands, r)
                q1, k1, v1 = DV.needle_operands(B, B, N, CAP, H, dqk, dv, nd, kind == "e4m3", dtype, seed=r + N,
                                                device="cuda")
                for dst, src in ((q, q1), (k, k1), (v, v1)):
                    dst.copy_(src)
                graph.replay()
                _assert_bits(out, DV.needle_expect(v.float(), H, in_range, live, nd, dtype, vd),
                             f"needle {WV.case_id(case)} N={N} band={band} causal={causal} window [{b0},{b1}) "
                             f"round {r}")


def test_attention_window_refusals():
    from perceiver_io_b200 import ops

    q = torch.zeros(1, 4, 64, dtype=torch.bfloat16, device="cuda")
    k = torch.zeros(1, 100, 64, dtype=torch.bfloat16, device="cuda")
    bounds = torch.tensor([0, 10], dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="needs causal"):
        ops.attention_window(q, k, k, bounds, 1, 1.0, band=4)
    with pytest.raises(ValueError, match="q's dtype"):
        ops.attention_window(q, k.half(), k.half(), bounds, 1, 1.0)
    with pytest.raises(ValueError, match="go with e4m3"):
        ops.attention_window(q, k, k, bounds, 1, 1.0, k_descale=torch.ones(1, device="cuda"),
                             v_descale=torch.ones(1, 64, device="cuda"))
    with pytest.raises(RuntimeError, match="more than 64 query rows"):
        ops.attention_window(torch.zeros(1, 65, 64, dtype=torch.bfloat16, device="cuda"), k, k, bounds, 1, 1.0)


# ---- the model loop ----------------------------------------------------------------------------------------------
N0, PREFIX, KEPT, REORDER_AT, VOCAB = 120, 90, 108, 28, 97
# ("s",) step; ("e", k) extend with k right tokens; ("d", k, m) a draft of k tokens whose last m are wrong, then
# rewind(m); ("o",) the beam reorder (at REORDER_AT fed tokens)
SCHEDULE = [("s",), ("e", 3), ("d", 5, 2), ("e", 5), ("e", 16), ("o",), ("s",), ("d", 16, 10), ("e", 64), ("e", 3),
            ("d", 3, 3), ("e", 5), ("s",)]


def _eager_loop(model, model64, fp64, arm, tokens0, pad0, cfg, monkeypatch, steps):
    """Per-token logits of the one-token loop: this package's eager cached loop ("bf16" / "fp8") or the fp64 model,
    with the beam reorder before the token at REORDER_AT."""
    import perceiver_io_b200 as P
    from perceiver_io_b200 import modules

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
        o = call(tokens[:, :N0], PREFIX, pad[:, :N0], [])
        out.append(o.logits[:, -1].double())
        cache = o.kv_cache
        for s, w in enumerate(P.decode_windows(N0, PREFIX, steps, cfg.max_seq_len, cfg.max_latents)):
            n, nlat = w.ca_end - w.ca_begin, w.sa_end - w.sa_begin
            cache = ([(cache[0][0][:, -(n - 1):], cache[0][1][:, -(n - 1):])]
                     + [(k[:, -(nlat - 1):], v[:, -(nlat - 1):]) for k, v in cache[1:]])
            if s == REORDER_AT:
                idx = torch.tensor([1, 0], device="cuda")
                cache = [(k.index_select(0, idx), v.index_select(0, idx)) for k, v in cache]
                tokens, pad = tokens[idx], pad[idx]
            pos = N0 + s
            o = call(tokens[:, pos:pos + 1], w.prefix_len, pad[:, pos + 1 - n:pos + 1], cache)
            out.append(o.logits[:, -1].double())
            cache = o.kv_cache
    return torch.stack(out, dim=1)          # (B, 1 + steps, vocab): [0] after the prompt, [1 + s] after token N0 + s


def _graphed_loop(model, kind, tokens0, pad0):
    import perceiver_io_b200 as P

    tokens = tokens0.clone()
    dec = P.GraphedDecoder(model, batch=2, max_new_tokens=KEPT, kv_cache=kind)
    got = {0: dec.prefill(tokens[:, :N0], PREFIX, pad0[:, :N0]).double()}
    fed = 0
    for op in SCHEDULE:
        if op[0] == "o":
            assert fed == REORDER_AT
            idx = torch.tensor([1, 0], device="cuda")
            dec.reorder(idx)
            tokens = tokens[idx]
            continue
        k = 1 if op[0] == "s" else op[1]
        feed = tokens[:, N0 + fed:N0 + fed + k].clone()
        wrong = op[2] if op[0] == "d" else 0
        if wrong:
            feed[:, k - wrong:] = (feed[:, k - wrong:] + 1) % VOCAB
        torch.cuda.set_sync_debug_mode("error")
        try:
            logits = dec.step(feed) if op[0] == "s" else dec.extend(feed)
            logits = logits[:, None] if op[0] == "s" else logits
            kept = logits[:, :k - wrong].double().clone()
            if wrong:
                dec.rewind(wrong)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        for i in range(k - wrong):
            got[fed + 1 + i] = kept[:, i]
        fed += k - wrong
    assert fed == KEPT and sorted(got) == list(range(KEPT + 1))
    assert dec.captures == len({1 if op[0] == "s" else op[1] for op in SCHEDULE if op[0] != "o"})
    with pytest.raises(RuntimeError, match="0 of max_new_tokens"):
        dec.extend(tokens[:, :2])
    with pytest.raises(ValueError, match="rewind"):
        dec.rewind(KEPT + 1)
    dec.rewind(3)                                  # gives three tokens back: one more 3-token step fits
    dec.extend(tokens[:, N0 + KEPT - 3:N0 + KEPT])
    return torch.stack([got[i] for i in range(KEPT + 1)], dim=1)


@pytest.mark.parametrize("abs_pos_emb", [False, True], ids=["rotary", "abs_pos"])
def test_graphed_extend_and_rewind_match_the_fp64_one_token_loop(monkeypatch, abs_pos_emb):
    cfg, model = _model(abs_pos_emb)
    model64 = copy.deepcopy(model).double()
    fp64 = _Fp64Attend(model64, _owners(model64))
    tokens0 = torch.randint(0, VOCAB, (2, N0 + KEPT + 1)).cuda()
    pad0 = torch.zeros(2, tokens0.shape[1], dtype=torch.bool, device="cuda")
    pad0[1, :7] = True
    truth = _eager_loop(model, model64, fp64, "fp64", tokens0, pad0, cfg, monkeypatch, KEPT)
    scale = truth.abs().max().item()
    for kind in ("bf16", "fp8"):
        e = (_eager_loop(model, model64, fp64, kind, tokens0, pad0, cfg, monkeypatch, KEPT) - truth).abs().max().item()
        got = _graphed_loop(model, kind, tokens0, pad0)
        assert torch.isfinite(got).all()
        err = (got - truth).abs().amax(dim=(0, 2))
        print(f"[parity] graphed {kind} extend/rewind: err {err.max().item():.3e}, eager {kind} err {e:.3e}, "
              f"max|logit| {scale:.3e}")
        assert (err <= 2.0 * e + 1e-3 * scale).all(), (kind, err.max().item(), e, scale, err.argmax().item())
