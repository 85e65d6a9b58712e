"""-m gpu: per-batch-row device rows (pcv_dev_rows.bounds_stride_b) and GraphedDecoder's per-row rewind.

Kernels: for every instantiation of the window attention, the window decode, the append into bf16 / e4m3 arenas and the
rotary (a key into an arena, q into a buffer, bf16 and e4m3 output), a call whose batch rows read their own bounds
through a strided (B, groups, 6) view equals, row by row and bit for bit, the shared-bounds call of the same batch with
that row's bounds; two launches are bit-identical.  The rows' bounds differ: an empty window, the whole arena, a begin
that is not tile-aligned, windows that split unevenly, a band that cuts one row's keys and not another's.

Model loop: three batch rows, one left-padded, fed through step, extend and drafts whose wrong-token count differs per
row (0 and k included), with a beam reorder after unequal rewinds, match the fp64 one-token loop of test_gpu_window.py at
every kept token index of every row, without a host synchronisation and with one capture per distinct step length;
equal per-row counts give the scalar rewind's logits bit for bit; the budget runs out exactly at the furthest row."""
import pytest
import torch

import window_variants as WV
from cached_fp8_variants import left_pad
from test_gpu_fp8_kv_cache import _Fp64Attend, _owners
from test_gpu_graph_decode import _model
import test_gpu_window as GW

pytestmark = pytest.mark.gpu

B, H, CAP, SCALE = 4, 2, 1000, 0.3
# per batch row (begin, end): an empty window, the whole arena, an unaligned begin over nine tiles (uneven splits),
# 65 keys at an unaligned begin
ROW_WINDOWS = [(50, 50), (0, CAP), (37, 613), (301, 366)]


def _state(cols, values, group=1):
    """A (B, 2, 6) int32 state whose group `group` holds values[b] in `cols`; returns it and the strided (B, 6) view
    of that group (row stride 12)."""
    st = torch.full((B, 2, 6), -7, dtype=torch.int32)
    for b, v in enumerate(values):
        st[b, group, cols] = torch.tensor(v, dtype=torch.int32)
    st = st.cuda()
    return st, st[:, group]


def _bits(t):
    return t.view(torch.uint8) if t.element_size() == 1 else t.view(torch.int16)


def _rowwise_equal(per_row, shared_of_row, what):
    for b in range(B):
        got, want = _bits(per_row[b]), _bits(shared_of_row(b)[b])
        assert torch.equal(got, want), f"{what}: batch row {b} differs from the shared call with its bounds"


def _per_row_vs_shared(call, view, cols, what):
    """call(bounds) -> output; the per-row call against B shared calls, plus a second per-row launch."""
    out = call(view[:, cols]).clone()
    again = call(view[:, cols])
    assert torch.equal(_bits(out), _bits(again)), f"{what}: two launches differ"
    _rowwise_equal(out, lambda b: call(view[b, cols].clone()).clone(), what)


# (rows, band): a band of 100 cuts the 576-key window's keys but not the 65-key one's
WINDOW_ROWS = [(1, 0), (5, 0), (64, 0), (5, 100), (17, 1), (64, 64)]


@pytest.mark.parametrize("case", WV.VARIANT_CASES, ids=[WV.case_id(c) for c in WV.VARIANT_CASES])
def test_window_kernel_reads_every_rows_bounds(case):
    from perceiver_io_b200 import ops

    dt, kind, dqk, dv = case
    pad = left_pad(B, CAP, device="cuda")
    st, view = _state(slice(0, 2), ROW_WINDOWS)
    for N, band in WINDOW_ROWS:
        for Bq in (B, 1):   # a batch-1 q still reads the bounds of the arena's batch row
            q, k, v, kd, vd, _, _ = WV.random_operands(B, Bq, N, CAP, H, dqk, dv, dt, kind, seed=N + band + Bq,
                                                       device="cuda")
            call = lambda bounds: ops.attention_window(q, k, v, bounds, H, SCALE, band=band, pad_mask=pad, causal=True,
                                                       k_descale=kd, v_descale=vd)
            _per_row_vs_shared(call, view, slice(0, 2), f"window {WV.case_id(case)} N={N} band={band} Bq={Bq}")
        out = ops.attention_window(q, k, v, view[:, 0:2], H, SCALE, band=band, pad_mask=pad, causal=True,
                                   k_descale=kd, v_descale=vd)
        assert (out[0] == 0).all(), "an empty window writes zeros"


@pytest.mark.parametrize("case", WV.VARIANT_CASES, ids=[WV.case_id(c) for c in WV.VARIANT_CASES])
def test_window_decode_reads_every_rows_bounds(case):
    from perceiver_io_b200 import ops

    dt, kind, dqk, dv = case
    pad = left_pad(B, CAP, device="cuda")
    st, view = _state(slice(0, 2), ROW_WINDOWS)
    for N in (1, 2, 4):
        q, k, v, kd, vd, _, _ = WV.random_operands(B, B, N, CAP, H, dqk, dv, dt, kind, seed=7 * N, device="cuda")
        call = lambda bounds: ops.attention_decode_window(q, k, v, bounds, H, SCALE, pad_mask=pad, causal=True,
                                                          k_descale=kd, v_descale=vd)
        _per_row_vs_shared(call, view, slice(0, 2), f"decode window {WV.case_id(case)} N={N}")


@pytest.mark.parametrize("arena", ["bf16", "e4m3"])
def test_append_writes_every_rows_rows(arena):
    from perceiver_io_b200 import ops

    C, n, cap = 64, 3, 80
    fp8 = arena == "e4m3"
    g = torch.Generator(device="cpu").manual_seed(5)
    k_new = torch.randn(B, n, C, generator=g).bfloat16().cuda()
    v_new = torch.randn(B, n, C, generator=g).bfloat16().cuda()
    inv = (torch.rand(C, generator=g) * 4 + 1).cuda() if fp8 else None
    kvt = torch.float8_e4m3fn if fp8 else torch.bfloat16
    base_k = torch.randn(B, cap, C, generator=g).to(kvt).cuda()
    base_v = torch.randn(B, cap, C, generator=g).to(kvt).cuda()
    st, view = _state(slice(2, 3), [[0], [17], [cap - 1], [41]])   # row cap - 1: two of its three rows are skipped

    def call(row):
        K, V = base_k.clone(), base_v.clone()
        ops.kv_append_at(K, V, k_new, v_new, row, *((inv, inv) if fp8 else ()))
        return torch.cat([K, V], dim=2)

    _per_row_vs_shared(call, view, slice(2, 3), f"append into {arena}")
    got = call(view[:, 2:3])
    assert torch.equal(_bits(got[1, 17 + n:]), _bits(torch.cat([base_k, base_v], dim=2)[1, 17 + n:]))


@pytest.mark.parametrize("out_kind", ["bf16", "e4m3"])
@pytest.mark.parametrize("target", ["key_into_arena", "q_into_buffer"])
def test_rotary_rotates_every_row_at_its_rows(out_kind, target):
    from perceiver_io_b200 import ops

    Hr, d, n, cap = 2, 64, 3, 80
    g = torch.Generator(device="cpu").manual_seed(9)
    x = torch.randn(B, n, Hr * d, generator=g).bfloat16().cuda()
    table = ops.rotary_angle_table(1.0 / (10000 ** (torch.arange(0, d // 2, 2).float() / (d // 2))), cap).cuda()
    fp8 = out_kind == "e4m3"
    inv = (torch.rand(Hr, generator=g) + 0.5).cuda() if fp8 else None
    odt = torch.float8_e4m3fn if fp8 else torch.bfloat16
    rows_out = cap if target == "key_into_arena" else n
    base = torch.randn(B, rows_out, Hr * d, generator=g).to(odt).cuda()
    flag = 1 if target == "key_into_arena" else 0
    st, view = _state(slice(2, 4), [[0, flag], [23, flag], [cap - 2, flag], [60, flag]])

    def call(rows):
        out = base.clone()
        return ops.rotary_apply_at(x, Hr, table, rows, out, inv)

    _per_row_vs_shared(call, view, slice(2, 4), f"rotary {target} -> {out_kind}")


def test_per_row_bounds_refusals():
    from perceiver_io_b200 import ops

    q = torch.zeros(B, 4, 64, dtype=torch.bfloat16, device="cuda")
    k = torch.zeros(B, 100, 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match=r"\(4, 2\) per row"):
        ops.attention_window(q, k, k, torch.zeros(B - 1, 2, dtype=torch.int32, device="cuda"), 1, 1.0)
    with pytest.raises(ValueError, match="unit stride"):
        ops.attention_decode_window(q, k, k, torch.zeros(2, B, dtype=torch.int32, device="cuda").t(), 1, 1.0)
    with pytest.raises(ValueError, match=r"\(4, 1\) per row"):
        ops.kv_append_at(k, k, q[:, :1], q[:, :1], torch.zeros(B, 0, dtype=torch.int32, device="cuda"))


# ---- the model loop ----------------------------------------------------------------------------------------------
ROWS, T, VOCAB = 3, 64, GW.VOCAB
# ("s",) step; ("e", k) extend with k right tokens; ("d", k, wrong) a draft of k tokens whose last wrong[b] are wrong in
# row b, then rewind(wrong); ("o", idx) the beam reorder
SCHEDULE = [("s",), ("e", 3), ("d", 5, [0, 2, 5]), ("e", 4), ("d", 8, [8, 0, 3]), ("o", [2, 0, 1]), ("s",),
            ("d", 16, [10, 16, 0]), ("e", 16), ("d", 3, [1, 1, 1]), ("e", 5), ("s",)]


def _graphed_rows(model, kind, tokens0, pad0, schedule, scalar_when_equal=False):
    """{(source row, token index): logits} of a GraphedDecoder driven through `schedule`, and the decoder."""
    import perceiver_io_b200 as P

    N0, PREFIX = GW.N0, GW.PREFIX
    tokens = tokens0.clone()
    src = list(range(ROWS))        # the row of tokens0 whose sequence batch row b carries
    dec = P.GraphedDecoder(model, batch=ROWS, max_new_tokens=T, kv_cache=kind)
    first = dec.prefill(tokens[:, :N0], PREFIX, pad0[:, :N0]).double()
    got = {(b, 0): first[b] for b in range(ROWS)}
    fed = [0] * ROWS
    for op in schedule:
        if op[0] == "o":
            idx = torch.tensor(op[1], device="cuda")
            dec.reorder(idx)
            tokens = tokens[idx]
            src, fed = [src[i] for i in op[1]], [fed[i] for i in op[1]]
            continue
        k = 1 if op[0] == "s" else op[1]
        wrong = op[2] if op[0] == "d" else [0] * ROWS
        feed = torch.stack([tokens[b, N0 + fed[b]:N0 + fed[b] + k] for b in range(ROWS)])
        for b in range(ROWS):
            if wrong[b]:
                feed[b, k - wrong[b]:] = (feed[b, k - wrong[b]:] + 1) % VOCAB
        torch.cuda.set_sync_debug_mode("error")
        try:
            logits = dec.step(feed)[:, None] if op[0] == "s" else dec.extend(feed)
            kept = logits.double().clone()
            if any(wrong):
                if scalar_when_equal and len(set(wrong)) == 1:
                    dec.rewind(wrong[0])
                else:
                    dec.rewind(wrong)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        for b in range(ROWS):
            for i in range(k - wrong[b]):
                got[(src[b], fed[b] + 1 + i)] = kept[b, i]
            fed[b] += k - wrong[b]
    assert dec.captures == len({1 if op[0] == "s" else op[1] for op in schedule if op[0] != "o"})
    assert dec._fed == max(fed) and dec._remaining == T - max(fed)
    return got, dec, tokens, fed


@pytest.mark.parametrize("abs_pos_emb", [False, True], ids=["rotary", "abs_pos"])
def test_per_row_rewind_matches_the_fp64_one_token_loop(monkeypatch, abs_pos_emb):
    import copy

    cfg, model = _model(abs_pos_emb)
    model64 = copy.deepcopy(model).double()
    fp64 = _Fp64Attend(model64, _owners(model64))
    torch.manual_seed(11)
    tokens0 = torch.randint(0, VOCAB, (ROWS, GW.N0 + T + 1)).cuda()
    pad0 = torch.zeros(ROWS, tokens0.shape[1], dtype=torch.bool, device="cuda")
    pad0[1, :7] = True
    monkeypatch.setattr(GW, "REORDER_AT", -1)   # the rows' sequences are independent: no reorder in the reference
    truth = GW._eager_loop(model, model64, fp64, "fp64", tokens0, pad0, cfg, monkeypatch, T)
    scale = truth.abs().max().item()
    for kind in ("bf16", "fp8"):
        e = (GW._eager_loop(model, model64, fp64, kind, tokens0, pad0, cfg, monkeypatch, T) - truth).abs().max().item()
        got, dec, tokens, fed = _graphed_rows(model, kind, tokens0, pad0, SCHEDULE)
        assert len({f for f in fed}) > 1, "the schedule leaves the rows at different counts"
        worst = 0.0
        for (row, t), logits in got.items():
            assert torch.isfinite(logits).all(), (kind, row, t)
            err = (logits - truth[row, t]).abs().max().item()
            worst = max(worst, err)
            assert err <= 2.0 * e + 1e-3 * scale, (kind, row, t, err, e, scale)
        assert len(got) == sum(f + 1 for f in fed)
        print(f"[parity] graphed {kind} per-row rewind: err {worst:.3e}, eager {kind} err {e:.3e}, "
              f"max|logit| {scale:.3e}")
        # the budget: the furthest row has T - max(fed) tokens left, the others more
        left = T - max(fed)
        with pytest.raises(RuntimeError, match=f"{left} of max_new_tokens={T} tokens remain"):
            dec.extend(torch.zeros(ROWS, left + 1, dtype=torch.long, device="cuda"))
        dec.extend(torch.stack([tokens[b, GW.N0 + fed[b]:GW.N0 + fed[b] + left] for b in range(ROWS)]))
        assert dec._remaining == 0
        with pytest.raises(ValueError, match="CUDA tensor"):
            dec.rewind(torch.zeros(ROWS, dtype=torch.long, device="cuda"))


def test_equal_per_row_counts_are_the_scalar_rewind():
    _, model = _model(False)
    torch.manual_seed(12)
    tokens0 = torch.randint(0, VOCAB, (ROWS, GW.N0 + T + 1)).cuda()
    pad0 = torch.zeros(ROWS, tokens0.shape[1], dtype=torch.bool, device="cuda")
    pad0[2, :5] = True
    schedule = [("e", 4), ("d", 6, [2, 2, 2]), ("s",), ("d", 5, [5, 5, 5]), ("e", 7), ("d", 3, [1, 1, 1]), ("s",)]
    for kind in ("bf16", "fp8"):
        a, _, _, _ = _graphed_rows(model, kind, tokens0, pad0, schedule)
        b, _, _, _ = _graphed_rows(model, kind, tokens0, pad0, schedule, scalar_when_equal=True)
        assert a.keys() == b.keys()
        for key in a:
            assert torch.equal(a[key], b[key]), (kind, key)
