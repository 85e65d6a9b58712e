"""GPU checks of the device logits processors: ``ops.process_logits`` against the numpy oracle bit for bit, its
determinism under repeated launches and graph replay, the neutral log-softmax mode chained into
``ops.beam_step(logprobs=True)`` against ``ops.beam_step``, and ``GraphedDecoder.generate`` / ``beam_search`` with
processors end to end against independent loops (``step`` on a second decoder, the oracle processors, greedy or the
beam oracle)."""
from unittest import mock

import numpy as np
import pytest
import torch

import process_oracle as P
from oracle import beam_oracle as O
from oracle import contrastive_oracle as CO

pytestmark = pytest.mark.gpu

_LOG_SOFTMAX = O.log_softmax   # the beam oracle's own, kept before any patch

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def _hist(R, cap, V, gen):
    """(R, cap) int64 histories with many repeats, pad ids (-1) and out-of-range ids."""
    h = torch.randint(0, min(V, 6), (R, cap), generator=gen)
    wide = torch.randint(0, V, (R, cap), generator=gen)
    h = torch.where(torch.rand(R, cap, generator=gen) < 0.5, h, wide)
    h[:, :3] = -1
    h[0, 5] = V + 3
    return h


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("V", [97, 1000, 32768])
def test_process_logits_matches_the_oracle(dt, V):
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(V)
    R, cap, tcap = 4, 4700, 40
    x = (torch.randn(R, V, generator=gen) * 3).to(DTYPES[dt])
    pre, tail = _hist(R, cap, V, gen), _hist(R, tcap, V, gen)
    lens = torch.tensor([0, 7, 1300, 4600], dtype=torch.int32)
    tl = torch.tensor([9], dtype=torch.int32)
    xf = x.float().numpy()
    for theta, N, M in ((1.0, 0, 0), (1.3, 0, 0), (0.8, 1, 0), (1.0, 2, 0), (1.2, 3, 5), (2.5, 4, 0), (1.1, 5, 9000),
                        (1.0, 8, 0)):
        for use_tail in (False, True):
            kw = dict(repetition_penalty=theta, no_repeat_ngram_size=N, min_new_tokens=M, prompt_len=3,
                      eos=(2, V - 1) if M else ())
            extra = dict(tail=tail.cuda(), tail_len=tl.cuda()) if use_tail else {}
            got = ops.process_logits(x.cuda(), pre.cuda(), lens.cuda(), **extra, **kw).cpu().numpy()
            for r in range(R):
                h = pre[r, :lens[r]].tolist() + (tail[r, :9].tolist() if use_tail else [])
                want = P.process(xf[r], h, **{k: v for k, v in kw.items() if k != "eos"}, eos=kw["eos"])
                np.testing.assert_array_equal(got[r].view(np.uint32), want.view(np.uint32),
                                              err_msg=f"{dt} V={V} {theta, N, M} tail={use_tail} row {r}")


def test_row_map_rows_per_hist_and_log_softmax():
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(1)
    B, K, V = 3, 4, 389
    x = (torch.randn(B * K, V, generator=gen) * 4).bfloat16().cuda()
    pre = _hist(B, 50, V, gen).cuda()
    sel = torch.tensor([2, 0, 3], dtype=torch.int32).cuda()
    out = torch.full((B * K, V), 7.0, device="cuda")
    ops.process_logits(x, pre, 30, row_map=sel, out=out, repetition_penalty=1.4, no_repeat_ngram_size=2)
    xf, o = x.float().cpu().numpy(), out.cpu().numpy()
    for b in range(B):
        for j in range(K):
            r = b * K + j
            if j == int(sel[b]):
                want = P.process(xf[r], pre[b, :30].tolist(), repetition_penalty=1.4, no_repeat_ngram_size=2)
                np.testing.assert_array_equal(o[r].view(np.uint32), want.view(np.uint32))
            else:
                assert (o[r] == 7.0).all()   # rows the map does not name are untouched
    # rows_per_hist: row r = b*k + i sees history row b with its own length
    pos = torch.tensor([[3, 4], [10, 11], [40, 41]], dtype=torch.int32).cuda()
    got = ops.process_logits(x[:6], pre, pos.reshape(-1), rows_per_hist=2, no_repeat_ngram_size=1).cpu().numpy()
    for r in range(6):
        want = P.process(xf[r], pre[r // 2, :int(pos.view(-1)[r])].tolist(), no_repeat_ngram_size=1)
        np.testing.assert_array_equal(got[r].view(np.uint32), want.view(np.uint32))
    # log-softmax mode: the beam step's arithmetic, then the processors (elements the oracle cannot place exactly, at
    # an fp32 rounding boundary within its fp64 reach, are skipped)
    got = ops.process_logits(x, pre.repeat_interleave(K, 0), 30, log_softmax=True, repetition_penalty=1.2,
                             no_repeat_ngram_size=3).cpu().numpy()
    checked = 0
    for r in range(B * K):
        lp, amb = O.log_softmax(xf[r])
        want = P.process(lp, pre[r // K, :30].tolist(), repetition_penalty=1.2, no_repeat_ngram_size=3)
        ok = ~amb
        np.testing.assert_array_equal(got[r][ok].view(np.uint32), want[ok].view(np.uint32))
        checked += int(ok.sum())
    assert checked > B * K * V * 0.99


def test_repeated_launches_and_graph_replay_give_identical_bits():
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(2)
    V = 32768
    x = (torch.randn(8, V, generator=gen) * 3).bfloat16().cuda()
    pre = _hist(8, 3000, V, gen).cuda()
    lens = torch.full((8,), 2900, dtype=torch.int32).cuda()
    kw = dict(repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=4, prompt_len=2890, eos=(5,))
    first = ops.process_logits(x, pre, lens, **kw).clone()
    for _ in range(3):
        assert torch.equal(ops.process_logits(x, pre, lens, **kw), first)
    out = torch.empty_like(first)
    ops.process_logits(x, pre, lens, out=out, **kw)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.process_logits(x, pre, lens, out=out, **kw)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first)


@pytest.mark.parametrize("K,V,eos", [(3, 389, (5,)), (2, 32768, ()), (4, 97, (1, 2))])
def test_neutral_log_softmax_then_logprobs_step_equals_beam_step(K, V, eos):
    from perceiver_io_b200 import ops

    B, n = 2, 6
    gen = torch.Generator().manual_seed(K * V)
    st_a = ops.BeamState(B, K, len(eos), n + 1, 0, "cuda")
    st_b = ops.BeamState(B, K, len(eos), n + 1, 0, "cuda")
    st_a.reset(n)
    st_b.reset(n)
    pre = torch.zeros(B * K, 4, dtype=torch.long, device="cuda")
    for _ in range(n):
        x = (torch.randn(B * K, V, generator=gen) * 3).bfloat16().cuda()
        ta, pa = ops.beam_step(x, st_a, eos)
        lp = ops.process_logits(x, pre, 4, tail=st_b.running_hist.view(B * K, -1), tail_len=st_b.counters[0:1],
                                log_softmax=True)
        tb, pb = ops.beam_step(lp, st_b, eos, logprobs=True)
        assert torch.equal(ta, tb) and torch.equal(pa, pb)
        for f in ("running", "finished", "finished_flags", "running_hist", "finished_hist", "counters"):
            assert torch.equal(getattr(st_a, f), getattr(st_b, f)), f


# ---- the decoder ------------------------------------------------------------------------------------------------------
N0, PREFIX = 150, 110


def _ids(B):
    torch.manual_seed(8)
    ids = torch.randint(0, 97, (B, N0)).cuda()
    pad = torch.zeros(B, N0, dtype=torch.bool, device="cuda")
    pad[1, :9] = True
    return ids, pad


def _greedy_loop(model, kind, ids, pad, n, kw, eos=(), pad_token=None):
    """step on a second decoder, the oracle processors on its logits, the first maximal index, 🤗 _sample's EOS rule."""
    import perceiver_io_b200 as PK

    B = ids.shape[0]
    dec = PK.GraphedDecoder(model, batch=B, max_new_tokens=n + 1, kv_cache=kind)
    logits = dec.prefill(ids, PREFIX, pad)
    hist = [r for r in ids.tolist()]
    done = [False] * B
    out = []
    for t in range(n + 1):
        x = logits.float().cpu().numpy()
        tok = []
        for b in range(B):
            row = P.process(x[b], hist[b], prompt_len=N0, eos=eos, **kw)
            v = pad_token if done[b] else int(np.argmax(row))
            done[b] = done[b] or v in eos
            tok.append(v)
            hist[b].append(v)
        out.append(tok)
        if t == n:
            break
        logits = dec.step(torch.tensor(tok, device="cuda")[:, None])
    return np.array(out).T   # (B, n + 1): the first token, then n


@pytest.mark.parametrize("kind", ["bf16", "fp8"])
@pytest.mark.parametrize("abs_pos", [False, True], ids=["rotary", "abs_pos"])
def test_greedy_generate_with_processors_matches_the_loop(kind, abs_pos):
    import perceiver_io_b200 as PK
    from test_gpu_graph_decode import _model

    _, model = _model(abs_pos)
    B, n = 2, 20
    ids, pad = _ids(B)
    kw = dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=6)
    dec = PK.GraphedDecoder(model, batch=B, max_new_tokens=n + 1, kv_cache=kind)
    logits = dec.prefill(ids, PREFIX, pad)
    dec.set_seed(1)
    dec.set_sampling(0.0, **kw, eos_token_id=[4])
    first = dec.draw(logits)
    got = torch.cat([first, dec.generate(first, n, check_every=4)], 1).cpu().numpy()
    want = _greedy_loop(model, kind, ids, pad, n, kw, eos=(4,), pad_token=4)
    np.testing.assert_array_equal(got, want)


def test_eos_stop_pads_and_keeps_the_budget():
    import perceiver_io_b200 as PK
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    B, n = 2, 24
    ids, pad = _ids(B)
    dec = PK.GraphedDecoder(model, batch=B, max_new_tokens=n + 1, kv_cache="bf16")
    logits = dec.prefill(ids, PREFIX, pad)
    dec.set_sampling(0.0)
    plain = dec.generate(dec.draw(logits), n).cpu().numpy()
    # EOS ids: tokens the plain greedy run emits early in each row, so every row finishes
    eos = sorted({int(plain[0, 2]), int(plain[1, 2])})
    logits = dec.prefill(ids, PREFIX, pad)
    dec.set_sampling(0.0, eos_token_id=eos, pad_token_id=0)
    first = dec.draw(logits)
    got = dec.generate(first, n, check_every=2).cpu().numpy()
    used = n + 1 - dec._remaining
    want = _greedy_loop(model, "bf16", ids, pad, n, {}, eos=tuple(eos), pad_token=0)[:, 1:]
    np.testing.assert_array_equal(got, want)
    assert used < n   # stopped early: the replays not run stay in the budget
    assert used % 2 == 0 or used == n


def test_sample_k_sees_each_draft_prefix_and_a_rewind_redraws():
    """Draw i of sample(k) is processed with the prompt and the first i+1 drafts as history (🤗's assisted decoding),
    on the replay's own logits; a rewound row re-fed the same drafts draws the same tokens; reorder carries the
    history."""
    import perceiver_io_b200 as PK
    from perceiver_io_b200 import ops
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    B, k = 2, 5
    ids, pad = _ids(B)
    kw = dict(repetition_penalty=1.5, no_repeat_ngram_size=2)
    dec = PK.GraphedDecoder(model, batch=B, max_new_tokens=3 * k, kv_cache="bf16")
    dec.prefill(ids, PREFIX, pad)
    dec.set_seed(5)
    dec.set_sampling(0.9, 20, 0.95, **kw)
    drafts = torch.randint(0, 97, (B, k), generator=torch.Generator().manual_seed(0)).cuda()
    raw = dec.extend(drafts).float().cpu().numpy()   # the k-token graph's logits
    dec.rewind(k)
    toks, processed = dec.sample(drafts)
    toks, processed = toks.clone(), processed.clone()
    hist = ids.tolist()
    for b in range(B):
        for i in range(k):
            want = P.process(raw[b, i], hist[b] + drafts[b, :i + 1].tolist(), **kw)
            np.testing.assert_array_equal(processed[b, i].cpu().numpy().view(np.uint32), want.view(np.uint32))
    pos = (N0 + 1 + torch.arange(k, dtype=torch.int32, device="cuda")).repeat(B, 1)
    assert torch.equal(toks, ops.sample_tokens(processed, dec._seeds, pos, 0.9, 20, 0.95))
    dec.rewind(k)
    again, _ = dec.sample(drafts)
    assert torch.equal(again, toks)
    dec.reorder(torch.tensor([1, 0], device="cuda"))
    assert torch.equal(dec._tokens[:, :N0], ids.flip(0)) and torch.equal(dec._tokens[:, N0:N0 + k], drafts.flip(0))


def test_neutral_values_record_the_plain_graphs():
    import perceiver_io_b200 as PK
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    B, n = 2, 12
    ids, pad = _ids(B)
    out = []
    for kw in ({}, dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0)):
        dec = PK.GraphedDecoder(model, batch=B, max_new_tokens=n + 1, kv_cache="bf16")
        logits = dec.prefill(ids, PREFIX, pad)
        dec.set_seed(3)
        dec.set_sampling(0.8, 10, 0.9, **kw)
        first = dec.draw(logits)
        out.append(dec.generate(first, n))
        assert dec.captures == 1 and list(dec._graphs) == [("sample", 1, (0.8, 10, 0.9))]
    assert torch.equal(out[0], out[1])


def test_beam_search_with_processors_matches_the_loop():
    import perceiver_io_b200 as PK
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    K, B, n = 3, 2, 16
    ids, pad = _ids(B)
    eos = (7,)
    kw = dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=4)
    dec = PK.GraphedDecoder(model, batch=B * K, max_new_tokens=n, kv_cache="bf16")
    out = dec.beam_search(ids, PREFIX, n, num_beams=K, pad_mask=pad, eos_token_id=list(eos), num_return_sequences=K,
                          **kw)
    assert dec.captures == 1
    # the loop: step, the device log-softmax with the oracle processors' rows checked, the beam oracle on the rows
    ref = PK.GraphedDecoder(model, batch=B * K, max_new_tokens=n, kv_cache="bf16")
    logits = ref.prefill(ids.repeat_interleave(K, 0), PREFIX, pad.repeat_interleave(K, 0))
    st = O.init_state(B, K, n, n + 1, O.fill_value(eos, None))
    hist = [r for r in ids.repeat_interleave(K, 0).tolist()]
    flagged = False
    with mock.patch.object(O, "log_softmax", lambda x: (np.asarray(x, np.float32), np.zeros(len(x), bool))):
        for t in range(n):
            rows = []
            for r, x in enumerate(logits.float().cpu().numpy()):
                lp, amb = _LOG_SOFTMAX(x)
                flagged |= bool(amb.any())
                rows.append(P.process(lp, hist[r], prompt_len=N0, eos=eos, **kw))
            tok, par, fl = O.step(st, np.stack(rows), eos, 1.0, False)
            flagged |= bool(fl.any())
            hist = [hist[p % (B * K)] + [int(v)] for p, v in zip(par, tok)]
            if t == n - 1:
                break
            ref.reorder(torch.from_numpy(par.astype(np.int64)).cuda())
            logits = ref.step(torch.from_numpy(tok).cuda()[:, None])
    if flagged:
        pytest.skip("a decision lies within the oracle's rounding reach")
    assert np.array_equal(out.sequences.cpu().numpy(), st.fin_hist[:, :K, :n])
    assert np.array_equal(out.scores.cpu().numpy().view(np.int32), st.fin[:, :K].view(np.int32))



def test_sampled_generate_with_processors_matches_the_loop():
    """temperature, top-k and top-p after the processors: each draw equals ops.sample_tokens on the oracle-processed
    rows of a step loop, at the same seed and position (the sampler is a pure function of those)."""
    import perceiver_io_b200 as PK
    from perceiver_io_b200 import ops
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    B, n = 2, 20
    ids, pad = _ids(B)
    kw = dict(repetition_penalty=1.4, no_repeat_ngram_size=3, min_new_tokens=5)
    samp = (0.8, 12, 0.9)
    dec = PK.GraphedDecoder(model, batch=B, max_new_tokens=n + 1, kv_cache="bf16")
    logits = dec.prefill(ids, PREFIX, pad)
    dec.set_seed([7, 9])
    dec.set_sampling(*samp, **kw, eos_token_id=[4])
    first = dec.draw(logits)
    got = torch.cat([first, dec.generate(first, n)], 1).cpu().numpy()

    ref = PK.GraphedDecoder(model, batch=B, max_new_tokens=n + 1, kv_cache="bf16")
    logits = ref.prefill(ids, PREFIX, pad)
    seeds = torch.tensor([7, 9], device="cuda")
    hist = ids.tolist()
    done = [False] * B
    want = []
    for t in range(n + 1):
        x = logits.float().cpu().numpy()
        rows = np.stack([P.process(x[b], hist[b], prompt_len=N0, eos=(4,), **kw) for b in range(B)])
        pos = torch.full((B,), N0 + t, dtype=torch.int32, device="cuda")
        tok = ops.sample_tokens(torch.from_numpy(rows).cuda(), seeds, pos, *samp).tolist()
        tok = [4 if done[b] else tok[b] for b in range(B)]
        done = [done[b] or tok[b] == 4 for b in range(B)]
        for b in range(B):
            hist[b].append(tok[b])
        want.append(tok)
        if t < n:
            logits = ref.step(torch.tensor(tok, device="cuda")[:, None])
    np.testing.assert_array_equal(got, np.array(want).T)


def _contrastive_loop(model, ids, pad, K, n, alpha, eos, fill, kw):
    """contrastive_oracle's 4.28 loop with the oracle processors on each selected row before its candidates: step on a
    second decoder, the oracle ranking on its logits and hidden rows, the whole-arena reorder to the selected row."""
    import perceiver_io_b200 as PK

    B = ids.shape[0]
    dec = PK.GraphedDecoder(model, batch=B * K, max_new_tokens=n, kv_cache="bf16")
    out = dec._prefill(ids.repeat_interleave(K, 0), PREFIX, pad.repeat_interleave(K, 0))
    ctx = [r for r in out.last_hidden_state[::K].double().cpu().numpy()]
    x = out.logits[::K, -1].float().cpu().numpy()
    del out
    cpad = [r for r in pad[:, PREFIX:].cpu().numpy()]
    hist = ids.tolist()
    unfinished = [True] * B
    toks = np.full((B, n), fill, np.int64)
    flagged = np.zeros((B, n), bool)
    sel_prev = None
    for t in range(n):
        cand, probs, xs = np.zeros((B, K), np.int64), np.zeros((B, K)), []
        for b in range(B):
            xp = P.process(x[b], hist[b], prompt_len=N0, eos=eos, **kw)
            cand[b], probs[b], _ = CO.candidates(xp, K)
            xs.append(xp)
        if sel_prev is not None:
            dec.reorder(torch.from_numpy(np.repeat(np.arange(B) * K + sel_prev, K)).cuda())
        lg = dec.step(torch.from_numpy(cand.reshape(-1, 1)).cuda()).float().view(B, K, -1).cpu().numpy()
        hid = dec._hidden[:, -1].view(B, K, -1).double().cpu().numpy()
        sel = np.zeros(B, np.int64)
        for b in range(B):
            pen = CO.penalty(ctx[b], cpad[b], hid[b])
            sel[b], _, flagged[b, t] = CO.select(probs[b], pen, alpha, xs[b][cand[b]], hid[b], x.shape[-1],
                                                 hid.shape[-1])
            emit = int(cand[b, sel[b]]) if unfinished[b] else fill
            toks[b, t] = emit
            hist[b].append(emit)
            unfinished[b] = unfinished[b] and emit not in eos
            ctx[b] = np.concatenate([ctx[b], hid[b, sel[b]][None]])
            cpad[b] = np.concatenate([cpad[b], [False]])
            x[b] = lg[b, sel[b]]
        sel_prev = sel
    return toks, flagged


def test_contrastive_search_with_processors_matches_the_loop():
    import perceiver_io_b200 as PK
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    K, B, n = 4, 2, 24
    ids, pad = _ids(B)
    checked = 0
    for alpha, eos, kw in ((0.6, (), dict(repetition_penalty=1.3, no_repeat_ngram_size=2)),
                           (0.4, (5, 6), dict(repetition_penalty=0.8, no_repeat_ngram_size=3, min_new_tokens=6)),
                           (0.0, (), dict(no_repeat_ngram_size=1))):
        dec = PK.GraphedDecoder(model, batch=B * K, max_new_tokens=n, kv_cache="bf16")
        out = dec.contrastive_search(ids, PREFIX, n, penalty_alpha=alpha, top_k=K, pad_mask=pad,
                                     eos_token_id=list(eos) or None, pad_token_id=0, **kw).cpu().numpy()
        assert dec.captures == 1
        want, flagged = _contrastive_loop(model, ids, pad, K, n, alpha, eos, 0 if eos else -1, kw)
        for b in range(B):
            upto = int(np.argmax(flagged[b])) if flagged[b].any() else n
            assert np.array_equal(out[b, :upto], want[b, :upto]), (alpha, kw, b, upto, out[b], want[b])
            checked += upto
    print(f"[process] contrastive: {checked} of {3 * B * n} tokens checked against the loop")
    assert checked >= 2 * B * n, checked


def test_neutral_beam_and_contrastive_record_the_plain_graphs():
    """With every processor off beam_search and contrastive_search return what the plain call returns, from the plain
    graph: one capture, under the plain key."""
    import perceiver_io_b200 as PK
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    K, B, n = 3, 2, 12
    ids, pad = _ids(B)
    neutral = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0)
    outs = []
    for kw in ({}, neutral):
        dec = PK.GraphedDecoder(model, batch=B * K, max_new_tokens=n, kv_cache="bf16")
        r = dec.beam_search(ids, PREFIX, n, num_beams=K, pad_mask=pad, eos_token_id=7, num_return_sequences=K, **kw)
        assert dec.captures == 1 and list(dec._graphs) == [("beam", K, (7,), 1.0, "False")]
        c = dec.contrastive_search(ids, PREFIX, n, penalty_alpha=0.6, top_k=K, pad_mask=pad, **kw)
        assert dec.captures == 2 and list(dec._graphs) == [("contrastive", K, 0.6, (), -1)]
        outs.append((r.sequences, r.scores, c))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
