"""GPU checks of the device beam search: ``ops.beam_step`` against the numpy oracle bit for bit over chained steps,
``ops.kv_gather_rows`` against ``index_select`` of the parents, and ``GraphedDecoder.beam_search`` end to end against an
independent loop (``step`` on a second decoder, the oracle on its logits and the whole-arena ``reorder``)."""
import numpy as np
import pytest
import torch

from oracle import beam_oracle as O

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}
# (K, V, eos, length_penalty, early_stopping)
CONFIGS = [(1, 389, (5,), 1.0, False), (2, 4, (), 1.0, False), (3, 6, (1, 2), 2.0, True), (3, 389, (5, 9), 0.0, False),
           (8, 16, (1, 2, 3), -0.5, "never"), (8, 32000, (7,), 2.0, "never"), (3, 32768, (), 1.0, True),
           (2, 389, (0, 1, 2, 3), 1.0, "never"), (3, 389, (5,), 0.6, "never"), (2, 16, (1, 2), 0.6, False),
           (3, 389, (5, 9), -0.3, True), (3, 389, (), 1.2, "never")]


def _state_tuple(st):
    return (st.running.cpu().numpy(), st.finished.cpu().numpy(), st.finished_flags.cpu().numpy().astype(bool),
            st.running_hist.cpu().numpy(), st.finished_hist.cpu().numpy(),
            st.item_flags.cpu().numpy().astype(bool), st.counters.cpu().numpy())


def _logits(R, V, dtype, gen, integer):
    if integer:   # integer values: many exact ties (the lowest flat index wins)
        return torch.randint(-4, 5, (R, V), generator=gen).to(dtype).cuda()
    return (torch.randn(R, V, generator=gen) * 3).to(dtype).cuda()


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
def test_beam_step_matches_the_oracle(dt, cfg):
    from perceiver_io_b200 import ops

    K, V, eos, lp, es = CONFIGS[cfg]
    B, n = 3, 6
    checked = flagged = 0
    for integer in (False, True):
        gen = torch.Generator().manual_seed(cfg * 10 + integer)
        fill = O.fill_value(eos, 0)
        st = ops.BeamState(B, K, len(eos), n + 1, fill, "cuda")
        st.reset(n)
        ref = O.init_state(B, K, n, n + 1, fill)
        for step in range(n):
            x = _logits(B * K, V, DTYPES[dt], gen, integer)
            tok, par = ops.beam_step(x, st, eos, lp, es)
            want_tok, want_par, fl = O.step(ref, x.float().cpu().numpy(), eos, lp, es)
            if fl.any():
                flagged += 1
                break
            assert np.array_equal(tok[:, 0].cpu().numpy(), want_tok), (step, integer)
            assert np.array_equal(par.cpu().numpy(), want_par), (step, integer)
            got = _state_tuple(st)
            want = (ref.running, ref.fin, ref.fin_flag, ref.run_hist, ref.fin_hist,
                    np.stack([ref.unsat, ref.done], 1), np.array([ref.gen, n, int(ref.all_done), 0]))
            for name, g, w in zip(("running", "finished", "flags", "run_hist", "fin_hist", "item", "counters"), got,
                                  want):
                assert np.array_equal(g.view(np.int32) if g.dtype == np.float32 else g,
                                      w.view(np.int32) if w.dtype == np.float32 else w), (name, step, integer, g, w)
            checked += 1
    assert checked >= 6 and flagged <= 1, (checked, flagged)


def test_launches_are_deterministic_and_graph_capture_changes_nothing():
    from perceiver_io_b200 import ops

    B, K, V, eos = 4, 3, 32000, (11, 12)
    gen = torch.Generator().manual_seed(5)
    xs = [_logits(B * K, V, torch.bfloat16, gen, False) for _ in range(3)]

    def run(graphed):
        st = ops.BeamState(B, K, len(eos), 8, 0, "cuda")
        st.reset(7)
        out = []
        x = xs[0].clone()
        if graphed:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                ops.beam_step(x, st, eos, 1.0, False)
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ops.beam_step(x, st, eos, 1.0, False)
            st.reset(7)
        for i in range(3):
            x.copy_(xs[i])
            if graphed:
                g.replay()
            else:
                ops.beam_step(x, st, eos, 1.0, False)
            out.append(tuple(t.clone() for t in (st.tokens, st.parents, st.running, st.finished, st.finished_hist)))
        return out

    a, b, c = run(False), run(False), run(True)
    for sa, sb, sc in zip(a, b, c):
        for ta, tb, tc in zip(sa, sb, sc):
            assert torch.equal(ta, tb) and torch.equal(ta, tc)
    # an item's result does not depend on the other items: the first item alone gives the same step
    st = ops.BeamState(1, K, len(eos), 8, 0, "cuda")
    st.reset(7)
    tok, par = ops.beam_step(xs[0][:K], st, eos, 1.0, False)
    assert torch.equal(tok, a[0][0][:K]) and torch.equal(par, a[0][1][:K])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float8_e4m3fn])
def test_kv_gather_rows_moves_only_the_generated_rows(dtype):
    from perceiver_io_b200 import ops

    R, cap = 6, 40
    gen = torch.Generator().manual_seed(1)

    def arena(C):
        return torch.randint(-100, 100, (R, cap, C), generator=gen).float().div(8).to(dtype).cuda()

    arenas = [arena(64), arena(128), arena(256)]
    first = [10, 25, 3]
    cols = [2, 8, 8]
    table = ops.KvGatherTable(list(zip(arenas, first, cols)))
    bounds = torch.zeros(R, 12, dtype=torch.int32, device="cuda")
    bounds[:, 2], bounds[:, 8] = 17, 30   # current rows of the two groups (the same for every beam row)
    cases = {"identity": [0, 1, 2, 3, 4, 5], "3-cycle": [1, 2, 0, 4, 5, 3], "many-to-one": [0, 0, 0, 5, 5, 3],
             "mixed": [2, 1, 1, 3, 3, 4]}
    for name, par in cases.items():
        before = [a.clone() for a in arenas]
        parents = torch.tensor(par, dtype=torch.int32, device="cuda")
        ops.kv_gather_rows(table, parents, bounds)
        for a, b0, f, c in zip(arenas, before, first, cols):
            cur = int(bounds[0, c])
            want = b0.clone()
            want[:, f:cur] = b0.index_select(0, parents.long())[:, f:cur]
            assert torch.equal(a.view(torch.uint8), want.view(torch.uint8)), name
        # undo for the next case
        for a, b0 in zip(arenas, before):
            a.copy_(b0)


# ---- the decoder ------------------------------------------------------------------------------------------------------
N0, PREFIX, EOS = 150, 110, 7   # both windows slide: 150 + 10 > 160 rows, 40 + 8 > 48 latents


def _reference(model, kind, ids, pad, K, n, eos, lp, es, R):
    """step on a second decoder, the oracle on its logits, and the whole-arena reorder."""
    import perceiver_io_b200 as P

    B = ids.shape[0]
    dec = P.GraphedDecoder(model, batch=B * K, max_new_tokens=n, kv_cache=kind)
    logits = dec.prefill(ids.repeat_interleave(K, 0), PREFIX, pad.repeat_interleave(K, 0))
    st = O.init_state(B, K, n, n + 1, O.fill_value(eos, None))
    flagged = False
    for t in range(n):
        tok, par, fl = O.step(st, logits.float().cpu().numpy(), eos, lp, es)
        flagged |= bool(fl.any())
        if t == n - 1:
            break
        dec.reorder(torch.from_numpy(par.astype(np.int64)).cuda())
        logits = dec.step(torch.from_numpy(tok).cuda()[:, None])
    return st.fin_hist[:, :R, :n], st.fin[:, :R], flagged, st


@pytest.mark.parametrize("kind", ["bf16", "fp8"])
def test_beam_search_matches_the_independent_loop(kind):
    import perceiver_io_b200 as P
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    K, B, n, R = 3, 2, 24, 3
    torch.manual_seed(8)
    ids = torch.randint(0, 97, (B, N0)).cuda()
    pad = torch.zeros(B, N0, dtype=torch.bool, device="cuda")
    pad[1, :9] = True
    checked = 0
    for eos, lp, es in (((EOS,), 1.0, False), ((EOS, 3), 2.0, True), ((), 1.0, "never")):
        dec = P.GraphedDecoder(model, batch=B * K, max_new_tokens=n, kv_cache=kind)
        prefill = dec.prefill

        def eager_prefill(*a, **kw):   # the eager prompt pass is outside the sync-free contract
            old = torch.cuda.get_sync_debug_mode()
            torch.cuda.set_sync_debug_mode(0)
            try:
                return prefill(*a, **kw)
            finally:
                torch.cuda.set_sync_debug_mode(old)

        dec.prefill = eager_prefill
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = dec.beam_search(ids, PREFIX, n, num_beams=K, pad_mask=pad, eos_token_id=list(eos) or None,
                                  length_penalty=lp, early_stopping=es, num_return_sequences=R, check_every=4)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert dec.captures == 1
        assert out.sequences.shape == (B, R, n) and out.scores.shape == (B, R)
        # stopping at every replay or never gives the same output
        if eos:
            again = dec.beam_search(ids, PREFIX, n, num_beams=K, pad_mask=pad, eos_token_id=list(eos),
                                    length_penalty=lp, early_stopping=es, num_return_sequences=R, check_every=1)
            full = dec.beam_search(ids, PREFIX, n, num_beams=K, pad_mask=pad, eos_token_id=list(eos),
                                   length_penalty=lp, early_stopping=es, num_return_sequences=R, check_every=n)
            assert torch.equal(again.sequences, full.sequences) and torch.equal(again.scores, full.scores)
            assert torch.equal(again.sequences, out.sequences) and torch.equal(again.scores, out.scores)
            scratch = [t.data_ptr() for t in dec._beam_table.scratch]
            dec.beam_search(ids, PREFIX, n, num_beams=K, pad_mask=pad, eos_token_id=list(eos), length_penalty=lp,
                            early_stopping=es, num_return_sequences=R)
            assert [t.data_ptr() for t in dec._beam_table.scratch] == scratch   # reused, not reallocated
        seqs, scores, flagged, _ = _reference(model, kind, ids, pad, K, n, eos, lp, es, R)
        if flagged:
            continue
        assert np.array_equal(out.sequences.cpu().numpy(), seqs), (eos, lp, es)
        assert np.array_equal(out.scores.cpu().numpy().view(np.int32), scores.view(np.int32)), (eos, lp, es)
        checked += 1
    assert checked >= 2


def test_an_eos_fires_mid_run():
    """With a frequent EOS the finished hypotheses end before n and are filled after their end."""
    import perceiver_io_b200 as P
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    K, B, n = 3, 2, 24
    torch.manual_seed(8)
    ids = torch.randint(0, 97, (B, N0)).cuda()
    pad = torch.zeros(B, N0, dtype=torch.bool, device="cuda")
    dec = P.GraphedDecoder(model, batch=B * K, max_new_tokens=n, kv_cache="bf16")
    logits = dec.prefill(ids.repeat_interleave(K, 0), PREFIX, pad.repeat_interleave(K, 0))
    # the EOS: a token the model ranks high after the prompt, so hypotheses end early
    eos = int(logits[0].float().topk(3).indices[1])
    out = dec.beam_search(ids, PREFIX, n, num_beams=K, pad_mask=pad, eos_token_id=eos, pad_token_id=0,
                          num_return_sequences=K, check_every=2)
    seqs = out.sequences.cpu().numpy()
    ended = (seqs == eos).any(-1)
    assert ended.any()
    for b, r in zip(*np.nonzero(ended)):
        end = int((seqs[b, r] == eos).argmax())
        assert (seqs[b, r, end + 1:] == eos).all()   # pad_token_id 0: 🤗 fills with eos_token_id[0]
    seqs_ref, scores_ref, flagged, _ = _reference(model, "bf16", ids, pad, K, n, (eos,), 1.0, False, K)
    if not flagged:
        fill_fixed = np.where(seqs_ref == O.fill_value((eos,), None), O.fill_value((eos,), 0), seqs_ref)
        assert np.array_equal(seqs, fill_fixed)
