"""-m gpu: the vocabulary-row kernels on the probe rows of vocab_variants.py, compared with the exact oracles with no
tolerance: ops.sample_tokens (sample_kernel) token for token and log-probability bit for bit; pcv_spec_verify
(spec_verify_kernel) verdict for verdict; the beam step's row candidates (beam_rows_kernel's cand_scores /
cand_index) and its whole state after one step, through both entries; the contrastive candidates (cs_candidates_kernel)
id for id with probabilities within 4 ulp; ops.process_logits (process_kernel) bit for bit (in its log-softmax mode
too, but where the fp64 log-softmax lies within its reach of an fp32 rounding boundary).  And one decoder-level regression: a sampled generate whose n-gram blocking bans the whole
vocabulary."""
import numpy as np
import pytest
import torch

import process_oracle as PO
import vocab_variants as VV
from oracle import beam_oracle as BO
from oracle import contrastive_oracle as CO
from oracle import sample_oracle as S
from oracle import spec_oracle as SP

pytestmark = pytest.mark.gpu

TORCH = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def _dev(rows, dt, pad=24):
    """(R, V) probe rows as a strided CUDA tensor of the dtype (row stride V + pad)."""
    R, V = rows.shape
    buf = torch.full((R, V + pad), float("nan"), dtype=TORCH[dt], device="cuda")
    out = buf[:, :V]
    out.copy_(torch.from_numpy(rows))
    assert torch.equal(out.float().cpu(), torch.from_numpy(rows)), "a probe value is not representable"
    return out


def _sample_cases(V, dt):
    """(rows, T, top_k, top_p, expected tokens or None) groups of sampler probes at V, one launch each."""
    cases = []
    radix = VV.radix_probes(V, dt)
    for k in sorted({p.k for p in radix}):
        rows = [p.x for p in radix if p.k == k]
        cases.append((rows, 1.0, k, 1.0, None))
    every = [p.x for p in radix] + [p.x for p in VV.max_probes(V, dt, V)]
    every += [p.x for p in VV.zero_probes(V, max(1, V // 2), dt, V)] if V >= 3 else []
    every += [p.x for k in (1, V // 2) for p in VV.inf_probes(V, max(1, k), dt, V + k)]
    for top_k in (0, 1, V - 1, V, V + 5):
        cases.append((every, 1.0, max(top_k, 0), 1.0, None))
    for top_p in (0.5, 0.75):
        tp = [p.x for p in VV.top_p_probes(V, dt) if p.claim["top_p"] == top_p]
        if tp:
            cases.append((tp, 1.0, 0, top_p, None))
    for T in (1.0, 0.5):
        zm = [(p.x, tok) for p, t, tok in VV.zero_mass_probes(V, dt) if t == T]
        if zm:
            cases.append(([x for x, _ in zm], T, 0, 1.0, [tok for _, tok in zm]))
    return cases


def _launch_sample(rows, dt, T, top_k, top_p, seeds, pos):
    from perceiver_io_b200 import ops

    R = len(rows)
    per = 4
    n = -(-R // per) * per
    x = np.stack(rows + [rows[0]] * (n - R))
    logits = _dev(x, dt).unflatten(0, (n // per, per))
    s = torch.as_tensor(seeds[:n // per], dtype=torch.int64, device="cuda")
    p = torch.as_tensor(np.resize(pos, n).reshape(n // per, per), dtype=torch.int32, device="cuda")
    toks, lps = ops.sample_tokens(logits, s, p, T, top_k, top_p, logprobs=True)
    return toks.view(-1)[:R].cpu().numpy(), lps.view(-1)[:R].cpu().numpy(), per


@pytest.mark.parametrize("V", VV.VOCABS)
@pytest.mark.parametrize("dt", VV.DTYPES)
def test_sample_tokens_on_the_probes(dt, V):
    rng = np.random.default_rng(V)
    checked = 0
    for rows, T, top_k, top_p, want in _sample_cases(V, dt):
        seeds = rng.integers(-2 ** 63, 2 ** 63 - 1, size=len(rows) + 4, dtype=np.int64)
        pos = rng.integers(0, 2 ** 31 - 1, size=len(rows) + 4)
        toks, lps, per = _launch_sample(rows, dt, T, top_k, top_p, seeds, pos)
        for r, x in enumerate(rows):
            b = r // per
            d = S.sample_row(x, T, top_k, top_p, int(seeds[b]), b, int(pos[r]))
            assert not d.ambiguous, (dt, V, T, top_k, top_p, r, d.why)
            assert toks[r] == d.token, (dt, V, T, top_k, top_p, r, d, toks[r])
            assert np.float32(lps[r]).view(np.uint32) == np.float32(d.logprob).view(np.uint32), (dt, V, r, lps[r], d)
            if want is not None:
                assert d.token == want[r] and d.logprob == 0.0, (r, d)
            checked += 1
    assert checked > 0


@pytest.mark.parametrize("dt", VV.DTYPES)
def test_sample_tokens_draws_at_segment_boundaries_and_in_a_mass_one_run(dt):
    from perceiver_io_b200 import ops

    for probe, picks in VV.segment_draw_probes(dt):
        for pos, tok in picks:
            got = ops.sample_tokens(_dev(probe.x[None], dt), torch.full((1,), 5, dtype=torch.int64, device="cuda"),
                                    torch.full((1,), pos, dtype=torch.int32, device="cuda"), 1.0, 0, 1.0)
            assert int(got) == tok, (probe.name, pos, int(got), tok)
    p = VV.dense_draw_probe(dt)
    for seed, b, pos in VV.DENSE_DRAW:
        d = S.sample_row(p.x, 1.0, 0, 1.0, seed, b, pos)
        got, lp = ops.sample_tokens(_dev(p.x[None], dt), torch.full((1,), seed, dtype=torch.int64, device="cuda"),
                                    torch.full((1,), pos, dtype=torch.int32, device="cuda"), 1.0, logprobs=True)
        assert int(got) == d.token < VV.MAX_VOCAB - 1 and float(lp) == d.logprob, (pos, int(got), d)


# ---- speculative verification -----------------------------------------------------------------------------------------
def _spec_rows(V, dt):
    rows = [p.x for p in VV.radix_probes(V, dt)] + [p.x for p in VV.top_p_probes(V, dt)]
    zm = [p.x for p, T, _ in VV.zero_mass_probes(V, dt) if T == 1.0]
    return rows, zm


@pytest.mark.parametrize("V", [33, 513, 32768])
@pytest.mark.parametrize("dt", VV.DTYPES)
def test_spec_verify_on_the_probes(dt, V):
    from perceiver_io_b200 import ops

    rng = np.random.default_rng(V + 1)
    rows, zm = _spec_rows(V, dt)
    G = 2
    # batch rows: probe target and draft rows, then a zero-mass target row and a zero-mass draft row
    B = len(rows) // 2
    tgt = np.stack([rows[(3 * b + i) % len(rows)] for b in range(B) for i in range(G + 1)]).reshape(B, G + 1, V)
    drf = np.stack([rows[(5 * b + i + 1) % len(rows)] for b in range(B) for i in range(G)]).reshape(B, G, V)
    tgt[0, 0], drf[1, 0], tgt[2, 1], drf[3, 1] = zm[0], zm[0], zm[1], zm[0]
    for sampling, draft_sampling in (((1.0, 0, 1.0), (1.0, 0, 1.0)), ((1.0, 0, 0.5), (1.0, 0, 0.75))):
        seeds = rng.integers(0, 2 ** 62, size=B)
        pos = rng.integers(0, 2 ** 31 - 1, size=(B, G + 1))
        tokens = np.zeros((B, G + 1), np.int64)
        for b in range(B):
            tokens[b, 0] = rng.integers(0, V)
            for i in range(G):   # the draft's own draw, the target's argmax, or any id in [0, V] (V: out of range)
                kind = (b + i) % 3
                if kind == 0:
                    tokens[b, i + 1] = S.sample_row(drf[b, i], *draft_sampling, int(seeds[b]), b, int(pos[b, i])).token
                elif kind == 1:
                    tokens[b, i + 1] = int(np.argmax(tgt[b, i]))
                else:
                    tokens[b, i + 1] = rng.integers(0, V + 1)
        out, acc = ops.spec_verify(_dev(tgt.reshape(-1, V), dt).unflatten(0, (B, G + 1)),
                                   _dev(drf.reshape(-1, V), dt).unflatten(0, (B, G)),
                                   torch.from_numpy(tokens).cuda(), torch.from_numpy(seeds).cuda(),
                                   torch.from_numpy(pos.astype(np.int32)).cuda(), sampling, draft_sampling)
        out, acc = out.cpu().numpy(), acc.cpu().numpy()
        for b in range(B):
            v = SP.verify_row(tgt[b], drf[b], tokens[b], sampling, draft_sampling, int(seeds[b]), b, pos[b])
            assert not v.ambiguous, (b, v.why)
            assert out[b].tolist() == v.tokens and acc[b] == v.n, (dt, V, sampling, b, out[b], v)


# ---- beam step ----------------------------------------------------------------------------------------------------------
def _radix_at(V, k, dt):
    return [VV.radix_probe(V, k, byte, neg, dt, seed=V + k + byte).x for byte in range(4 if dt == "fp32" else 2)
            for neg in (False, True)]


def _beam_rows(V, nsel, dt):
    rows = _radix_at(V, nsel, dt)
    rows += [p.x for p in VV.tie_probes(V, nsel, dt, V)]
    rows += [p.x for p in VV.inf_probes(V, nsel, dt, V + 1)] if nsel <= V else []
    rows += [p.x for p in VV.zero_probes(V, min(nsel, V - 1), dt, V + 2)] if V >= 3 else []
    return rows


def _check_beam(V, K, E, rows, dt, logprobs):
    from perceiver_io_b200 import ops

    keep = VV.beams_to_keep(K, E)
    B = -(-len(rows) // K)
    x = np.stack((rows * K)[:B * K]).astype(np.float32)
    eos = list(range(1, E + 1))
    st = ops.BeamState(B, K, E, 4, 0, "cuda")
    st.reset(3)
    ops.beam_step(_dev(x, dt) if not logprobs else torch.from_numpy(x).cuda(), st, eos, logprobs=logprobs)
    cs, ci = st.cand_scores.cpu().numpy(), st.cand_index.cpu().numpy()
    ost = BO.init_state(B, K, 3, 4, 0)
    lps = []
    for r in range(B * K):
        lp, amb = (x[r], np.zeros(V, bool)) if logprobs else BO.log_softmax(x[r])
        acc = (np.float32(ost.running[r // K, r % K]) + lp).astype(np.float32)
        scores, idx = VV.row_candidates(acc, keep)
        top = np.array([i for i in idx if i >= 0])
        if amb[VV.top_reference(acc, min(keep + 1, V))].any():
            continue
        assert np.array_equal(ci[r], np.where(idx >= 0, (r % K) * V + idx, -1)), (V, K, E, r, ci[r], idx)
        assert np.array_equal(cs[r].view(np.uint32), scores.view(np.uint32)), (V, K, E, r)
        assert top.shape[0] == min(keep, V)
        lps.append(lp)
    if len(lps) < B * K:
        return 0
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(BO, "log_softmax", lambda v: (np.asarray(v, np.float32), np.zeros(len(v), bool)))
        tok, par, fl = BO.step(ost, np.stack(lps), eos)
    assert not fl.any()
    assert np.array_equal(st.tokens.view(-1).cpu().numpy(), tok) and np.array_equal(st.parents.cpu().numpy(), par)
    for name, want in (("running", ost.running), ("finished", ost.fin), ("running_hist", ost.run_hist),
                       ("finished_hist", ost.fin_hist)):
        got = getattr(st, name).cpu().numpy()
        assert np.array_equal(got.view(np.uint32) if got.dtype == np.float32 else got,
                              want.view(np.uint32) if want.dtype == np.float32 else want), name
    assert np.array_equal(st.finished_flags.cpu().numpy() != 0, ost.fin_flag)
    return B * K


@pytest.mark.parametrize("V", [20, 33, 513, 32767])
@pytest.mark.parametrize("dt", VV.DTYPES)
def test_beam_rows_on_the_probes(dt, V):
    checked = 0
    for K, E in ((2, 0), (4, 3), (8, 4)):   # beams_to_keep 4, 16, 40: fillers at V = 20 and 33
        keep = VV.beams_to_keep(K, E)
        rows = _beam_rows(V, min(keep, V), dt)
        for logprobs in ((False, True) if dt == "fp32" else (False,)):
            checked += _check_beam(V, K, E, rows, dt, logprobs)
    assert checked > 0


@pytest.mark.parametrize("V", [20, 97, 1000])
def test_beam_logprobs_with_fewer_finite_values_than_kept(V):
    """n-gram blocking (N = 1) over a history that covers all but a few ids: the log-softmax rows have fewer finite
    values than beams_to_keep, so -inf candidates (ranked before the fillers) enter the step."""
    from perceiver_io_b200 import ops

    rng = np.random.default_rng(V)
    K, E = 4, 2
    keep = VV.beams_to_keep(K, E)
    x = (rng.standard_normal((2 * K, V)) * 3).astype(np.float32)
    hist = np.stack([rng.permutation(V) for r in range(2 * K)])
    lens = torch.tensor([V - 1 - r % 5 for r in range(2 * K)], dtype=torch.int32, device="cuda")
    lp = ops.process_logits(torch.from_numpy(x).cuda(), torch.from_numpy(hist).cuda(), lens, log_softmax=True,
                            no_repeat_ngram_size=1)
    lpc = lp.cpu().numpy()
    for r in range(2 * K):
        assert np.isfinite(lpc[r]).sum() == 1 + r % 5 < keep
    assert _check_beam(V, K, E, list(lpc), "fp32", True) == 2 * K


# ---- contrastive candidates ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [20, 33, 513, 32768])
@pytest.mark.parametrize("dt", VV.DTYPES)
def test_contrastive_candidates_on_the_probes(dt, V):
    from perceiver_io_b200 import ops

    for K in (4, 16):
        rows = _radix_at(V, K, dt) + [p.x for p in VV.tie_probes(V, K, dt, V)]
        rows += [p.x for p in VV.zero_probes(V, K, dt, V + 3)] if K < V else []
        rows += [p.x for p in VV.inf_probes(V, K, dt, V + 4) if p.claim["finite"] >= 1]
        B = len(rows)
        x = np.zeros((B * K, V), np.float32)
        x[::K] = np.stack(rows)
        st = ops.ContrastiveState(B, K, 8, 4, 4, 0, torch.bfloat16, "cuda")
        toks = ops.contrastive_candidates(_dev(x, dt), st)
        cand, probs = st.cand.cpu().numpy(), st.probs.cpu().numpy()
        for b in range(B):
            idx, p, _ = CO.candidates(rows[b], K)
            assert cand[b].tolist() == idx.tolist(), (dt, V, K, b, cand[b], idx)
            assert toks.view(B, K)[b].tolist() == idx.tolist()
            ulp = np.spacing(np.abs(p))
            assert np.all(np.abs(probs[b] - p) <= 4 * ulp), (dt, V, K, b, probs[b], p)


# ---- logits processors --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", VV.PROCESS_VOCABS)
@pytest.mark.parametrize("dt", VV.DTYPES)
def test_process_logits_on_the_probes(dt, V):
    from perceiver_io_b200 import ops

    rng = np.random.default_rng(V)
    for name, hists, kw in VV.processor_cases(V, V):
        R = len(hists)
        x = torch.from_numpy(rng.standard_normal((R, V)) * 3).to(TORCH[dt]).float().numpy()
        cap = max(len(h) for h in hists) + 3
        pre = np.zeros((R, cap), np.int64)
        for r, h in enumerate(hists):
            pre[r, :len(h)] = h
        lens = torch.tensor([len(h) for h in hists], dtype=torch.int32, device="cuda")
        for log_softmax in (False, True):
            got = ops.process_logits(_dev(x, dt), torch.from_numpy(pre).cuda(), lens, log_softmax=log_softmax,
                                     **kw).cpu().numpy()
            for r, h in enumerate(hists):
                base, amb = BO.log_softmax(x[r]) if log_softmax else (x[r], np.zeros(V, bool))
                want = PO.process(base, h, **kw)
                # bit for bit, but where the fp64 log-softmax lies within its reach of an fp32 rounding boundary: there
                # within 1 ulp of the log-softmax, times the penalty's one rounding
                ok = ~amb | np.isinf(want)
                np.testing.assert_array_equal(got[r][ok].view(np.uint32), want[ok].view(np.uint32),
                                              err_msg=f"{dt} V={V} {name} row {r} log_softmax={log_softmax}")
                np.testing.assert_array_less(np.abs(got[r][~ok] - want[~ok]), 2.5 * np.spacing(np.abs(want[~ok])))


# ---- the decoder --------------------------------------------------------------------------------------------------------
def test_sampled_generate_past_a_vocabulary_banned_by_ngram_blocking():
    """no_repeat_ngram_size=1 bans every id of the history; past the draw that uses the last free id every processed
    row is all -inf, which the sampler takes as greedy: token 0 with log-probability 0.  Each draw equals the step loop
    with the oracle processors and ops.sample_tokens, and every all -inf row of the loop is the oracle's token 0."""
    import perceiver_io_b200 as PK
    from perceiver_io_b200 import ops
    from test_gpu_graph_decode import _model
    from test_gpu_process import N0, PREFIX, _ids

    _, model = _model(False)
    B, n, V = 2, 40, 97
    ids, pad = _ids(B)
    kw = dict(no_repeat_ngram_size=1)
    samp = (0.8, 0, 1.0)
    dec = PK.GraphedDecoder(model, batch=B, max_new_tokens=n + 1, kv_cache="bf16")
    logits = dec.prefill(ids, PREFIX, pad)
    dec.set_seed([3, 4])
    dec.set_sampling(*samp, **kw)
    first = dec.draw(logits)
    got = torch.cat([first, dec.generate(first, n)], 1).cpu().numpy()
    assert ((got >= 0) & (got < V)).all(), got

    ref = PK.GraphedDecoder(model, batch=B, max_new_tokens=n + 1, kv_cache="bf16")
    logits = ref.prefill(ids, PREFIX, pad)
    seeds = torch.tensor([3, 4], device="cuda")
    hist = ids.tolist()
    want, banned = [], 0
    for t in range(n + 1):
        x = logits.float().cpu().numpy()
        rows = np.stack([PO.process(x[b], hist[b], **kw) for b in range(B)])
        pos = torch.full((B,), N0 + t, dtype=torch.int32, device="cuda")
        tok = ops.sample_tokens(torch.from_numpy(rows).cuda(), seeds, pos, *samp).tolist()
        for b in range(B):
            if np.isneginf(rows[b]).all():
                banned += 1
                assert tok[b] == S.sample_row(rows[b], *samp, 3 + b, b, N0 + t).token == 0
            hist[b].append(tok[b])
        want.append(tok)
        if t < n:
            logits = ref.step(torch.tensor(tok, device="cuda")[:, None])
    assert banned > 0
    np.testing.assert_array_equal(got, np.array(want).T)
