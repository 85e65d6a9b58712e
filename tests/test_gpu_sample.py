"""-m gpu: the device token sampler (pcv_sample) and GraphedDecoder's sampling graphs.

Kernel: the exported random bits equal the numpy hash bit for bit; every token of bf16 / fp16 / fp32 rows at V from 1 to
32768 under every filter combination equals the oracle's (oracle/sample_oracle.py) unless the oracle flags the draw
ambiguous, where it must be a kept neighbour; exact probes (every mass exact) match bit for bit; 2^20 draws from fixed
logits pass a chi-square test against the exact filtered distribution; launches are deterministic, independent of R and
of graph capture.  Decoder: generate equals step + ops.sample_tokens bit for bit (left padding, a beam reorder, per-row
rewinds, sync-debug "error"), a rewound row regenerates its tokens, sample(drafts) equals ops.sample_tokens on its own
logits, and teacher-forced draws agree with the oracle on the fp64 one-token loop outside the logits' error gate."""
import numpy as np
import pytest
import torch

from oracle import sample_oracle as S

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def _configs(V):
    return [(1.0, 0, 1.0), (0.7, 0, 1.0), (1.3, 10, 1.0), (1.0, 1, 1.0), (1.0, V - 1, 1.0), (1.0, V, 1.0),
            (1.0, V + 5, 1.0), (1.0, 0, 0.95), (1.0, 0, 0.5), (1.0, 0, 1e-3), (0.7, 10, 0.95), (1.3, 50, 0.5),
            (0.0, 0, 1.0)]


def _logits(R, V, dtype, gen):
    """Rows of varied sharpness; every fourth row integer-valued (ties at the cuts)."""
    scale = torch.tensor([0.05, 1.0, 4.0, 12.0])[torch.arange(R) % 4][:, None]
    x = torch.randn(R, V, generator=gen) * scale
    x[3::4] = torch.round(x[3::4] / 4)
    return x.to(dtype)


def _counters(B, lead, gen):
    seeds = torch.randint(-2 ** 63, 2 ** 63 - 1, (B,), generator=gen, dtype=torch.int64)
    pos = torch.randint(-2 ** 31, 2 ** 31 - 1, lead, generator=gen, dtype=torch.int64).to(torch.int32)
    return seeds, pos


def test_uniform_export_is_the_numpy_hash():
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(1)
    seeds, pos = _counters(37, (37, 5), gen)
    pos[0, :3] = torch.tensor([0, 1, 2 ** 31 - 1], dtype=torch.int32)
    got = ops.sample_uniforms(seeds.cuda(), pos.cuda()).cpu().numpy().view(np.uint64)
    want = S.uniform_bits(seeds.numpy()[:, None], np.arange(37)[:, None], pos.numpy())
    assert np.array_equal(got, want)
    got1 = ops.sample_uniforms(seeds.cuda(), pos[:, 0].contiguous().cuda()).cpu().numpy().view(np.uint64)
    assert np.array_equal(got1, want[:, 0])


def _neighbours(kept, tok):
    idx = np.nonzero(kept)[0]
    j = np.searchsorted(idx, tok)
    return set(idx[max(0, j - 1):j + 2].tolist())


AMBIGUOUS = {"draws": 0, "ambiguous": 0}


@pytest.mark.parametrize("V", [1, 2, 262, 389, 1000, 32000, 32768])
@pytest.mark.parametrize("dt", list(DTYPES))
def test_kernel_against_the_oracle(dt, V):
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(V * 7 + len(dt))
    R = 16 if V > 1000 else (1024 if (V, dt) == (262, "bf16") else 128)
    k = 4 if R % 4 == 0 else 1
    logits = _logits(R, V, DTYPES[dt], gen)
    B = R // k
    seeds, pos = _counters(B, (B, k), gen)
    x32 = logits.float().numpy()
    for T, top_k, top_p in _configs(V):
        toks, lps = ops.sample_tokens(logits.cuda().view(B, k, V), seeds.cuda(), pos.cuda(), T, top_k, top_p,
                                      logprobs=True)
        toks, lps = toks.view(-1).cpu().numpy(), lps.view(-1).cpu().numpy()
        for r in range(R):
            b = r // k
            d = S.sample_row(x32[r], T, top_k, top_p, int(seeds[b]), b, int(pos.view(-1)[r]))
            AMBIGUOUS["draws"] += 1
            if d.ambiguous:
                AMBIGUOUS["ambiguous"] += 1
                kept = S.filter_row(x32[r], T, top_k, top_p).kept
                assert toks[r] in _neighbours(kept, d.token), (dt, V, T, top_k, top_p, r, d)
                continue
            assert toks[r] == d.token, (dt, V, T, top_k, top_p, r, d, toks[r])
            assert abs(lps[r] - d.logprob) <= 1e-6 * max(1.0, abs(d.logprob)), (dt, V, T, top_k, top_p, r)
    frac = AMBIGUOUS["ambiguous"] / AMBIGUOUS["draws"]
    print(f"[sample] oracle-ambiguous draws so far: {AMBIGUOUS['ambiguous']} of {AMBIGUOUS['draws']} ({frac:.2e})")
    assert frac <= 1e-3


def test_exact_probes_and_greedy_ties():
    """Equal logits among the kept tokens and the rest 100 below: every mass is exactly 2^40 or 0, so each draw is the
    oracle's bit for bit, with no ambiguity allowance."""
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(4)
    for V, kept in ((389, [0, 7, 8, 200, 388]), (32000, list(range(3, 32000, 997))), (2, [1])):
        base = torch.full((V,), -90.0)
        base[kept] = 10.0
        R = 64
        logits = base.repeat(R, 1)
        seeds, pos = _counters(R, (R,), gen)
        for T, top_k, top_p in ((1.0, 0, 1.0), (0.5, len(kept), 1.0), (1.0, 0, 0.999), (2.0, 3, 1.0)):
            toks = ops.sample_tokens(logits.cuda(), seeds.cuda(), pos.cuda(), T, top_k, top_p).cpu()
            for r in range(R):
                d = S.sample_row(logits[r].numpy(), T, top_k, top_p, int(seeds[r]), r, int(pos[r]))
                assert not d.ambiguous and S.filter_row(logits[r].numpy(), T, top_k, top_p).slack == 0
                assert int(toks[r]) == d.token and d.token in kept, (V, T, top_k, top_p, r)
        greedy = ops.sample_tokens(logits.cuda(), seeds.cuda(), pos.cuda(), 0.0).cpu()
        assert (greedy == kept[0]).all()
    z = torch.tensor([[-1.0, -0.0, 0.0, 0.0], [3.0, 1.0, 3.0, 3.0]])
    got = ops.sample_tokens(z.cuda(), torch.zeros(2, dtype=torch.long, device="cuda"),
                            torch.zeros(2, dtype=torch.int32, device="cuda"), 0.0, logprobs=True)
    assert got[0].tolist() == [1, 0] and got[1].tolist() == [0.0, 0.0]


def test_distribution_matches_the_filtered_probabilities():
    from scipy.stats import chi2

    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(9)
    V, T, top_k, top_p = 389, 0.8, 60, 0.9
    row = torch.randn(V, generator=gen) * 2
    p = S.probs(row.numpy(), T, top_k, top_p)
    R, launches = 4096, 256                      # 2^20 draws at positions 0 .. 2^20 - 1, one seed
    logits = row.repeat(R, 1).cuda()
    seeds = torch.full((1,), 20260101, dtype=torch.long, device="cuda")
    counts = torch.zeros(V, dtype=torch.long, device="cuda")
    for i in range(launches):
        pos = torch.arange(i * R, (i + 1) * R, dtype=torch.int32, device="cuda")[None]
        toks = ops.sample_tokens(logits[None], seeds, pos, T, top_k, top_p).view(-1)
        counts += torch.bincount(toks, minlength=V)
    counts = counts.cpu().numpy()
    n = R * launches
    assert counts[p == 0].sum() == 0
    exp = p[p > 0] * n
    obs = counts[p > 0]
    big = exp >= 5
    e, o = np.append(exp[big], exp[~big].sum()), np.append(obs[big], obs[~big].sum())
    if e[-1] == 0:
        e, o = e[:-1], o[:-1]
    stat = ((o - e) ** 2 / e).sum()
    pval = chi2.sf(stat, len(e) - 1)
    print(f"[sample] chi-square {stat:.1f} on {len(e) - 1} dof over {n} draws: p = {pval:.3f}")
    assert pval > 1e-4


def test_launches_are_deterministic_and_row_independent():
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(2)
    B, k, V = 8, 4, 1000
    logits = _logits(B * k, V, torch.bfloat16, gen).view(B, k, V).cuda()
    seeds, pos = (t.cuda() for t in _counters(B, (B, k), gen))
    for T, top_k, top_p in ((1.0, 0, 1.0), (0.9, 20, 0.8), (1.0, 0, 0.3)):
        a = ops.sample_tokens(logits, seeds, pos, T, top_k, top_p)
        assert torch.equal(a, ops.sample_tokens(logits, seeds, pos, T, top_k, top_p))
        # R rows of batch row 0 in one launch equal R launches of one row each
        rows = ops.sample_tokens(logits.view(1, B * k, V), seeds[:1], pos.view(1, B * k), T, top_k, top_p)
        for r in range(B * k):
            one = ops.sample_tokens(logits.view(B * k, V)[r:r + 1, None], seeds[:1], pos.view(1, B * k)[:, r:r + 1],
                                    T, top_k, top_p)
            assert int(one) == int(rows[0, r]), r
        assert torch.equal(rows.view(B, k)[0], a[0])
        strided = torch.empty(B, k, V + 24, dtype=logits.dtype, device="cuda")[..., :V]
        strided.copy_(logits)
        assert torch.equal(a, ops.sample_tokens(strided, seeds, pos, T, top_k, top_p))
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            ops.sample_tokens(logits, seeds, pos, T, top_k, top_p)
        torch.cuda.current_stream().wait_stream(side)
        with torch.cuda.graph(g):
            out = ops.sample_tokens(logits, seeds, pos, T, top_k, top_p)
        g.replay()
        assert torch.equal(out, a)


# ---- the decoder ------------------------------------------------------------------------------------------------------
ROWS, N0, PREFIX = 3, 120, 90
SAMPLING = (0.9, 20, 0.9)


def _decoder(model, kind, tokens0, pad0, T=40, seeds=(11, 22, 33)):
    import perceiver_io_b200 as P

    dec = P.GraphedDecoder(model, batch=ROWS, max_new_tokens=T, kv_cache=kind)
    logits = dec.prefill(tokens0[:, :N0], PREFIX, pad0[:, :N0])
    dec.set_seed(list(seeds))
    dec.set_sampling(*SAMPLING)
    return dec, logits


@pytest.mark.parametrize("kind", ["bf16", "fp8"])
def test_generate_is_step_then_sample_tokens(kind):
    from perceiver_io_b200 import ops
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    torch.manual_seed(21)
    tokens0 = torch.randint(0, 97, (ROWS, N0 + 1)).cuda()
    pad0 = torch.zeros(ROWS, N0 + 1, dtype=torch.bool, device="cuda")
    pad0[1, :9] = True
    idx = torch.tensor([2, 0, 0], device="cuda")
    # the graphed arm: draw, generate 12, reorder, generate 12
    dec, logits0 = _decoder(model, kind, tokens0, pad0)
    first = dec.draw(logits0)
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = dec.generate(first, 12)
        dec.reorder(idx)
        b = dec.generate(a[:, -1:][idx], 12)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert dec.captures == 1
    # the eager arm: step + ops.sample_tokens at the same positions
    ref, logits = _decoder(model, kind, tokens0, pad0)
    seeds = torch.tensor([11, 22, 33], device="cuda")
    pos = lambda j: torch.full((ROWS, 1), N0 + j, dtype=torch.int32, device="cuda")
    tok = ops.sample_tokens(logits[:, None], seeds, pos(0), *SAMPLING)
    assert torch.equal(tok, first)
    got = []
    for j in range(24):
        if j == 12:
            ref.reorder(idx)
            seeds, tok = seeds[idx], tok[idx]
        tok = ops.sample_tokens(ref.step(tok)[:, None], seeds, pos(j + 1), *SAMPLING)
        got.append(tok)
    got = torch.cat(got, dim=1)
    assert torch.equal(got[:, :12], a) and torch.equal(got[:, 12:], b)
    # per-row rewind and regenerate: row r drops counts[r] tokens and draws the same ones again
    counts = [5, 2, 7]
    fed = torch.cat([a[idx], b], dim=1)   # row r's fed tokens after the first: rows N0+1 .. N0+24 (the last is drawn)
    dec.rewind(counts)
    nxt = torch.stack([fed[r, 23 - counts[r]] for r in range(ROWS)])[:, None]
    again = dec.generate(nxt, 2)
    for r in range(ROWS):
        assert torch.equal(again[r], fed[r, 24 - counts[r]:26 - counts[r]]), r


@pytest.mark.parametrize("kind", ["bf16", "fp8"])
def test_sample_drafts_match_sample_tokens_on_their_logits(kind):
    from perceiver_io_b200 import ops
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    torch.manual_seed(22)
    tokens0 = torch.randint(0, 97, (ROWS, N0 + 40)).cuda()
    pad0 = torch.zeros(ROWS, N0 + 40, dtype=torch.bool, device="cuda")
    pad0[0, :4] = True
    dec, _ = _decoder(model, kind, tokens0, pad0)
    fed = 0
    for k in (5, 1, 16):
        drafts = tokens0[:, N0 + fed:N0 + fed + k]
        toks, logits = dec.sample(drafts)
        pos = (N0 + fed + 1 + torch.arange(k, dtype=torch.int32, device="cuda")).repeat(ROWS, 1)
        want = ops.sample_tokens(logits.clone(), torch.tensor([11, 22, 33], device="cuda"), pos, *SAMPLING)
        assert torch.equal(toks, want), k
        accept = drafts[:, 1:] == toks[:, :-1]        # speculative acceptance on the device
        assert accept.shape == (ROWS, k - 1)
        fed += k
    assert dec.captures == 3


def test_teacher_forced_draws_agree_with_the_oracle_on_the_fp64_loop(monkeypatch):
    """Feed the same tokens as the fp64 one-token loop and compare each replay's draw with the oracle's draw on the fp64
    logits: equal unless the oracle flags the draw as one that a perturbation of every logit by the replay's own
    measured error against fp64 (its largest, over the row) could change."""
    import copy

    import test_gpu_window as GW
    from test_gpu_fp8_kv_cache import _Fp64Attend, _owners
    from test_gpu_graph_decode import _model

    cfg, model = _model(False)
    model64 = copy.deepcopy(model).double()
    fp64 = _Fp64Attend(model64, _owners(model64))
    T = 24
    torch.manual_seed(23)
    tokens0 = torch.randint(0, GW.VOCAB, (ROWS, GW.N0 + T + 1)).cuda()
    pad0 = torch.zeros(ROWS, tokens0.shape[1], dtype=torch.bool, device="cuda")
    pad0[2, :6] = True
    monkeypatch.setattr(GW, "REORDER_AT", -1)
    truth = GW._eager_loop(model, model64, fp64, "fp64", tokens0, pad0, cfg, monkeypatch, T).cpu()
    agree = flagged = 0
    worst = 0.0
    for kind in ("bf16", "fp8"):
        for vals in (SAMPLING, (0.0, 0, 1.0), (1.0, 3, 1.0)):
            dec, _ = _decoder(model, kind, tokens0, pad0, T=T)
            dec.set_sampling(*vals)
            fed = 0
            for k in (1, 4, 1, 8, 2):
                toks, logits = dec.sample(tokens0[:, GW.N0 + fed:GW.N0 + fed + k])
                toks, logits = toks.cpu(), logits.double().cpu()
                for r in range(ROWS):
                    for i in range(k):
                        t = fed + 1 + i    # truth[:, t]: the logits after fed token t - 1, drawn at row N0 + t
                        err = (logits[r, i] - truth[r, t]).abs().max().item()
                        worst = max(worst, err)
                        d = S.sample_row(truth[r, t].float().numpy(), *vals, seed=(11, 22, 33)[r], b=r, pos=GW.N0 + t,
                                         logit_err=err * 1.01 + 1e-6)
                        if d.ambiguous:
                            flagged += 1
                            continue
                        assert int(toks[r, i]) == d.token, (kind, vals, r, t, d)
                        agree += 1
                fed += k
    print(f"[sample] teacher-forced draws: {agree} equal to the fp64 oracle's, {flagged} within the replays' logit "
          f"error (at most {worst:.2e})")
    assert agree >= 0.2 * (agree + flagged)
