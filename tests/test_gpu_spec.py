"""-m gpu: speculative sampling (pcv_spec_verify) and GraphedDecoder.verify / speculative_generate.

Kernel: the exported accept and residual bits equal the numpy streams bit for bit; tokens and counts of bf16 / fp16 /
fp32 rows at V from 1 to 32768 and G in {1, 4, 63} equal the oracle's (oracle/spec_oracle.py) outside flagged
verdicts, with drafts drawn from Q by ops.sample_tokens and some adversarial drafts Q gives no mass; exact probes;
2^20 rounds against p and Σ min(p, q); launches are deterministic, independent of B and of graph capture.  Decoder:
generate(logits=True), a verify replay against eager extend + ops.spec_verify, speculative_generate against a loop
of the public methods, the oracle on a real two-model loop's own logits, and the per-round synchronisation."""
import warnings

import numpy as np
import pytest
import torch

from oracle import sample_oracle as S
from oracle import spec_oracle as SP

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}
TRIPLES = [((0.0, 0, 1.0), (0.0, 0, 1.0)), ((0.0, 0, 1.0), (1.0, 0, 1.0)), ((1.0, 0, 1.0), (0.0, 0, 1.0)),
           ((1.0, 10, 1.0), (1.0, 20, 1.0)), ((1.0, 0, 0.9), (1.0, 0, 0.95)), ((0.7, 0, 1.0), (1.3, 0, 1.0))]


def _counters(B, G1, gen):
    seeds = torch.randint(-2 ** 63, 2 ** 63 - 1, (B,), generator=gen, dtype=torch.int64)
    pos = torch.randint(0, 2 ** 31 - 100, (B, 1), generator=gen, dtype=torch.int64).to(torch.int32)
    return seeds, pos + torch.arange(G1, dtype=torch.int32)


def test_stream_export_is_the_numpy_hash():
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(1)
    seeds, pos = _counters(37, 5, gen)
    for stream in ("accept", "residual"):
        got = ops.spec_uniforms(seeds.cuda(), pos.cuda(), stream).cpu().numpy().view(np.uint64)
        want = SP.stream_bits(seeds.numpy()[:, None], np.arange(37)[:, None], pos.numpy(), stream)
        assert np.array_equal(got, want), stream
        got1 = ops.spec_uniforms(seeds.cuda(), pos[:, 0].contiguous().cuda(), stream).cpu().numpy().view(np.uint64)
        assert np.array_equal(got1, want[:, 0])


FLAGGED = {"rows": 0, "flagged": 0}


def _case(B, G, V, dt, tp, tq, gen):
    """Target logits, draft logits near them, drafts drawn from Q by ops.sample_tokens (every third row's last draft
    replaced by a token Q gives no mass where one exists)."""
    from perceiver_io_b200 import ops

    scale = torch.tensor([0.5, 2.0, 4.0])[torch.arange(B) % 3][:, None, None]
    tgt = (torch.randn(B, G + 1, V, generator=gen) * scale).to(DTYPES[dt])
    dft = (tgt[:, :G].float() + torch.randn(B, G, V, generator=gen) * 0.7).to(DTYPES[dt])
    seeds, pos = _counters(B, G + 1, gen)
    drafts = ops.sample_tokens(dft.cuda(), seeds.cuda(), pos[:, 1:].contiguous().cuda(), *tq).cpu()
    t0 = torch.randint(0, V, (B, 1), generator=gen)
    toks = torch.cat([t0, drafts], dim=1)
    for b in range(0, B, 3):
        Q = SP.masses(dft[b, G - 1].float().numpy(), *tq)
        zero = [y for y in range(V) if Q.w[y] == 0]
        if zero:
            toks[b, G] = zero[b % len(zero)]
    return tgt, dft, toks, seeds, pos


@pytest.mark.parametrize("V", [1, 2, 389, 32000, 32768])
@pytest.mark.parametrize("dt", list(DTYPES))
def test_kernel_against_the_oracle(dt, V):
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(V * 3 + len(dt))
    for G in (1, 4, 63):
        B = 4 if (V > 1000 or G == 63) else 12
        if V > 1000 and G == 63:
            B = 1
        for tp, tq in TRIPLES:
            tgt, dft, toks, seeds, pos = _case(B, G, V, dt, tp, tq, gen)
            out, acc = ops.spec_verify(tgt.cuda(), dft.cuda(), toks.cuda(), seeds.cuda(), pos.cuda(), tp, tq)
            out, acc = out.cpu(), acc.cpu()
            for b in range(B):
                v = SP.verify_row(tgt[b].float().numpy(), dft[b].float().numpy(), toks[b].tolist(), tp, tq,
                                  int(seeds[b]), b, pos[b].tolist())
                FLAGGED["rows"] += 1
                if v.ambiguous:
                    FLAGGED["flagged"] += 1
                    continue
                assert int(acc[b]) == v.n and out[b].tolist() == v.tokens, (dt, V, G, tp, tq, b, v)
    print(f"[spec] oracle-flagged verdicts so far: {FLAGGED['flagged']} of {FLAGGED['rows']}")
    assert FLAGGED["flagged"] <= 0.01 * FLAGGED["rows"] + 2


def test_exact_probes():
    from perceiver_io_b200 import ops

    dev = "cuda"
    gen = torch.Generator().manual_seed(5)
    B, G, V = 16, 4, 389
    seeds, pos = (t.cuda() for t in _counters(B, G + 1, gen))
    tgt = torch.randn(B, G + 1, V, generator=gen).to(torch.bfloat16).cuda()
    # p = q (same logits, same values): every draft drawn from Q is accepted
    for vals in ((1.0, 0, 1.0), (0.8, 10, 0.9)):
        drafts = ops.sample_tokens(tgt[:, :G], seeds, pos[:, 1:].contiguous(), *vals)
        toks = torch.cat([torch.zeros(B, 1, dtype=torch.long, device=dev), drafts], dim=1)
        out, acc = ops.spec_verify(tgt, tgt[:, :G], toks, seeds, pos, vals, vals)
        assert (acc == G).all() and torch.equal(out[:, :G], drafts)
    # both greedy with different argmaxes: n = 0 and the correction is the target's argmax
    dft = tgt[:, :G].clone()
    dft[..., 0] = 100.0
    tgt2 = tgt.clone()
    tgt2[..., 1] = 100.0
    toks = torch.zeros(B, G + 1, dtype=torch.long, device=dev)
    out, acc = ops.spec_verify(tgt2, dft, toks, seeds, pos, (0.0, 0, 1.0), (0.0, 0, 1.0))
    assert (acc == 0).all() and (out[:, 0] == 1).all() and (out[:, 1:] == -1).all()
    # a greedy draft on a token P gives no mass is rejected
    tgt3 = tgt.clone()
    tgt3[..., 0] = -1000.0
    out, acc = ops.spec_verify(tgt3, dft, toks, seeds, pos, (1.0, 10, 1.0), (0.0, 0, 1.0))
    assert (acc == 0).all() and (out[:, 0] != 0).all()


def _distribution(tp, tq, label):
    from scipy.stats import chi2

    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(17)
    V = 64
    lp = torch.randn(V, generator=gen) * 1.5
    lq = lp + torch.randn(V, generator=gen)
    P, Q = SP.masses(lp.numpy(), *tp), SP.masses(lq.numpy(), *tq)
    p = np.array(P.w, dtype=np.float64) / P.Z
    q = np.array(Q.w, dtype=np.float64) / Q.Z
    B, launches = 4096, 256                       # 2^20 rounds at distinct (b, pos)
    tgt = lp.repeat(B, 2, 1).cuda()
    dft = lq.repeat(B, 1, 1).cuda()
    seeds = torch.full((B,), 4242, dtype=torch.long, device="cuda")
    counts = torch.zeros(V, dtype=torch.long, device="cuda")
    accepted = torch.zeros((), dtype=torch.long, device="cuda")
    for i in range(launches):
        pos = (i * 2 + torch.arange(2, dtype=torch.int32, device="cuda")).repeat(B, 1)
        drafts = ops.sample_tokens(dft, seeds, pos[:, 1:].contiguous(), *tq)
        toks = torch.cat([torch.zeros(B, 1, dtype=torch.long, device="cuda"), drafts], dim=1)
        out, acc = ops.spec_verify(tgt, dft, toks, seeds, pos, tp, tq)
        counts += torch.bincount(out[:, 0], minlength=V)
        accepted += acc.sum()
    counts = counts.cpu().numpy()
    n = B * launches
    assert counts[p == 0].sum() == 0
    exp, obs = p[p > 0] * n, counts[p > 0]
    big = exp >= 5
    e, o = np.append(exp[big], exp[~big].sum()), np.append(obs[big], obs[~big].sum())
    if e[-1] == 0:
        e, o = e[:-1], o[:-1]
    stat = ((o - e) ** 2 / e).sum()
    pval = chi2.sf(stat, len(e) - 1)
    rate = np.minimum(p, q).sum()
    sigma = np.sqrt(n * rate * (1 - rate))
    got = int(accepted)
    print(f"[spec] {label}: chi-square {stat:.1f} on {len(e) - 1} dof, p = {pval:.3f}; accepted {got} of {n}, "
          f"Σ min(p, q) n = {rate * n:.0f} ({(got - rate * n) / max(sigma, 1e-9):+.2f} σ)")
    assert pval > 1e-4
    assert abs(got - rate * n) <= 5 * sigma + 1


def test_distribution_matches_p_and_acceptance_sum_min():
    _distribution((1.0, 0, 1.0), (1.0, 0, 1.0), "plain")


def test_distribution_with_target_top_p():
    _distribution((1.0, 0, 0.8), (1.0, 0, 1.0), "target top-p 0.8")


def test_launches_are_deterministic_batch_independent_and_capturable():
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(2)
    B, G, V = 8, 4, 1000
    tp, tq = (0.9, 20, 0.9), (1.0, 0, 1.0)
    tgt, dft, toks, seeds, pos = (t.cuda() for t in _case(B, G, V, "bf16", tp, tq, gen))
    a = ops.spec_verify(tgt, dft, toks, seeds, pos, tp, tq)
    b = ops.spec_verify(tgt, dft, toks, seeds, pos, tp, tq)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    sub =ops.spec_verify(tgt[:1], dft[:1], toks[:1], seeds[:1], pos[:1], tp, tq)
    assert torch.equal(sub[0][0], a[0][0]) and int(sub[1][0]) == int(a[1][0])
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.spec_verify(tgt, dft, toks, seeds, pos, tp, tq)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(g):
        out = ops.spec_verify(tgt, dft, toks, seeds, pos, tp, tq)
    g.replay()
    assert torch.equal(out[0], a[0]) and torch.equal(out[1], a[1])


# ---- the decoder ------------------------------------------------------------------------------------------------------
ROWS, N0, PREFIX, G = 3, 120, 90, 4
TARGET_VALS, DRAFT_VALS = (0.9, 20, 0.9), (1.0, 10, 1.0)


def _pair(kind, T=48):
    import copy

    import perceiver_io_b200 as P
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    draft_model = copy.deepcopy(model)
    with torch.no_grad():
        for prm in draft_model.parameters():
            prm.add_(0.05 * torch.randn_like(prm))
    torch.manual_seed(31)
    tokens0 = torch.randint(0, 97, (ROWS, N0)).cuda()
    pad0 = torch.zeros(ROWS, N0, dtype=torch.bool, device="cuda")
    pad0[1, :7] = True
    decs = []
    for m, vals in ((model, TARGET_VALS), (draft_model, DRAFT_VALS)):
        dec = P.GraphedDecoder(m, batch=ROWS, max_new_tokens=T, kv_cache=kind)
        logits = dec.prefill(tokens0, PREFIX, pad0)
        dec.set_seed([11, 22, 33])
        dec.set_sampling(*vals)
        decs.append((dec, logits))
    return decs


@pytest.mark.parametrize("kind", ["bf16", "fp8"])
def test_generate_with_logits_and_verify_equal_their_eager_forms(kind):
    from perceiver_io_b200 import ops
    from perceiver_io_b200.generation import sample_positions

    (tgt, lt), (dft, _) = _pair(kind)
    first = tgt.draw(lt)
    torch.cuda.set_sync_debug_mode("error")
    try:
        toks, lg = dft.generate(first, G + 1, logits=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    toks, lg = toks.clone(), lg.clone()
    dft.rewind(G + 1)
    assert torch.equal(dft.generate(first, G + 1), toks)
    pos = sample_positions(dft._bounds, dft._steps, 1) - (G + 1) + torch.arange(G + 1, device="cuda", dtype=torch.int32)
    assert torch.equal(ops.sample_tokens(lg, dft._seeds, pos, *DRAFT_VALS), toks)
    fed = torch.cat([first, toks[:, :G]], dim=1)
    snapshot = tgt._bounds.clone()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out, acc = tgt.verify(fed, lg[:, :G], draft_sampling=DRAFT_VALS)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    out, acc = out.clone(), acc.clone()
    tgt.rewind(G + 1)
    assert torch.equal(tgt._bounds, snapshot)
    pos = sample_positions(tgt._bounds, tgt._steps, G + 1)
    logits = tgt.extend(fed).clone()
    want = ops.spec_verify(logits, lg[:, :G].contiguous(), fed, tgt._seeds, pos, TARGET_VALS, DRAFT_VALS)
    assert torch.equal(out, want[0]) and torch.equal(acc, want[1])


@pytest.mark.parametrize("kind", ["bf16", "fp8"])
def test_speculative_generate_is_the_loop_of_public_methods(kind):
    from perceiver_io_b200.generation import speculative_budget, speculative_generate

    n = 14
    T = speculative_budget(n, G, ROWS)
    (tgt, lt), (dft, _) = _pair(kind, T)
    first = tgt.draw(lt)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            got, stats = speculative_generate(tgt, dft, first, n, draft_tokens=G)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in caught if "synchroniz" in str(w.message).lower()]
    assert len(syncs) == stats["rounds"], [str(w.message) for w in syncs]
    # the hand-written loop
    (tgt, lt), (dft, _) = _pair(kind, T)
    t0 = tgt.draw(lt)
    rows = [[] for _ in range(ROWS)]
    while min(len(r) for r in rows) < n:
        drafts, q = dft.generate(t0, G + 1, logits=True)
        out, acc = tgt.verify(torch.cat([t0, drafts[:, :G]], dim=1), q[:, :G], draft_sampling=DRAFT_VALS)
        acc, out = acc.tolist(), out.cpu()
        back, nxt = [], []
        for b in range(ROWS):
            if len(rows[b]) >= n:
                back.append(G + 1)
                nxt.append(int(t0[b]))
                continue
            rows[b] += out[b, :acc[b] + 1].tolist()
            back.append(G - acc[b])
            nxt.append(int(out[b, acc[b]]))
        tgt.rewind(back)
        dft.rewind(back)
        t0 = torch.tensor(nxt, device="cuda")[:, None]
    assert got.tolist() == [r[:n] for r in rows]
    print(f"[spec] {kind}: {stats['rounds']} rounds, accepted {stats['accepted']} of {stats['proposed']}")


def test_teacher_forced_verdicts_are_the_oracles():
    """A real two-model loop: the oracle applied to the draft logits and the verify graph's own target logits gives the
    loop's tokens and counts."""
    (tgt, lt), (dft, _) = _pair("bf16")
    t0 = tgt.draw(lt)
    checked = flagged = 0
    for _ in range(5):
        drafts, q = dft.generate(t0, G + 1, logits=True)
        fed = torch.cat([t0, drafts[:, :G]], dim=1)
        pos0 = tgt._bounds[:, 0, 2].clone()
        out, acc = tgt.verify(fed, q[:, :G], draft_sampling=DRAFT_VALS)
        p_logits = tgt._verify_logits.float().cpu().numpy()
        out, acc, fedc, qc = out.cpu(), acc.cpu(), fed.cpu(), q[:, :G].float().cpu().numpy()
        for b in range(ROWS):
            pos = [int(pos0[b]) + 1 + i for i in range(G + 1)]
            v = SP.verify_row(p_logits[b], qc[b], fedc[b].tolist(), TARGET_VALS, DRAFT_VALS, (11, 22, 33)[b], b, pos)
            if v.ambiguous:
                flagged += 1
                continue
            assert out[b].tolist() == v.tokens and int(acc[b]) == v.n, (b, v)
            checked += 1
        back = [G - int(a) for a in acc]
        tgt.rewind(back)
        dft.rewind(back)
        t0 = out.gather(1, acc.long()[:, None]).cuda()
    print(f"[spec] teacher-forced verdicts: {checked} equal to the oracle's, {flagged} flagged")
    assert checked >= 12


def test_a_dropped_decoder_frees_its_graphs_without_the_cycle_collector():
    """A decoder that recorded its sampling and verify graphs is freed when its last reference goes, not at some later
    cycle collection, which could destroy its graphs while another stream is capturing and invalidate that capture."""
    import gc
    import weakref

    gc.collect()
    gc.disable()
    try:
        (tgt, lt), (dft, _) = _pair("bf16")
        first = tgt.draw(lt)
        drafts, q = dft.generate(first, G + 1, logits=True)
        tgt.verify(torch.cat([first, drafts[:, :G]], dim=1), q[:, :G], draft_sampling=DRAFT_VALS)
        tgt.step(first)
        assert tgt.captures == 2 and dft.captures == 1
        refs = [weakref.ref(tgt), weakref.ref(dft)]
        del tgt, dft, lt, first, drafts, q
        assert all(r() is None for r in refs)
    finally:
        gc.enable()
