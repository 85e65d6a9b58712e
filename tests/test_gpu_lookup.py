"""-m gpu: prompt-lookup drafts (pcv_prompt_lookup) and GraphedDecoder.prompt_lookup_generate.

Kernel: drafts and counts equal oracle/lookup_oracle.py's bit for bit on histories of length 1, 2, N, N + 1, around
the 256-thread stride and up to the arena's width, with left-pad starts (a match only in the padding does not count),
ids >= 2^31, EOS cuts, per-row limits, G in {1, 10, 63}, N in {1, 2, 16} and B up to 64; two launches and a launch
under graph capture give the same result.  Decoder: prompt_lookup_generate equals a loop of the public methods
(sample with oracle drafts on the host history, then a per-row rewind) token for token and round for round, on bf16
and FP8 arenas, greedy and top-k, B = 1 and B = 4 with left padding, with both windows sliding, an EOS mid-run and
processors on, with one device-to-host read per round (and one before the first); greedy agrees with plain greedy
generate up to the first near-tie; a run at exactly the stated budget completes."""
import warnings

import numpy as np
import pytest
import torch

from oracle import lookup_oracle as LO

pytestmark = pytest.mark.gpu


# ---- the kernel ---------------------------------------------------------------------------------------------------------
def _histories(B, cap, vocab, gen, big=False):
    ids = torch.randint(0, vocab, (B, cap), generator=gen)
    if big:
        ids = ids + (2 ** 31 - 2)   # ids from 2^31 - 2 up: the comparisons are 64-bit
    return ids


def _check(ids, lengths, G, N, starts=None, limits=None, eos=()):
    from perceiver_io_b200 import ops

    B = ids.shape[0]
    dev = lambda t: None if t is None else torch.as_tensor(t, dtype=torch.int32).cuda()
    drafts, counts = ops.prompt_lookup(ids.cuda(), dev(lengths), G, N, start=dev(starts), limit=dev(limits), eos=eos)
    want_d, want_c = LO.lookup_rows(ids.tolist(), lengths, G, N, starts, limits, eos)
    assert counts.cpu().tolist() == want_c, (G, N)
    assert drafts.cpu().tolist() == want_d, (G, N)
    return want_c


LENGTHS = [1, 2, 3, 16, 17, 255, 256, 257, 258, 511, 512, 513, 1000]


@pytest.mark.parametrize("G,N", [(1, 1), (10, 2), (63, 2), (10, 16), (63, 16), (4, 3)])
def test_kernel_equals_the_oracle(G, N):
    gen = torch.Generator().manual_seed(G * 100 + N)
    found = 0
    for vocab in (2, 3, 5, 40):
        for big in (False, True):
            cap = 1024
            ids = _histories(len(LENGTHS), cap, vocab, gen, big)
            lengths = [min(L, cap) for L in LENGTHS]
            found += sum(c > 0 for c in _check(ids, lengths, G, N))
            lengths = [N, N + 1] + lengths[2:]
            _check(ids, lengths, G, N)
            # left padding: a start, and a match that lies only in the padding
            starts = [int(s) for s in torch.randint(0, 40, (len(LENGTHS),), generator=gen)]
            _check(ids, [s + L for s, L in zip(starts, lengths)][:len(LENGTHS)], G, N, starts=starts)
            # EOS ids and per-row limits
            eos = [int(ids[0, 5]), int(ids[1, 7])]
            limits = [int(x) for x in torch.randint(-2, G + 3, (len(LENGTHS),), generator=gen)]
            _check(ids, lengths, G, N, limits=limits, eos=eos)
            _check(ids, lengths, G, N, starts=starts, limits=limits, eos=eos[:1])
    assert found > 10


def test_a_match_in_the_padding_does_not_count():
    ids = torch.tensor([[7, 8, 9, 1, 2, 3, 7, 8], [5, 6, 1, 2, 3, 4, 5, 5]])
    # row 0: (7, 8) occurs at 0 .. 1 only, inside 3 padding positions: no draft; with no padding: 9, 1, ...
    assert _check(ids, [8, 8], 4, 2, starts=[3, 0]) == [0, 4]
    assert _check(ids, [8, 8], 4, 2, starts=[0, 0]) == [4, 4]
    # the suffix (5,) matches at 0 (continuation 6, 1, 2, 3) unless padded, then at 6 (continuation 5)
    assert _check(ids, [8, 8], 4, 1, starts=[0, 1]) == [4, 1]


def test_batch_of_64_at_the_arena_width_and_every_edge():
    gen = torch.Generator().manual_seed(5)
    B, cap = 64, 6144 + 256
    ids = _histories(B, cap, 4, gen)
    lengths = [int(x) for x in torch.randint(1, cap + 1, (B,), generator=gen)]
    lengths[:6] = [1, 2, cap, cap - 1, 257, 256]
    starts = [int(x) for x in torch.randint(0, 100, (B,), generator=gen)]
    starts[:6] = [0, 0, 0, 50, 256, 255]
    for G, N in ((10, 2), (63, 16), (1, 1)):
        _check(ids, lengths, G, N, starts=starts, eos=[3])
        _check(ids, lengths, G, N)
    # the EOS cut: first (empty, no fallback) and mid-draft
    ids = torch.tensor([[1, 2, 9, 4, 1, 2, 1, 2], [1, 2, 3, 9, 5, 6, 1, 2]])
    assert _check(ids, [8, 8], 5, 2, eos=[9]) == [0, 1]
    assert _check(ids, [8, 8], 5, 2) == [5, 5]


def test_launches_are_deterministic_and_graph_capture_changes_nothing():
    from perceiver_io_b200 import ops

    gen = torch.Generator().manual_seed(9)
    ids = _histories(16, 6400, 3, gen).cuda()
    lengths = torch.randint(1, 6401, (16,), generator=gen).to(torch.int32).cuda()
    a = ops.prompt_lookup(ids, lengths, 10, 2, eos=[2])
    b = ops.prompt_lookup(ids, lengths, 10, 2, eos=[2])
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.prompt_lookup(ids, lengths, 10, 2, eos=[2])
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(g):
        out = ops.prompt_lookup(ids, lengths, 10, 2, eos=[2])
    g.replay()
    assert torch.equal(out[0], a[0]) and torch.equal(out[1], a[1])


def test_ops_refuse_before_any_launch():
    from perceiver_io_b200 import ops

    ids = torch.zeros(2, 8, dtype=torch.long, device="cuda")
    L = torch.ones(2, dtype=torch.int32, device="cuda")
    for kw, match in ((dict(num_output_tokens=0), "G=0"), (dict(num_output_tokens=64), "G=64"),
                      (dict(max_matching_ngram_size=0), "N=0"), (dict(max_matching_ngram_size=17), "N=17"),
                      (dict(eos=[1, 2, 3, 4, 5]), "at most 4")):
        with pytest.raises(ValueError, match=match):
            ops.prompt_lookup(ids, L, **kw)
    with pytest.raises(ValueError, match="lengths must be"):
        ops.prompt_lookup(ids, L.long())
    with pytest.raises(ValueError, match="ids must be"):
        ops.prompt_lookup(ids.int(), L)


# ---- the decoder --------------------------------------------------------------------------------------------------------
N0, PREFIX = 120, 90
MOTIF = [5, 17, 33, 2, 61, 8, 40]


def _decoder(kind, B, T, pad_rows=(), seed=11):
    import perceiver_io_b200 as P
    from test_gpu_graph_decode import _model

    _, model = _model(False)
    ids = torch.tensor((MOTIF * (N0 // len(MOTIF) + 1))[:N0]).repeat(B, 1).cuda()
    pad = torch.zeros(B, N0, dtype=torch.bool, device="cuda")
    for b in pad_rows:
        pad[b, :5 + 3 * b] = True
        ids[b, :5 + 3 * b] = 0
    dec = P.GraphedDecoder(model, batch=B, max_new_tokens=T, kv_cache=kind)
    logits = dec.prefill(ids, PREFIX, pad)
    dec.set_seed([seed + b for b in range(B)])
    return dec, logits, ids.cpu(), pad.cpu()


def _loop(dec, first, n, G, Nn, ids, pad, eos):
    """prompt_lookup_generate as a loop of public methods: oracle drafts on the host history, sample, per-row rewind."""
    B = dec.batch
    hist = [ids[b, int(pad[b].sum()):].tolist() + [int(first[b])] for b in range(B)]
    t0 = [int(first[b]) for b in range(B)]
    unf = [t not in eos for t in t0]
    left = [n] * B
    drafts = [LO.lookup(hist[b], G, Nn, eos, min(G, n - 1)) if unf[b] else [] for b in range(B)]
    out = [[] for _ in range(B)]
    ks, backs = [], []
    while any(u and l > 0 for u, l in zip(unf, left)):
        live = [u and l > 0 for u, l in zip(unf, left)]
        k = max(len(d) for d, l in zip(drafts, live) if l) + 1
        fed = [[t0[b]] + drafts[b] + [t0[b]] * (k - 1 - len(drafts[b])) for b in range(B)]
        toks, _ = dec.sample(torch.tensor(fed, device="cuda"))
        toks = toks.cpu().tolist()
        back = []
        for b in range(B):
            s = LO.settle(fed[b], toks[b], len(drafts[b]), unf[b], left[b], eos)
            if not live[b]:
                back.append(k)
                drafts[b] = []
                continue
            out[b] += s.emitted
            hist[b] += s.emitted
            unf[b], left[b], t0[b] = s.unfinished, s.left, s.t0
            back.append(k - 1 - s.accepted)
            drafts[b] = LO.lookup(hist[b], G, Nn, eos, min(G, left[b] - 1)) if unf[b] and left[b] > 0 else []
        dec.rewind(back)
        ks.append(k)
        backs.append(back)
    return out, ks, backs


def _run(dec, first, n, G, Nn):
    backs = []
    rewind = dec.rewind

    def spy(counts):
        backs.append(list(counts))
        rewind(counts)

    dec.rewind = spy
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            got, stats = dec.prompt_lookup_generate(first, n, num_output_tokens=G, max_matching_ngram_size=Nn)
        finally:
            torch.cuda.set_sync_debug_mode(0)
            del dec.rewind
    syncs = [w for w in caught if "called a synchronizing" in str(w.message)]
    assert len(syncs) == stats["rounds"] + 1, [str(w.message) for w in syncs]
    return got, stats, backs


CASES = {
    "bf16-greedy-B1": ("bf16", 1, (0.0, 0, 1.0), {}, ()),
    "fp8-greedy-B4-pad": ("fp8", 4, (0.0, 0, 1.0), {}, (1, 3)),
    "bf16-topk-B4-pad": ("bf16", 4, (1.0, 10, 1.0), {}, (0, 2)),
    "fp8-topk-B1": ("fp8", 1, (0.8, 10, 1.0), {}, ()),
    "bf16-processors-B4": ("bf16", 4, (0.0, 0, 1.0), dict(repetition_penalty=1.3, no_repeat_ngram_size=3), (2,)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_prompt_lookup_generate_is_the_loop_of_public_methods(name):
    from perceiver_io_b200.generation import prompt_lookup_budget

    kind, B, vals, proc, pad_rows = CASES[name]
    n, G, Nn = 50, 10, 2   # 120 + 50 rows: both the 160-row and the 48-latent windows slide
    T = prompt_lookup_budget(n, G, B)
    runs = []
    for _ in range(2):
        dec, logits, ids, pad = _decoder(kind, B, T, pad_rows)
        dec.set_sampling(*vals, **proc)
        runs.append((dec, dec.draw(logits), ids, pad))
    (dec, first, ids, pad), (ref, first_r, _, _) = runs
    assert torch.equal(first, first_r)
    got, stats, backs = _run(dec, first, n, G, Nn)
    want, ks, want_backs = _loop(ref, first.cpu()[:, 0], n, G, Nn, ids, pad, ())
    assert got.tolist() == want
    assert stats["k"] == ks and backs == want_backs
    assert torch.equal(dec._bounds, ref._bounds) and (dec._fed, dec._lag, dec._remaining) == (
        ref._fed, ref._lag, ref._remaining)
    assert sum(stats["accepted"]) > 0, stats
    print(f"[lookup] {name}: {stats['rounds']} rounds for {n} tokens, accepted {stats['accepted']} of "
          f"{stats['proposed']}")


def test_eos_mid_run_pads_and_stops():
    B, n, G, Nn = 4, 40, 6, 2
    dec, logits, ids, pad = _decoder("bf16", B, 200, (1,))
    dec.set_sampling(1.0, 10, 1.0)   # sampled: a greedy row of this random model repeats one token
    first = dec.draw(logits)
    plain = dec.generate(first, n).cpu()
    # a token some row emits after its first one
    row, eos = next((b, t) for b in range(B) for t in plain[b].tolist() if t != int(first[b]))
    runs = []
    for _ in range(2):
        d, lg, _, _ = _decoder("bf16", B, 200, (1,))
        d.set_sampling(1.0, 10, 1.0, eos_token_id=eos, pad_token_id=3)
        runs.append((d, d.draw(lg)))
    (dec, first), (ref, first_r) = runs
    got, stats, backs = _run(dec, first, n, G, Nn)
    want, ks, want_backs = _loop(ref, first_r.cpu()[:, 0], n, G, Nn, ids, pad, (eos,))
    for b in range(B):
        assert got[b, :len(want[b])].tolist() == want[b]
        assert (got[b, len(want[b]):] == 3).all()
    assert want[row] and want[row][-1] == eos
    assert stats["k"] == ks and backs == want_backs


def test_greedy_agrees_with_plain_generate_up_to_a_near_tie():
    B, n, G, Nn = 4, 40, 10, 2
    dec, logits, _, _ = _decoder("bf16", B, 200, (1,))
    dec.set_sampling(0.0)
    first = dec.draw(logits)
    plain, lg = dec.generate(first, n, logits=True)
    plain, lg = plain.cpu(), lg.float().cpu()
    # the extend-vs-step difference on these rows: the same 16 tokens fed in one replay and one at a time
    dec.rewind(n)
    fed = torch.cat([first, plain[:, :15].cuda()], dim=1)
    ext = dec.extend(fed).float().cpu()
    dec.rewind(16)
    steps = torch.stack([dec.step(fed[:, i:i + 1]).float().cpu() for i in range(16)], dim=1)
    diff = (ext - steps).abs().max().item()
    lk, logits2, _, _ = _decoder("bf16", B, 200, (1,))
    lk.set_sampling(0.0)
    got, stats = lk.prompt_lookup_generate(lk.draw(logits2), n, num_output_tokens=G, max_matching_ngram_size=Nn)
    got = got.cpu()
    for b in range(B):
        neq = (got[b] != plain[b]).nonzero()
        if len(neq) == 0:
            continue
        i = int(neq[0])
        top = lg[b, i].topk(2).values
        margin = float(top[0] - top[1])
        assert margin <= 2 * diff + 1e-6, (b, i, margin, diff)
    print(f"[lookup] greedy vs generate: extend-vs-step difference {diff:.3e}, {stats['rounds']} rounds")


def test_a_run_at_exactly_the_stated_budget_completes():
    from perceiver_io_b200.generation import prompt_lookup_budget

    for B in (1, 4):
        n, G = 30, 10
        need = prompt_lookup_budget(n, G, B)
        dec, logits, _, _ = _decoder("bf16", B, need, (1,) if B > 1 else ())
        dec.set_sampling(0.0)
        first = dec.draw(logits)
        got, _ = dec.prompt_lookup_generate(first, n, num_output_tokens=G)
        assert got.shape == (B, n) and dec._remaining >= 0
        dec2, logits2, _, _ = _decoder("bf16", B, need - 1, (1,) if B > 1 else ())
        with pytest.raises(RuntimeError, match=f"needs {need}"):
            dec2.prompt_lookup_generate(dec2.draw(logits2), n, num_output_tokens=G)
