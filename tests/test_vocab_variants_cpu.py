"""CPU companion of test_gpu_vocab_variants.py: the restated rules of vocab_variants.py against plain numpy
selections on every probe, the structure every probe builder claims, the mutants of the oracles that the probe set must
reject (the evidence that the GPU tests would catch a subtly wrong kernel), and the rule for a sampling row with no
finite mass in sample_oracle and spec_oracle."""
import numpy as np
import pytest

import process_oracle as PO
import vocab_variants as VV
from oracle import sample_oracle as S
from oracle import spec_oracle as SP


def _selection_probes(dt):
    out = []
    for V in VV.VOCABS:
        out += VV.radix_probes(V, dt) + VV.max_probes(V, dt, V)
        out += VV.zero_probes(V, max(1, V // 2), dt, V) + VV.zero_probes(V, min(4, V - 1), dt, V + 1)
        for n in (4, 16, 40):
            out += VV.tie_probes(V, n, dt, V + n) + VV.inf_probes(V, min(n, V), dt, V + n)
    return out


@pytest.fixture(scope="module")
def probes():
    return {dt: _selection_probes(dt) for dt in VV.DTYPES}


# ---- the restated rules -------------------------------------------------------------------------------------------------
def test_segments_cover_every_shape():
    shapes = {V: VV.segment_shape(V) for V in VV.VOCABS}
    for V, (live, last, seg, empty) in shapes.items():
        segs = [VV.warp_segment(V, w) for w in range(VV.WARPS)]
        covered = [i for s0, s1 in segs for i in range(s0, s1)]
        assert covered == list(range(V)), V
    assert any(live == 1 and last < 32 for live, last, _, _ in shapes.values())       # one ragged warp
    assert any(live == 1 and last == 32 for live, last, _, _ in shapes.values())      # one full warp
    assert shapes[33] == (2, 1, 32, 14) and shapes[513] == (9, 1, 64, 7)            # a one-element last warp, empties
    assert shapes[511] == (16, 31, 32, 0) and shapes[512] == (16, 32, 32, 0)
    assert shapes[32767] == (16, 2047, 2048, 0) and shapes[32768] == (16, 2048, 2048, 0)


@pytest.mark.parametrize("dt", VV.DTYPES)
def test_restated_select_and_collect_equal_numpy_sorts(dt, probes):
    for p in probes[dt]:
        keys = np.sort(VV.order_key(p.x))[::-1]
        for k in {p.k, 1, p.x.shape[0]}:
            assert VV.select_key(p.x, k)[0] == int(keys[k - 1]), (p.name, k)
            assert VV.collect_top(p.x, k) == VV.top_reference(p.x, k), (p.name, k)
        assert VV.representable(p.x, dt), p.name


def test_every_radix_pass_decides_in_each_sign_half():
    seen = {}
    for dt in VV.DTYPES:
        for V in VV.VOCABS:
            for p in VV.radix_probes(V, dt):
                if p.claim["pass_"] is not None:
                    seen.setdefault(dt, set()).add((p.claim["pass_"], p.claim["negative"]))
                    keys = np.sort(VV.order_key(p.x))[::-1]
                    assert int(keys[p.k - 1]) - int(keys[p.k]) == 1 or dt != "fp32", p.name   # consecutive fp32 keys
    assert seen["fp32"] == {(q, neg) for q in (1, 2, 3, 4) for neg in (False, True)}
    assert seen["bf16"] == {(q, neg) for q in (1, 2) for neg in (False, True)}
    assert {q for q, _ in seen["fp16"]} >= {2, 3}


def test_zero_probes_cut_at_the_sign_change():
    for dt in VV.DTYPES:
        tie, sub0, zsub = VV.zero_probes(513, 100, dt, 1)
        i0, i1 = tie.claim["at"]
        assert np.signbit(tie.x[i0]) and tie.x[i0] == 0 and not np.signbit(tie.x[i1]) and tie.x[i1] == 0
        assert VV.collect_top(tie.x, 100)[-1] == i0       # -0 and +0 tie: the lower index is taken
        if dt == "fp32":
            assert VV.deciding_pass(sub0.x, 100) == 4 and VV.deciding_pass(zsub.x, 100) == 1


# ---- structure ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", VV.DTYPES)
def test_sampler_probes_are_exact(dt, probes):
    """slack == 0: every mass of every sampler probe is exact, so every draw is the oracle's bit for bit."""
    rows = [p.x for p in probes[dt] if np.isfinite(p.x).any()]
    rows += [p.x for V in VV.VOCABS for p in VV.top_p_probes(V, dt)]
    rows += [p.x for p, _ in VV.segment_draw_probes(dt)] + [VV.dense_draw_probe(dt).x]
    for x in rows:
        assert S.filter_row(x, 1.0, 0, 1.0).slack == 0


@pytest.mark.parametrize("dt", VV.DTYPES)
def test_top_p_probes_sit_on_the_cut(dt):
    n = 0
    for V in VV.VOCABS:
        for p in VV.top_p_probes(V, dt):
            c = p.claim
            f = S.filter_row(p.x, 1.0, 0, c["top_p"])
            assert c["W"] == f.cut + c["over"] and c["slack"] == 0, p.name
            g = p.x == np.float32(c["group"])
            assert g.sum() == c["ng"] and (f.kept[g].all() if c["over"] else not f.kept[g].any()), p.name
            n += 1
    assert n >= 8 * (len(VV.VOCABS) - 2)


def test_tie_probes_straddle_the_segment_boundaries():
    kinds = set()
    for V in VV.VOCABS:
        for n in (4, 16, 40):
            for p in VV.tie_probes(V, n, "fp32", V):
                group, need = p.claim["group"], p.claim["need"]
                assert need < len(group) and p.claim["crosses"], p.name
                assert VV.collect_top(p.x, n)[-need:] and set(VV.collect_top(p.x, n)) >= set(group[:need])
                kinds.add(p.name.split(" V=")[0])
    assert kinds == {"tie across one boundary", "tie across several boundaries", "tie across the empty segments"}


def test_draw_probes_draw_both_tokens_and_land_in_the_mass_one_run():
    for dt in VV.DTYPES:
        for p, picks in VV.segment_draw_probes(dt):
            assert sorted(t for _, t in picks) == sorted(p.claim["tokens"])
            for pos, tok in picks:
                assert S.sample_row(p.x, 1.0, 0, 1.0, 5, 0, pos).token == tok
        assert {p.claim["empty_after"] for p, _ in VV.segment_draw_probes(dt)} == {False, True}
        d = VV.dense_draw_probe(dt)
        w, _ = VV.masses(d.x, d.x.max())
        assert (w[:-1] == 1).all() and w[-1] == VV.MASS_ONE
        for seed, b, pos in VV.DENSE_DRAW:
            t = (int(S.uniform_bits(np.uint64(seed), b, pos)) * int(w.sum())) >> 64
            assert t < VV.MAX_VOCAB - 1 and S.sample_row(d.x, 1.0, 0, 1.0, seed, b, pos).token == t


# ---- mutants ------------------------------------------------------------------------------------------------------------
def _topk_drops_ties(x, k):
    kept = np.zeros(x.shape[0], bool)
    kept[VV.top_reference(x, k)] = True
    return kept


def _top_p_kept(x, top_p, mode):
    f = S.filter_row(x, 1.0, 0, 1.0)
    cut = S.filter_row(x, 1.0, 0, top_p).cut
    if mode == "splits":   # token by token in ascending order (index order on ties)
        order = np.lexsort((np.arange(x.shape[0]), x.astype(np.float64)))
        cs = np.cumsum(f.w[order].astype(np.float64))
        kept = np.zeros(x.shape[0], bool)
        kept[order[cs > cut]] = True
        return kept
    over = np.nonzero(f.W >= np.uint64(cut))[0]   # "keeps W<= == cut"
    return x >= f.vals[over[0]]


def _draw_ge(x, seed, b, pos):
    f = S.filter_row(x, 1.0, 0, 1.0)
    t = (int(S.uniform_bits(np.uint64(seed), b, pos)) * f.z_kept) >> 64
    return int(np.searchsorted(np.cumsum(f.w), np.uint64(t), side="left"))


def _draw_without_last(x, seed, b, pos):
    y = x.copy()
    y[-1] = -np.inf
    return S.sample_row(y, 1.0, 0, 1.0, seed, b, pos).token


def _process_mutant(x, hist, mode, **kw):
    V, L, N = x.shape[0], len(hist), kw["no_repeat_ngram_size"]
    if mode == "L > N":          # the one n-gram start at L == N is skipped
        return PO.process(x, hist, **dict(kw, no_repeat_ngram_size=0)) if L == N else PO.process(x, hist, **kw)
    if mode == "L + 1 > N":
        return PO.process(x, hist, **dict(kw, no_repeat_ngram_size=0)) if L + 1 == N else PO.process(x, hist, **kw)
    out = PO.process(x, hist, **kw)   # "out of range": a banned id outside [0, V) is written at id mod V
    if L + 1 >= N:
        suffix = hist[L - N + 1:] if N > 1 else []
        for s in range(L - N + 1):
            if hist[s:s + N - 1] == suffix and not 0 <= hist[s + N - 1] < V:
                out[hist[s + N - 1] % V] = -np.inf
    return out


def test_the_probes_reject_every_mutant(capsys, probes):
    """Each mutant of an oracle rule differs from the rule on at least one probe; the probe is printed."""
    rejected = {}

    def note(mutant, name):
        rejected.setdefault(mutant, name)

    for dt in VV.DTYPES:
        for p in probes[dt]:
            x, k = p.x, p.k
            V = x.shape[0]
            if not np.array_equal(S.filter_row(x, 1.0, k, 1.0).kept, _topk_drops_ties(x, k)) and 0 < k < V:
                note("top-k drops ties with the k-th", p.name)
            ref = VV.top_reference(x, k)
            for mutant, kw in (("-0 != +0", dict(fold_zero=False)), ("ties highest index first", dict(eq_order="reversed")),
                               ("ties in reversed warp order", dict(eq_order="reversed_warps")),
                               ("the last warp segment loses its last element", dict(lose_last=True))):
                if VV.collect_top(x, k, **kw) != ref:
                    note(mutant, p.name)
            if V < 40 and not np.isfinite(x).all():
                keep = VV.beams_to_keep(8, 4)
                if not np.array_equal(VV.row_candidates(x, keep)[1], VV.row_candidates(x, keep, fillers_first=True)[1]):
                    note("beam fillers before -inf candidates", p.name)
        for V in VV.VOCABS:
            for p in VV.top_p_probes(V, dt):
                kept = S.filter_row(p.x, 1.0, 0, p.claim["top_p"]).kept
                for mode, mutant in (("keeps", "top-p keeps W<= == cut"), ("splits", "top-p splits a straddling group")):
                    if not np.array_equal(_top_p_kept(p.x, p.claim["top_p"], mode), kept):
                        note(mutant, p.name)
            for p, T, tok in VV.zero_mass_probes(V, dt):
                if p.claim["greedy"]:
                    assert S.sample_row(p.x, T, 0, 1.0, 1, 0, 0).token == tok
                    note("the zero-mass row writes nothing", p.name)
                    if tok != V - 1:
                        note("the zero-mass row writes token V-1", p.name)
        d = VV.dense_draw_probe(dt)
        for seed, b, pos in VV.DENSE_DRAW:
            if _draw_ge(d.x, seed, b, pos) != S.sample_row(d.x, 1.0, 0, 1.0, seed, b, pos).token:
                note("the draw uses >= for exceeds", d.name)
        for p, picks in VV.segment_draw_probes(dt):
            for pos, tok in picks:
                if _draw_without_last(p.x, 5, 0, pos) != tok:
                    note("the last warp segment loses its last element (draw)", p.name)
    rng = np.random.default_rng(0)
    equivalent = 0
    for V in VV.PROCESS_VOCABS:
        for name, hists, kw in VV.processor_cases(V, V):
            for h in hists:
                x = (rng.standard_normal(V) * 3).astype(np.float32)
                want = PO.process(x, h, **kw)
                if kw.get("repetition_penalty", 1.0) != 1.0 and V % 32:
                    hm = [t if t < 32 * (V // 32) else -1 for t in h]
                    if not np.array_equal(PO.process(x, hm, **kw), want):
                        note("seen has V/32 words", f"{name} V={V}")
                if "no_repeat_ngram_size" in kw:
                    N, L = kw["no_repeat_ngram_size"], len(h)
                    if L + 1 == N:
                        # `L + 1 > N` is equivalent to the kernel's `L + 1 >= N`: at L + 1 == N there is no n-gram start
                        assert np.array_equal(_process_mutant(x, h, "L + 1 > N", **kw), want)
                        equivalent += 1
                    if L == N and not np.array_equal(_process_mutant(x, h, "L > N", **kw), want):
                        note("the n-gram condition is L > N (its one start at L == N skipped)", f"{name} V={V}")
                    if not np.array_equal(_process_mutant(x, h, "out of range", **kw), want):
                        note("an out-of-range history id gets written", f"{name} V={V}")
    with capsys.disabled():
        for mutant, name in sorted(rejected.items()):
            print(f"[vocab] rejected: {mutant:<62} by {name}")
        print(f"[vocab] `L + 1 > N` agrees with `L + 1 >= N` on all {equivalent} rows at L + 1 == N (no start there)")
    assert equivalent > 0
    assert set(rejected) == {
        "top-k drops ties with the k-th", "-0 != +0", "ties highest index first", "ties in reversed warp order",
        "the last warp segment loses its last element", "the last warp segment loses its last element (draw)",
        "beam fillers before -inf candidates", "top-p keeps W<= == cut", "top-p splits a straddling group",
        "the zero-mass row writes nothing", "the zero-mass row writes token V-1", "the draw uses >= for exceeds",
        "seen has V/32 words", "the n-gram condition is L > N (its one start at L == N skipped)",
        "an out-of-range history id gets written"}


# ---- the zero-mass rule -------------------------------------------------------------------------------------------------
def test_a_row_without_finite_mass_is_greedy_in_both_oracles():
    V = 40
    ninf = np.full(V, -np.inf, np.float32)
    big = np.linspace(-3, 3, V).astype(np.float32)
    big[[30, 7]] = 3e38                       # / 0.5 overflows: +inf at 7 and 30
    one = ninf.copy()
    one[11] = -2.0
    for x, T, tok in ((ninf, 1.0, 0), (ninf, 0.3, 0), (big, 0.5, 7), (one, 1.0, 11)):
        assert S.greedy_token(x, T) == (None if x is one else tok)
        d = S.sample_row(x, T, 5, 0.9, seed=3, b=0, pos=1)
        assert d.token == tok and d.logprob == 0.0 and not d.ambiguous
        p = S.probs(x, T, 0, 1.0)
        assert p[tok] == 1.0 and p.sum() == 1.0
        f = S.filter_row(x, T, 0, 0.5)
        assert f.kept.sum() == 1 and f.kept[tok] and f.z_kept == VV.MASS_ONE and f.slack == 0
        m = SP.masses(x, T, 0, 1.0)
        assert m.w[tok] == SP.ONE and m.Z == SP.ONE and sum(m.w) == SP.ONE
    assert S.greedy_token(big, 1.0) is None   # 3e38 itself is finite
    # the verifier: a zero-mass target row rejects any other draft and corrects to its greedy token; a zero-mass draft
    # row is a greedy draft (Q one-hot at 0), accepted with probability min(1, p(0))
    rng = np.random.default_rng(1)
    tgt = (rng.standard_normal((2, V)) * 2).astype(np.float32)
    drf = (rng.standard_normal((1, V)) * 2).astype(np.float32)
    v = SP.verify_row(np.stack([ninf, tgt[1]]), drf, [4, 9], (1.0, 0, 1.0), (1.0, 0, 1.0), 7, 0, [0, 1])
    assert v.tokens == [0, -1] and v.n == 0
    v = SP.verify_row(tgt, ninf[None], [4, 0], (1.0, 0, 1.0), (0.8, 0, 1.0), 7, 0, [0, 1])
    assert v.n in (0, 1) and not v.ambiguous and (v.n == 1) == (v.tokens[0] == 0)
