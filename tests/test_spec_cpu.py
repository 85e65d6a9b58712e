"""CPU checks of speculative sampling (pcv_spec_verify) and its host logic.

The oracle's rule (oracle/spec_oracle.py) is exact: with every uniform counted in closed form, the first emitted token
is distributed as the target's filtered p to within V 2^-63 and a draft is accepted with probability Σ min(p, q) to
within 2^-62.  The accept and residual streams are uniform and independent of each other and of the draw stream.
Every refusal of the C ABI comes before any CUDA call and the ctypes layout matches the header.  GraphedDecoder.verify,
generate(logits=True) and speculative_generate are checked on fake graphs: refusals, draw positions, per-row rewinds,
token assembly, the stated budget and one device read per round."""
import ctypes
import math
import os
import types
from fractions import Fraction

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import sample_oracle as S
from oracle import spec_oracle as SP
from perceiver_io_b200 import _lib

TWO64 = 1 << 64


# ---- the rule is exact ------------------------------------------------------------------------------------------------
def _below(c: int, total: int) -> int:
    """#{u in [0, 2^64): (u * total) >> 64 < c}: the first ceil(c 2^64 / total) values."""
    return min(TWO64, -(-c * TWO64 // total))


def _emitted(P: SP.Masses, Q: SP.Masses):
    """(distribution of the first emitted token, acceptance probability) of one round with a draft x ~ Q / Zq, every
    uniform counted in closed form."""
    V = len(P.w)
    R = SP.residual(P, Q)
    SR = sum(R)
    weights, total = (R, SR) if SR else (P.w, P.Z)
    res, acc = [], 0
    for v in weights:                          # P(residual draw = y)
        res.append(Fraction(_below(acc + v, total) - _below(acc, total), TWO64))
        acc += v
    dist = [Fraction(0)] * V
    accept = Fraction(0)
    for x in range(V):
        if not Q.w[x]:
            continue
        qx = Fraction(Q.w[x], Q.Z)
        a = Fraction(_below(P.w[x] * Q.Z, Q.w[x] * P.Z), TWO64)   # accept iff hi(u Q(x) Zp) < P(x) Zq
        accept += qx * a
        dist[x] += qx * a
        for y in range(V):
            dist[y] += qx * (1 - a) * res[y]
    return dist, accept


TRIPLES = {
    "greedy/greedy": ((0.0, 0, 1.0), (0.0, 0, 1.0)),
    "greedy/sampled": ((0.0, 0, 1.0), (1.0, 0, 1.0)),
    "sampled/greedy": ((1.0, 0, 1.0), (0.0, 0, 1.0)),
    "top-k": ((1.0, 3, 1.0), (1.0, 5, 1.0)),
    "top-p": ((1.0, 0, 0.7), (1.0, 0, 0.9)),
    "temperatures": ((0.6, 0, 1.0), (1.7, 0, 1.0)),
}


@pytest.mark.parametrize("name", list(TRIPLES))
def test_rule_emits_the_target_distribution_and_accepts_sum_min(name):
    tp, tq = TRIPLES[name]
    rng = np.random.default_rng(len(name))
    for trial in range(6):
        V = int(rng.integers(2, 13))
        lp = (rng.standard_normal(V) * 1.5).astype(np.float32)
        lq = (lp + rng.standard_normal(V) * (0.2 + trial * 0.3)).astype(np.float32)
        P, Q = SP.masses(lp, *tp), SP.masses(lq, *tq)
        dist, accept = _emitted(P, Q)
        p = [Fraction(w, P.Z) for w in P.w]
        q = [Fraction(w, Q.Z) for w in Q.w]
        assert sum(dist) == 1
        for y in range(V):
            assert abs(dist[y] - p[y]) <= Fraction(V, 2 ** 63), (name, trial, y, float(dist[y]), float(p[y]))
        assert abs(accept - sum(min(a, b) for a, b in zip(p, q))) <= Fraction(1, 2 ** 62), (name, trial)


def test_uniform_drafts_are_always_accepted():
    """The issue's example: p and q uniform over the same 10 tokens: Σ p q = 0.1 but Σ min(p, q) = 1."""
    lp = np.array([0.0] * 10 + [-60.0] * 6, dtype=np.float32)
    P = SP.masses(lp, 1.0, 10, 1.0)
    Q = SP.masses(lp * 0.5, 1.0, 10, 1.0)
    _, accept = _emitted(P, Q)
    assert accept == 1


def test_verify_row_follows_the_counters():
    """verify_row's accept / residual / bonus decisions are the integer rule at the stream bits of each position."""
    rng = np.random.default_rng(3)
    V, G = 9, 4
    tgt = rng.standard_normal((G + 1, V)).astype(np.float32)
    dft = (tgt[:G] + rng.standard_normal((G, V))).astype(np.float32)
    for seed in range(40):
        toks = [5] + [int(t) for t in rng.integers(0, V, G)]
        pos = list(range(100 + seed, 100 + seed + G + 1))
        v = SP.verify_row(tgt, dft, toks, (1.0, 0, 1.0), (1.0, 0, 1.0), seed, 2, pos)
        n = v.n
        for i in range(n):
            P, Q = SP.masses(tgt[i], 1.0, 0, 1.0), SP.masses(dft[i], 1.0, 0, 1.0)
            u = int(SP.stream_bits(np.uint64(seed), 2, pos[i], "accept"))
            assert (u * Q.w[toks[i + 1]] * P.Z) >> 64 < P.w[toks[i + 1]] * Q.Z
        assert v.tokens[:n] == toks[1:n + 1] and v.tokens[n] >= 0 and v.tokens[n + 1:] == [-1] * (G - n)


def test_adversarial_draft_with_no_mass_falls_back_to_p():
    """A greedy draft on a token P gives no mass is rejected; with P = Q (ΣR = 0) the correction is P's draw."""
    lp = np.array([3.0, 1.0, -80.0, 0.5], dtype=np.float32)
    out = SP.verify_row(np.stack([lp, lp]), lp[None], [0, 2], (1.0, 0, 1.0), (1.0, 0, 1.0), 7, 0, [10, 11])
    assert out.n == 0
    P = SP.masses(lp, 1.0, 0, 1.0)
    t = (int(SP.stream_bits(np.uint64(7), 0, 10, "residual")) * P.Z) >> 64
    assert out.tokens == [SP.first_exceeding(P.w, t)[0], -1]


# ---- the streams ------------------------------------------------------------------------------------------------------
N_HASH = 1 << 20


def _uniform01(bits):
    return (bits >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


@pytest.mark.parametrize("stream", ["accept", "residual"])
def test_spec_streams_are_uniform(stream):
    pos = np.arange(N_HASH, dtype=np.int64)
    for seed, b in ((0, 0), (12345, 3), (2 ** 63 + 7, 1)):
        bits = SP.stream_bits(np.uint64(seed), b, pos, stream)
        for shift in (0, 24, 56):
            counts = np.bincount(((bits >> np.uint64(shift)) & np.uint64(255)).astype(np.int64), minlength=256)
            chi2 = ((counts - N_HASH / 256) ** 2 / (N_HASH / 256)).sum()
            assert chi2 < 255 + 6 * np.sqrt(2 * 255), (seed, b, shift, chi2)
        assert abs(_uniform01(bits).mean() - 0.5) < 6 * np.sqrt(1 / 12 / N_HASH)
        assert len(np.unique(bits)) == N_HASH


def test_accept_residual_and_draw_streams_are_independent():
    pos = np.arange(N_HASH, dtype=np.int64)
    floor = 6 / np.sqrt(N_HASH)
    streams = {"draw": S.uniform_bits(np.uint64(1000), 2, pos),
               "accept": SP.stream_bits(np.uint64(1000), 2, pos, "accept"),
               "residual": SP.stream_bits(np.uint64(1000), 2, pos, "residual")}
    names = list(streams)
    for i, a in enumerate(names):
        for c in names[i + 1:]:
            x, y = streams[a], streams[c]
            assert abs(np.corrcoef(_uniform01(x), _uniform01(y))[0, 1]) < floor, (a, c)
            agree = np.mean((x >> np.uint64(63)) == (y >> np.uint64(63)))
            assert abs(agree - 0.5) < 6 * 0.5 / np.sqrt(N_HASH), (a, c)
            assert not np.any(x == y), (a, c)
    for what, other in (("adjacent seed", SP.stream_bits(np.uint64(1001), 2, pos, "accept")),
                        ("adjacent row", SP.stream_bits(np.uint64(1000), 3, pos, "accept")),
                        ("adjacent position", SP.stream_bits(np.uint64(1000), 2, pos + 1, "accept"))):
        assert abs(np.corrcoef(_uniform01(streams["accept"]), _uniform01(other))[0, 1]) < floor, what


# ---- the C ABI --------------------------------------------------------------------------------------------------------
def _params(**kw):
    p = _lib.SpecVerifyParams()
    p.target, p.t_stride_b, p.t_stride_row = 0x1000, 5 * 400, 400
    p.draft, p.d_stride_b, p.d_stride_row = 0x2000, 4 * 400, 400
    p.tokens, p.seeds, p.positions = 0x3000, 0x4000, 0x5000
    p.B, p.G, p.V, p.dtype, p.draft_dtype = 3, 4, 389, _lib.PCV_BF16, _lib.PCV_BF16
    p.temperature, p.top_k, p.top_p = 1.0, 10, 0.9
    p.draft_temperature, p.draft_top_k, p.draft_top_p = 0.8, 0, 1.0
    p.out_tokens, p.accepted = 0x6000, 0x7000
    for k, v in kw.items():
        setattr(p, k, v)
    return p


REFUSALS = [(dict(**{f: None}), b"pointer is NULL") for f in
            ("target", "draft", "tokens", "seeds", "positions", "out_tokens", "accepted")] + [
    (dict(V=0), b"V=0 must be in [1, 32768]"),
    (dict(V=32769, t_stride_b=10 ** 6, t_stride_row=40000, d_stride_b=10 ** 6, d_stride_row=40000),
     b"V=32769 must be in [1, 32768]"),
    (dict(G=0), b"G=0 must be in [1, 63]"),
    (dict(G=64), b"G=64 must be in [1, 63]"),
    (dict(B=0), b"B=0 must be >= 1"),
    (dict(t_stride_row=388), b"is below V=389"),
    (dict(t_stride_b=388), b"is below V=389"),
    (dict(d_stride_row=388), b"is below V=389"),
    (dict(d_stride_b=100), b"is below V=389"),
    (dict(draft_dtype=_lib.PCV_F16), b"differs from the target logits' dtype"),
    (dict(dtype=_lib.PCV_E4M3, draft_dtype=_lib.PCV_E4M3), b"unknown dtype 3"),
    (dict(out_tokens=0x3000 + 8 * 7), b"out_tokens overlaps tokens"),
    (dict(temperature=-1.0), b"target temperature must be >= 0"),
    (dict(top_k=-1), b"target top_k must be >= 0"),
    (dict(top_p=0.0), b"target top_p must be in (0, 1]"),
    (dict(draft_temperature=float("nan")), b"draft temperature must be >= 0"),
    (dict(draft_top_k=-3), b"draft top_k must be >= 0"),
    (dict(draft_top_p=1.5), b"draft top_p must be in (0, 1]"),
]


@pytest.mark.parametrize("kw,reason", REFUSALS, ids=[f"refuse{i}" for i in range(len(REFUSALS))])
def test_abi_refusals_come_before_any_cuda_call(kw, reason):
    lib = _lib.lib()
    p = _params(**kw)
    assert lib.pcv_spec_verify_supported(ctypes.byref(p)) == 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()
    assert lib.pcv_spec_verify(ctypes.byref(p), None) != 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()


def test_abi_accepts_the_edges_and_refuses_null():
    lib = _lib.lib()
    for kw in (dict(), dict(V=1, t_stride_b=1, t_stride_row=1, d_stride_b=1, d_stride_row=1), dict(G=1), dict(G=63),
               dict(V=32768, t_stride_b=32768, t_stride_row=32768, d_stride_b=32768, d_stride_row=32768),
               dict(temperature=0.0, draft_temperature=0.0), dict(dtype=_lib.PCV_F32, draft_dtype=_lib.PCV_F32)):
        assert lib.pcv_spec_verify_supported(ctypes.byref(_params(**kw))) == 1, (kw, lib.pcv_last_error())
    assert lib.pcv_spec_verify_supported(None) == 0 and b"params is NULL" in lib.pcv_last_error()
    assert lib.pcv_spec_uniforms(None, 0x10, 0x20, 4, 1, 0, None) != 0 and b"NULL" in lib.pcv_last_error()
    assert lib.pcv_spec_uniforms(0x30, 0x10, 0x20, 5, 2, 0, None) != 0
    assert b"multiple of rows_per_batch=2" in lib.pcv_last_error()
    assert lib.pcv_spec_uniforms(0x30, 0x10, 0x20, 4, 2, 2, None) != 0
    assert b"stream_id=2" in lib.pcv_last_error()


def test_spec_params_layout_matches_the_header(tmp_path):
    import subprocess

    header = os.path.join(ROOT, "include", "pcv_attn.h")
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void){",
             'printf("size %zu\\n", sizeof(pcv_spec_verify_params));',
             'printf("maxdrafts %d\\n", PCV_SPEC_MAX_DRAFTS);']
    lines += [f'printf("{f} %zu\\n", offsetof(pcv_spec_verify_params, {f}));' for f, _ in _lib.SpecVerifyParams._fields_]
    lines.append("return 0;}")
    (tmp_path / "l.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-o", str(tmp_path / "l"), str(tmp_path / "l.c")])
    got = dict(l.split() for l in subprocess.check_output([str(tmp_path / "l")]).decode().split("\n") if l)
    assert int(got["size"]) == ctypes.sizeof(_lib.SpecVerifyParams)
    assert int(got["maxdrafts"]) == _lib.SPEC_MAX_DRAFTS == 63
    for f, _ in _lib.SpecVerifyParams._fields_:
        assert int(got[f]) == getattr(_lib.SpecVerifyParams, f).offset, f


def test_spec_kernels_have_no_spills():
    log = os.path.join(ROOT, "build", "pcv_sample.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was not built in this tree")
    text = open(log).read()
    entries = text.split("Compiling entry function")[1:]
    names = ("spec_verify_kernel", "spec_resolve_kernel", "spec_uniforms_kernel")
    kernels = [e for e in entries if any(n in e.split("\n")[0] for n in names)]
    assert len(kernels) == 5, len(kernels)   # three logits dtypes, resolve, uniforms
    for e in kernels:
        assert "0 bytes spill stores, 0 bytes spill loads" in e, e[:300]
    assert "C7515" not in text and "C7512" not in text


def test_ops_refuse_before_any_launch():
    from perceiver_io_b200 import ops

    with pytest.raises(ValueError, match="stream must be 'accept' or 'residual'"):
        ops.spec_uniforms(torch.zeros(1, dtype=torch.long), torch.zeros(1, dtype=torch.int32), "draw")


# ---- GraphedDecoder and speculative_generate on fake graphs -------------------------------------------------------------
class _Acc:
    """Stands in for the device's accepted counts; counts the reads to the host."""

    def __init__(self, counts, reads):
        self.counts, self.reads = counts, reads

    def to(self, device):
        assert device == "cpu"
        self.reads.append(1)
        return torch.tensor(self.counts, dtype=torch.int32)


class _SpecGraphs(dict):
    """Fake graphs: a replay moves the bounds as _step_fn does and records what it was given.  The draft's sampling
    replays return tokens 7 (and logits rows); the verify replays return scripted accept counts."""

    def __init__(self, dec, script=None, V=11):
        super().__init__()
        self.dec, self.script, self.V, self.calls, self.reads = dec, list(script or []), V, [], []

    def get(self, key):
        from perceiver_io_b200.generation import advance_bounds_, sample_positions

        k = key[1] if isinstance(key, tuple) else key

        def replay(tokens, *extra):
            d = self.dec
            pos = sample_positions(d._bounds, d._steps, k)
            self.calls.append((key, tokens.clone(), pos, [e.clone() for e in extra]))
            advance_bounds_(d._bounds, d._inc, d._wmax, k)
            if key[0] == "verify":
                counts = self.script.pop(0)
                out = torch.full((d.batch, k), -1, dtype=torch.long)
                for b, n in enumerate(counts):
                    out[b, :n] = tokens[b, 1:n + 1]
                    out[b, n] = 500 + len(self.calls) * 10 + b
                return out, _Acc(counts, self.reads)
            return (torch.full((d.batch, k), 7, dtype=torch.long) + pos.long(),
                    torch.arange(d.batch * k * self.V, dtype=torch.float32).view(d.batch, k, self.V) + len(self.calls))

        return replay


def _decoder(B=3, T=40, script=None, V=11):
    from test_window_rows_cpu import _decoder as rows_decoder

    dec = rows_decoder(B, 30, 10, 40, 16, T)
    dec._graphs = _SpecGraphs(dec, script, V)
    dec._seeds, dec._seeded, dec._sampling = torch.zeros(B, dtype=torch.int64), True, (1.0, 0, 1.0)
    dec._steps = torch.arange(1, 65, dtype=torch.int32)
    dec.dtype = torch.float32
    dec.model = types.SimpleNamespace(config=types.SimpleNamespace(vocab_size=V))
    return dec


def test_generate_with_logits_returns_each_draws_logits():
    dec = _decoder()
    toks, lg = dec.generate(torch.zeros(3, 1, dtype=torch.long), 4, logits=True)
    assert toks.shape == (3, 4) and lg.shape == (3, 4, 11)
    for i in range(4):
        assert torch.equal(lg[:, i], torch.arange(33, dtype=torch.float32).view(3, 11) + i + 1)
    assert torch.equal(dec.generate(torch.zeros(3, 1, dtype=torch.long), 2), toks[:, :2] + 4)


def test_verify_refusals_leave_the_state_untouched():
    dec = _decoder(T=10, script=[[0, 0, 0]])
    ok_t, ok_q = torch.zeros(3, 4, dtype=torch.long), torch.zeros(3, 3, 11)
    dec.generate(torch.zeros(3, 1, dtype=torch.long), 5)
    before = (dec._bounds.clone(), dec._fed, dec._remaining, len(dec._graphs.calls))
    for args, exc, match in (
            ((torch.zeros(3, 1, dtype=torch.long), torch.zeros(3, 0, 11)), ValueError, "1 <= G <= 63"),
            ((torch.zeros(3, 65, dtype=torch.long), torch.zeros(3, 64, 11)), ValueError, "1 <= G <= 63"),
            ((ok_t, torch.zeros(3, 2, 11)), ValueError, r"\(3, 3, 11\) torch.float32 draft logits"),
            ((ok_t, torch.zeros(3, 3, 12)), ValueError, "draft logits"),
            ((ok_t, torch.zeros(3, 3, 11, dtype=torch.float16)), ValueError, "draft logits"),
            ((torch.zeros(2, 4, dtype=torch.long), torch.zeros(3, 3, 11)), ValueError, "int64 tokens"),
            ((torch.zeros(3, 6, dtype=torch.long), torch.zeros(3, 5, 11)), RuntimeError, "5 of max_new_tokens=10")):
        with pytest.raises(exc, match=match):
            dec.verify(*args)
    for bad in ((-1.0, 0, 1.0), (1.0, -2, 1.0), (1.0, 0, 0.0), (1.0, 0)):
        with pytest.raises(ValueError, match="draft_sampling"):
            dec.verify(ok_t, ok_q, draft_sampling=bad)
    assert torch.equal(dec._bounds, before[0]) and (dec._fed, dec._remaining, len(dec._graphs.calls)) == before[1:]
    for call in (lambda: dec.generate(torch.zeros(3, 2, dtype=torch.long), 1, logits=True),
                 lambda: dec.generate(torch.zeros(3, 1, dtype=torch.long), 6, logits=True)):
        with pytest.raises((ValueError, RuntimeError)):
            call()
    assert torch.equal(dec._bounds, before[0]) and (dec._fed, dec._remaining) == before[1:3]
    fresh = _decoder()
    fresh._bounds = None
    with pytest.raises(RuntimeError, match="prefill"):
        fresh.verify(ok_t, ok_q)


def test_verify_draws_at_the_sample_positions():
    dec = _decoder(script=[[1, 0, 3], [2, 2, 2]])
    dec.rewind([0, 0, 0])
    dec.generate(torch.zeros(3, 1, dtype=torch.long), 2)
    dec.rewind([1, 0, 2])
    tok, acc = dec.verify(torch.zeros(3, 4, dtype=torch.long), torch.zeros(3, 3, 11), draft_sampling=(0.5, 3, 0.9))
    key, _, pos, extra = dec._graphs.calls[-1]
    assert key == ("verify", 4, (1.0, 0, 1.0), (0.5, 3, 0.9))
    fed = [1, 2, 0]
    assert pos.tolist() == [[30 + f + 1 + i for i in range(4)] for f in fed]
    assert extra[0].shape == (3, 3, 11)


@pytest.mark.parametrize("B,G,n", [(1, 3, 7), (3, 2, 9), (2, 4, 5)])
def test_speculative_generate_rewinds_assembles_and_reads_once_per_round(B, G, n):
    from perceiver_io_b200.generation import speculative_budget, speculative_generate

    rng = np.random.default_rng(B * 100 + G)
    script = [[int(c) for c in rng.integers(0, G + 1, B)] for _ in range(4 * n)]
    need = speculative_budget(n, G, B)
    tgt, dft = _decoder(B=B, T=need, script=list(script)), _decoder(B=B, T=need)
    first = torch.full((B, 1), 3, dtype=torch.long)
    out, stats = speculative_generate(tgt, dft, first, n, draft_tokens=G)
    rounds = stats["rounds"]
    assert len(tgt._graphs.reads) == rounds   # one device read per round
    # replay the script: each row's emitted tokens in order, its rewinds and its fed count
    done, fed, t0 = [0] * B, [0] * B, [3] * B
    want = [[] for _ in range(B)]
    verify_calls = [c for c in tgt._graphs.calls if c[0][0] == "verify"]
    assert len(verify_calls) == rounds
    for r in range(rounds):
        key, toks, pos, _ = verify_calls[r]
        assert toks[:, 0].tolist() == t0
        counts = script[r]
        for b in range(B):
            assert pos[b].tolist() == [30 + fed[b] + 1 + i for i in range(G + 1)]
            if done[b] >= n:
                continue
            nb = counts[b]
            emitted = toks[b, 1:nb + 1].tolist() + [500 + (r + 1) * 10 + b]
            want[b] += emitted
            done[b] += nb + 1
            fed[b] += nb + 1
            t0[b] = emitted[-1]
            assert stats["accepted"][b] >= 0
    assert out.tolist() == [w[:n] for w in want]
    assert fed == [tgt._fed - (tgt._lag[b] if tgt._lag else 0) for b in range(B)]
    assert fed == [dft._fed - (dft._lag[b] if dft._lag else 0) for b in range(B)]
    assert stats["proposed"] == [G * sum(1 for r in range(rounds) if sum(min(script[q][b], G) + 1
                                                                          for q in range(r)) < n) for b in range(B)]


@pytest.mark.parametrize("B", [1, 2])
def test_speculative_generate_needs_exactly_its_stated_budget(B):
    from perceiver_io_b200.generation import speculative_budget, speculative_generate

    G, n = 3, 6
    need = speculative_budget(n, G, B)
    # the worst case: row 0 accepts everything (overshoots to n + G), row 1 accepts nothing
    script = [[G] + [0] * (B - 1)] * 20
    for T, ok in ((need - 1, False), (need, True)):
        tgt, dft = _decoder(B=B, T=T, script=list(script)), _decoder(B=B, T=T)
        first = torch.zeros(B, 1, dtype=torch.long)
        if not ok:
            with pytest.raises(RuntimeError, match=f"needs {need}"):
                speculative_generate(tgt, dft, first, n, draft_tokens=G)
            assert tgt._graphs.calls == [] and dft._graphs.calls == []
            continue
        out, stats = speculative_generate(tgt, dft, first, n, draft_tokens=G)
        assert out.shape == (B, n)
        assert tgt._remaining >= 0 and dft._remaining >= 0


def test_speculative_generate_refusals():
    from perceiver_io_b200.generation import speculative_generate

    tgt, dft = _decoder(), _decoder(B=2)
    first = torch.zeros(3, 1, dtype=torch.long)
    with pytest.raises(ValueError, match="batch 2 != the target's 3"):
        speculative_generate(tgt, dft, first, 4)
    dft = _decoder(V=12)
    with pytest.raises(ValueError, match="vocabulary 12 != the target's 11"):
        speculative_generate(tgt, dft, first, 4)
    dft = _decoder()
    for kw, match in ((dict(draft_tokens=0), "draft_tokens"), (dict(draft_tokens=64), "draft_tokens"),
                      (dict(n=0), "n must be")):
        args = dict(n=4, draft_tokens=2)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            speculative_generate(tgt, dft, first, args["n"], draft_tokens=args["draft_tokens"])
    with pytest.raises(ValueError, match=r"\(3, 1\) int64 first"):
        speculative_generate(tgt, dft, torch.zeros(3, 2, dtype=torch.long), 4)
    assert tgt._graphs.calls == [] and dft._graphs.calls == []
