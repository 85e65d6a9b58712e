"""CPU checks of the device token sampler (pcv_sample) and GraphedDecoder's sampling host logic.

The numpy oracle (oracle/sample_oracle.py) against 🤗's TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper
on random fp32 logits; the tie rules on integer logits; the statistics of the counter-based random bits; every refusal
of the C ABI before any CUDA call; the ptxas log; and the decoder's argument checks and draw positions, which must be
the rows the one-token loop feeds, after per-row rewinds and a beam reorder."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import sample_oracle as S
from perceiver_io_b200 import _lib

VOCABS = [1, 2, 262, 389, 32000]


def _hf_probs(logits: np.ndarray, temperature: float, top_k: int, top_p: float) -> np.ndarray:
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper

    scores = torch.from_numpy(logits.astype(np.float32))[None]
    ids = torch.zeros(1, 1, dtype=torch.long)
    warpers = [TemperatureLogitsWarper(temperature)]
    if top_k > 0:
        warpers.append(TopKLogitsWarper(top_k))
    if top_p < 1.0:
        warpers.append(TopPLogitsWarper(top_p))
    for w in warpers:
        scores = w(ids, scores)
    return torch.softmax(scores, dim=-1)[0].double().numpy()


def _random_logits(V: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(V) * 2.5).astype(np.float32)   # continuous: no ties at any cut


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("temperature", [0.7, 1.0, 1.3])
def test_oracle_equals_the_hf_warpers(V, temperature):
    logits = _random_logits(V, V + int(temperature * 10))
    assert S.greedy_token(logits, temperature) is None   # 🤗 raises on a row with no finite mass: not compared here
    checked = 0
    for top_k in (0, 1, 10, V - 1, V, V + 5):
        for top_p in (1.0, 0.95, 0.5, 1e-3):
            ref = _hf_probs(logits, temperature, top_k, top_p)
            got = S.probs(logits, temperature, top_k, top_p)
            f = S.filter_row(logits, temperature, top_k, top_p)
            if top_p < 1.0:
                # 🤗 sums fp32 probabilities: skip a cut that lies within its rounding of a tie-group boundary
                edge = np.abs(f.W.astype(np.float64) / float(f.W[-1]) - (1.0 - top_p))
                if edge.min() < 1e-5:
                    continue
            assert np.array_equal(f.kept, ref > 0), (top_k, top_p)
            np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-9, err_msg=f"top_k={top_k} top_p={top_p}")
            checked += 1
    assert checked >= 20


def test_tie_rules_on_integer_logits():
    # top-k keeps every token tied with the k-th largest
    logits = np.array([1, 5, 3, 5, 3, 3, 0, 2], dtype=np.float32)
    f = S.filter_row(logits, 1.0, 3, 1.0)
    assert f.kept.tolist() == [False, True, True, True, True, True, False, False]
    assert S.filter_row(logits, 1.0, 2, 1.0).kept.tolist() == [False, True, False, True, False, False, False, False]
    # a tie group straddling the top-p cut is kept whole: the 3s hold 3e^-2 / (2 + 3e^-2) ≈ 0.17 of the mass (with
    # the top two at 5); 1 - top_p = 0.1 falls inside that group, so all three 3s stay
    f = S.filter_row(logits, 1.0, 5, 0.9)
    assert f.kept.tolist() == [False, True, True, True, True, True, False, False]
    # and with 1 - top_p beyond the group, none stays
    assert S.filter_row(logits, 1.0, 5, 0.8).kept.tolist() == [False, True, False, True, False, False, False, False]
    # the top group always stays, whatever top_p
    assert S.filter_row(logits, 1.0, 0, 1e-9).kept.tolist() == [False, True, False, True, False, False, False, False]
    # greedy takes the first maximal index, -0 and +0 tie
    assert S.sample_row(logits, 0.0, 0, 1.0, 1, 0, 0).token == 1
    assert S.sample_row(np.array([-1.0, 0.0, -0.0], dtype=np.float32), 0.0, 0, 1.0, 1, 0, 0).token == 1


def test_draw_is_inverse_cdf_in_index_order():
    """Equal logits among the kept tokens make every mass exactly 2^40: token j is drawn iff t in [j, j+1) * 2^40."""
    logits = np.full(16, -100.0, dtype=np.float32)
    kept = [2, 5, 6, 11]
    logits[kept] = 3.0
    for pos in range(200):
        bits = int(S.uniform_bits(99, 1, pos))
        t = (bits * (4 << 40)) >> 64
        d = S.sample_row(logits, 1.0, 0, 1.0, 99, 1, pos)
        assert d.token == kept[t >> 40] and not d.ambiguous
        assert d.logprob == pytest.approx(np.log(0.25), abs=1e-6)


# ---- the random bits --------------------------------------------------------------------------------------------------
N_HASH = 1 << 20


def _uniform01(bits: np.ndarray) -> np.ndarray:
    return (bits >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def test_hash_is_uniform():
    pos = np.arange(N_HASH, dtype=np.int64)
    for seed, b in ((0, 0), (12345, 3), (2 ** 63 + 7, 1)):
        bits = S.uniform_bits(np.uint64(seed), b, pos)
        for shift in (0, 24, 56):   # low, middle and top bytes
            counts = np.bincount(((bits >> np.uint64(shift)) & np.uint64(255)).astype(np.int64), minlength=256)
            chi2 = ((counts - N_HASH / 256) ** 2 / (N_HASH / 256)).sum()
            assert chi2 < 255 + 6 * np.sqrt(2 * 255), (seed, b, shift, chi2)   # 6 sigma of chi2(255)
        u = _uniform01(bits)
        assert abs(u.mean() - 0.5) < 6 * np.sqrt(1 / 12 / N_HASH)
        assert len(np.unique(bits)) == N_HASH


def test_hash_is_independent_across_seeds_rows_positions_and_halves():
    pos = np.arange(N_HASH, dtype=np.int64)
    floor = 6 / np.sqrt(N_HASH)   # 6 sigma of a correlation of independent uniforms
    base = _uniform01(S.uniform_bits(np.uint64(1000), 2, pos))
    others = {
        "adjacent seed": S.uniform_bits(np.uint64(1001), 2, pos),
        "adjacent high seed word": S.uniform_bits(np.uint64(1000 + (1 << 32)), 2, pos),
        "adjacent batch row": S.uniform_bits(np.uint64(1000), 3, pos),
        "adjacent position": S.uniform_bits(np.uint64(1000), 2, pos + 1),
    }
    for what, bits in others.items():
        c = np.corrcoef(base, _uniform01(bits))[0, 1]
        assert abs(c) < floor, (what, c)
        agree = np.mean((S.uniform_bits(np.uint64(1000), 2, pos) >> np.uint64(63)) == (bits >> np.uint64(63)))
        assert abs(agree - 0.5) < 6 * 0.5 / np.sqrt(N_HASH), (what, agree)
    bits = S.uniform_bits(np.uint64(1000), 2, pos)
    lo = (bits & np.uint64(0xFFFFFFFF)).astype(np.float64)
    hi = (bits >> np.uint64(32)).astype(np.float64)
    assert abs(np.corrcoef(lo, hi)[0, 1]) < floor
    for lag in (1, 2, 64, 1024):
        assert abs(np.corrcoef(base[:-lag], base[lag:])[0, 1]) < floor, lag


# ---- the C ABI --------------------------------------------------------------------------------------------------------
def _params(**kw):
    p = _lib.SampleParams()
    p.logits, p.stride_row, p.R, p.V, p.dtype, p.rows_per_batch = 0x1000, 400, 6, 389, _lib.PCV_BF16, 3
    p.seeds, p.positions, p.tokens, p.logprobs = 0x2000, 0x3000, 0x4000, None
    p.temperature, p.top_k, p.top_p = 1.0, 10, 0.9
    for k, v in kw.items():
        setattr(p, k, v)
    return p


REFUSALS = [
    (dict(logits=None), b"pointer is NULL"),
    (dict(seeds=None), b"pointer is NULL"),
    (dict(positions=None), b"pointer is NULL"),
    (dict(tokens=None), b"pointer is NULL"),
    (dict(V=0), b"V=0 must be in [1, 32768]"),
    (dict(V=32769, stride_row=40000), b"V=32769 must be in [1, 32768]"),
    (dict(stride_row=388), b"stride_row=388 is below V=389"),
    (dict(R=7), b"R=7 is not a multiple of rows_per_batch=3"),
    (dict(rows_per_batch=0), b"not a multiple of rows_per_batch=0"),
    (dict(R=0), b"R=0 must be >= 1"),
    (dict(temperature=-0.5), b"temperature must be >= 0"),
    (dict(temperature=float("nan")), b"temperature must be >= 0"),
    (dict(top_k=-1), b"top_k must be >= 0"),
    (dict(top_p=0.0), b"top_p must be in (0, 1]"),
    (dict(top_p=1.5), b"top_p must be in (0, 1]"),
    (dict(top_p=float("nan")), b"top_p must be in (0, 1]"),
    (dict(dtype=_lib.PCV_E4M3), b"unknown dtype 3"),
    (dict(dtype=9), b"unknown dtype 9"),
]


@pytest.mark.parametrize("kw,reason", REFUSALS, ids=[f"refuse{i}" for i in range(len(REFUSALS))])
def test_abi_refusals_come_before_any_cuda_call(kw, reason):
    lib = _lib.lib()
    p = _params(**kw)
    assert lib.pcv_sample_supported(ctypes.byref(p)) == 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()
    assert lib.pcv_sample(ctypes.byref(p), None) != 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()


def test_abi_accepts_the_edges_and_refuses_null():
    lib = _lib.lib()
    for kw in (dict(), dict(V=1, stride_row=1), dict(V=32768, stride_row=32768), dict(temperature=0.0),
               dict(top_k=0, top_p=1.0), dict(top_k=2 ** 31 - 1), dict(dtype=_lib.PCV_F32), dict(dtype=_lib.PCV_F16)):
        assert lib.pcv_sample_supported(ctypes.byref(_params(**kw))) == 1, (kw, lib.pcv_last_error())
    assert lib.pcv_sample_supported(None) == 0 and b"params is NULL" in lib.pcv_last_error()
    assert lib.pcv_sample(None, None) != 0 and b"params is NULL" in lib.pcv_last_error()
    assert lib.pcv_sample_uniforms(None, 0x10, 0x20, 4, 1, None) != 0 and b"NULL" in lib.pcv_last_error()
    assert lib.pcv_sample_uniforms(0x30, 0x10, 0x20, 5, 2, None) != 0
    assert b"multiple of rows_per_batch=2" in lib.pcv_last_error()


def test_sample_params_layout_matches_the_header(tmp_path):
    import subprocess

    header = os.path.join(ROOT, "include", "pcv_attn.h")
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void){",
             'printf("size %zu\\n", sizeof(pcv_sample_params));']
    lines += [f'printf("{f} %zu\\n", offsetof(pcv_sample_params, {f}));' for f, _ in _lib.SampleParams._fields_]
    lines.append("return 0;}")
    (tmp_path / "l.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-o", str(tmp_path / "l"), str(tmp_path / "l.c")])
    got = dict(l.split() for l in subprocess.check_output([str(tmp_path / "l")]).decode().split("\n") if l)
    assert int(got["size"]) == ctypes.sizeof(_lib.SampleParams)
    for f, _ in _lib.SampleParams._fields_:
        assert int(got[f]) == getattr(_lib.SampleParams, f).offset, f
    assert _lib.SAMPLE_MAX_VOCAB == S.MAX_VOCAB == 32768


def test_build_has_no_spills():
    log = os.path.join(ROOT, "build", "pcv_sample.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was not built in this tree")
    text = open(log).read()
    entries = text.split("Compiling entry function")[1:]
    kernels = [e for e in entries if "sample_kernel" in e.split("\n")[0] or "sample_uniforms_kernel" in e.split("\n")[0]]
    assert len(kernels) == 4, len(kernels)
    for e in kernels:
        assert "0 bytes spill stores, 0 bytes spill loads" in e, e[:300]
    assert "C7515" not in text and "C7512" not in text


# ---- GraphedDecoder: sampling host logic ------------------------------------------------------------------------------
class _Graphs(dict):
    """Stands in for the recorded graphs: a replay moves the bounds as _step_fn does and records the positions a
    sampling replay draws at."""

    def __init__(self, dec):
        super().__init__()
        self.dec, self.positions = dec, []

    def get(self, key):
        from perceiver_io_b200.generation import advance_bounds_, sample_positions

        k = key[1] if isinstance(key, tuple) else key

        def replay(tokens):
            d = self.dec
            if isinstance(key, tuple):
                self.positions.append(sample_positions(d._bounds, d._steps, k))
            advance_bounds_(d._bounds, d._inc, d._wmax, k)
            out = torch.zeros(d.batch, k, dtype=torch.long)
            return (out, torch.zeros(d.batch, k, 1)) if isinstance(key, tuple) else out

        return replay


def _decoder(B=3, n0=30, prefix=10, max_seq_len=40, max_latents=16, T=40, vocab=97):
    from test_window_rows_cpu import _decoder as rows_decoder

    dec = rows_decoder(B, n0, prefix, max_seq_len, max_latents, T)
    dec._graphs = _Graphs(dec)
    dec._seeds, dec._seeded, dec._sampling = torch.zeros(B, dtype=torch.int64), False, (1.0, 0, 1.0)
    dec._steps = torch.arange(1, 65, dtype=torch.int32)
    dec.model = types.SimpleNamespace(config=types.SimpleNamespace(vocab_size=vocab))
    return dec


BAD_SAMPLING = [
    (dict(temperature=-1.0), "temperature"), (dict(temperature=float("nan")), "temperature"),
    (dict(temperature=float("inf")), "temperature"), (dict(top_k=-1), "top_k"), (dict(top_k=2.5), "top_k"),
    (dict(top_k=True), "top_k"), (dict(top_p=0.0), "top_p"), (dict(top_p=1.01), "top_p"),
    (dict(top_p=float("nan")), "top_p"),
]


@pytest.mark.parametrize("kw,match", BAD_SAMPLING, ids=[f"bad{i}" for i in range(len(BAD_SAMPLING))])
def test_set_sampling_refusals_leave_the_values(kw, match):
    dec = _decoder()
    dec.set_sampling(0.8, 10, 0.9)
    with pytest.raises(ValueError, match=match):
        dec.set_sampling(**kw)
    assert dec._sampling == (0.8, 10, 0.9)
    dec.set_sampling(temperature=0)
    assert dec._sampling == (0.0, 0, 1.0)


def test_set_seed_takes_one_or_b_integers():
    dec = _decoder()
    dec.set_seed(7)
    assert dec._seeds.tolist() == [7, 7, 7] and dec._seeded
    dec.set_seed([1, 2 ** 64 - 1, 2 ** 63])
    assert dec._seeds.tolist() == [1, -1, -2 ** 63]
    dec.set_seed(torch.tensor([4, 5, 6]))
    assert dec._seeds.tolist() == [4, 5, 6]
    for bad, match in (([1, 2], "3 integers"), ("x", "3 integers"), ([1, -1, 0], "batch row 1"),
                       ([0, 0, 2 ** 64], "batch row 2"), ([0, 1.0, 0], "batch row 1"), (1.5, "3 integers")):
        with pytest.raises(ValueError, match=match):
            dec.set_seed(bad)
        assert dec._seeds.tolist() == [4, 5, 6]


def test_an_unseeded_decoder_draws_its_seed_from_torchs_generator():
    from perceiver_io_b200 import ops

    a, b = _decoder(), _decoder()
    torch.manual_seed(5)
    a.generate(torch.zeros(3, 1, dtype=torch.long), 2)
    torch.manual_seed(5)
    want = ops.new_dropout_seed()
    torch.manual_seed(5)
    b.sample(torch.zeros(3, 4, dtype=torch.long))
    assert a._seeds.tolist() == [want] * 3 == b._seeds.tolist()


def test_generate_refusals_leave_the_state_untouched():
    dec = _decoder(T=10)
    dec.set_seed(1)
    dec.generate(torch.zeros(3, 1, dtype=torch.long), 6)
    before = (dec._bounds.clone(), dec._fed, dec._remaining, len(dec._graphs.positions))
    for n, exc, match in ((5, RuntimeError, "4 of max_new_tokens=10 tokens remain to the furthest batch row, 5 asked"),
                          (0, ValueError, "n must be an integer >= 1"), (2.0, ValueError, "n must be an integer"),
                          (True, ValueError, "n must be an integer")):
        with pytest.raises(exc, match=match):
            dec.generate(torch.zeros(3, 1, dtype=torch.long), n)
    with pytest.raises(ValueError, match=r"\(3, 1\) int64 first tokens"):
        dec.generate(torch.zeros(3, 2, dtype=torch.long), 2)
    assert torch.equal(dec._bounds, before[0]) and (dec._fed, dec._remaining, len(dec._graphs.positions)) == before[1:]
    dec.generate(torch.zeros(3, 1, dtype=torch.long), 4)
    assert dec._remaining == 0


def test_a_vocabulary_above_the_limit_is_refused():
    dec = _decoder(vocab=32769)
    for call in (lambda: dec.draw(torch.zeros(3, 32769)), lambda: dec.sample(torch.zeros(3, 1, dtype=torch.long)),
                 lambda: dec.generate(torch.zeros(3, 1, dtype=torch.long), 1)):
        with pytest.raises(RuntimeError, match="vocabularies up to 32768, this model has 32769"):
            call()
    assert dec._fed == 0


def test_draw_positions_are_the_rows_of_the_one_token_loop():
    """Every draw's position is the cross-attention row its token would be fed at: after prefill n0 + fed[b] + 1 for
    the token after fed token fed[b], through samples, generates, per-row rewinds and a reorder."""
    B, n0 = 3, 30
    dec = _decoder(B=B, n0=n0, T=60)
    dec.set_seed(3)
    fed = [0] * B
    dec.set_sampling(0.9, 5, 0.8)

    def expect(k):
        got = dec._graphs.positions[-1]
        assert got.dtype == torch.int32
        assert got.tolist() == [[n0 + f + 1 + i for i in range(k)] for f in fed]

    for op in (("s", 4), ("r", [1, 3, 0]), ("g", 3), ("s", 1), ("r", [0, 2, 4]), ("o", [2, 0, 0]), ("s", 7),
               ("r", 2), ("g", 2), ("s", 16)):
        if op[0] == "s":
            dec.sample(torch.zeros(B, op[1], dtype=torch.long))
            expect(op[1])
            fed = [f + op[1] for f in fed]
        elif op[0] == "g":
            n0_pos = len(dec._graphs.positions)
            dec.generate(torch.zeros(B, 1, dtype=torch.long), op[1])
            got = dec._graphs.positions[n0_pos:]
            assert [p.tolist() for p in got] == [[[n0 + f + 1 + i] for f in fed] for i in range(op[1])]
            fed = [f + op[1] for f in fed]
        elif op[0] == "r":
            counts = op[1] if isinstance(op[1], list) else [op[1]] * B
            dec.rewind(op[1])
            fed = [f - c for f, c in zip(fed, counts)]
        else:
            dec.reorder(torch.tensor(op[1]))
            fed = [fed[i] for i in op[1]]
        # draw: the position of the row the next token is fed at
        assert (dec._bounds[:, 0, 2]).tolist() == [n0 + f for f in fed]


def test_reorder_moves_the_seeds_with_their_rows():
    dec = _decoder()
    dec.set_seed([10, 20, 30])
    dec.reorder(torch.tensor([2, 2, 0]))
    assert dec._seeds.tolist() == [30, 30, 10]
