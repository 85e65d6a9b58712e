"""CPU checks of the device beam search (pcv_beam_step, pcv_kv_gather_rows) and GraphedDecoder.beam_search's host logic.

The numpy oracle (oracle/beam_oracle.py) against 🤗's own ``GenerationMixin._beam_search``, driven by a toy model whose
logits are a seeded function of the sequence; every refusal of the C ABI before any CUDA call; the header layout; the
ptxas log; and beam_search's argument checks, which come before any CUDA work."""
import ctypes
import os
import types
from unittest import mock

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import beam_oracle as O
from perceiver_io_b200 import _lib

transformers = pytest.importorskip("transformers")
from transformers import GenerationMixin, PretrainedConfig, PreTrainedModel  # noqa: E402
from transformers.generation.configuration_utils import GenerationConfig, GenerationMode  # noqa: E402
from transformers.modeling_outputs import CausalLMOutput  # noqa: E402

PROMPT = 3


def _logits_of(seq, V: int, seed: int) -> np.ndarray:
    h = seed
    for t in seq:
        h = (h * 1000003 + int(t) + 1) % (2 ** 61 - 1)
    return (np.random.default_rng(h).standard_normal(V) * 3.0).astype(np.float32)


class _Cfg(PretrainedConfig):
    model_type = "pcv_toy_beam"

    def __init__(self, vocab_size=50, **kw):
        super().__init__(**kw)
        self.vocab_size = vocab_size


class _Toy(PreTrainedModel, GenerationMixin):
    """Logits a seeded function of the whole sequence, at every position."""
    config_class = _Cfg

    def __init__(self, cfg, seed):
        super().__init__(cfg)
        self.dummy = torch.nn.Parameter(torch.zeros(1))
        self.seed = seed

    def prepare_inputs_for_generation(self, input_ids, **kw):
        return {"input_ids": input_ids}

    def forward(self, input_ids, **kw):
        V = self.config.vocab_size
        rows = torch.stack([torch.from_numpy(_logits_of(r.tolist(), V, self.seed)) for r in input_ids])
        return CausalLMOutput(logits=rows[:, None].expand(-1, input_ids.shape[1], -1))


_greedy_mode = GenerationConfig.get_generation_mode


def _beam_mode(self, *a, **kw):   # num_beams=1 routes to greedy search in 🤗; K = 1 beam search is what we compare
    mode = _greedy_mode(self, *a, **kw)
    return GenerationMode.BEAM_SEARCH if mode == GenerationMode.GREEDY_SEARCH else mode


def _compare(K, V, n, eos, lp, es, R, pad, seed, B=2):
    model = _Toy(_Cfg(vocab_size=V), seed).eval()
    ids = torch.randint(0, V, (B, PROMPT), generator=torch.Generator().manual_seed(seed))
    with mock.patch.object(GenerationConfig, "get_generation_mode", _beam_mode):
        out = model.generate(ids, num_beams=K, max_new_tokens=n, do_sample=False, length_penalty=lp,
                             early_stopping=es, num_return_sequences=R, output_scores=True,
                             return_dict_in_generate=True, use_cache=False, pad_token_id=pad,
                             eos_token_id=list(eos) if eos else None)

    def logits_fn(rows):
        return np.stack([_logits_of(ids[i // K].tolist() + r, V, seed) for i, r in enumerate(rows)])

    seqs, scores, flagged, _ = O.beam_search(logits_fn, B, K, n, eos, lp, es, R, pad, tie_tol=1e-6)
    hf = out.sequences[:, PROMPT:].numpy().reshape(B, R, -1)
    want = np.full((B, R, n), O.fill_value(eos, pad), np.int64)
    want[:, :, :hf.shape[2]] = hf
    return flagged, want, seqs, out.sequences_scores.numpy().reshape(B, R), scores


EOS_CASES = [((), 1.0, False), ((1,), 1.0, False), ((1, 2, 3), 2.0, True), ((1,), -0.5, "never"),
             ((1, 2), 0.0, False), ((2,), 2.0, "never"), ((3, 0), 1.0, True), ((1,), 0.0, "never"),
             ((1,), 0.6, False), ((2,), 0.6, "never"), ((1, 3), -0.3, True), ((), 1.2, "never")]


@pytest.mark.parametrize("K", [1, 2, 3, 8])
@pytest.mark.parametrize("V", ["2K", 389, 32000])
def test_oracle_equals_hf_beam_search(K, V):
    V = 2 * K if V == "2K" else V
    checked = flagged_n = 0
    for i, (eos, lp, es) in enumerate(EOS_CASES):
        eos = tuple(e for e in eos if e < V)
        if K * V < O.MAX_EOS and len(eos) > 1:
            continue
        if K * V < max(2, len(eos) + 1) * K:
            continue
        n = 4 if V == 32000 else 7
        for R in sorted({1, K}):
            for pad in (None, 0):
                if V == 32000 and (pad is None or R != K):
                    continue   # the toy model's full-vocabulary rows are slow on the CPU: one variant each
                flagged, want, got, hf_scores, scores = _compare(K, V, n, eos, lp, es, R, pad, seed=K * 1000 + V + i)
                if flagged:
                    flagged_n += 1
                    continue
                assert np.array_equal(got, want), (eos, lp, es, R, pad, got, want)
                np.testing.assert_allclose(scores, hf_scores, rtol=1e-5, atol=1e-4)
                checked += 1
    assert checked >= max(4, 2 * flagged_n), (checked, flagged_n)


def test_an_eos_that_fires_mid_run_finishes_hypotheses_early():
    """A hypothesis that ends mid-run is padded with the fill value, and an item whose heuristic is satisfied stops."""
    found = False
    for seed in range(40):
        flagged, want, got, _, _ = _compare(3, 12, 8, (2,), 1.0, False, 3, 0, seed)
        if flagged:
            continue
        assert np.array_equal(got, want)
        ends = (got == 2).argmax(-1)
        if ((got == 2).any(-1) & (ends < 6)).any():
            found = True
            break
    assert found


def test_stopping_early_gives_the_same_output():
    V, K, B = 16, 3, 2
    for seed in range(12):
        def fn(rows):
            return np.stack([_logits_of([b] + r, V, seed) for b, r in zip(np.repeat(np.arange(B), K), rows)])
        a = O.beam_search(fn, B, K, 12, (1, 4), 1.0, True, 3, None, stop_early=True)
        b = O.beam_search(fn, B, K, 12, (1, 4), 1.0, True, 3, None, stop_early=False)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_tie_rule_lowest_flat_index_wins():
    st = O.init_state(1, 2, 3, 4, -1)
    logits = np.array([[1, 5, 5, 0], [1, 5, 5, 0]], np.float32)
    tok, par, fl = O.step(st, logits)
    assert tok.tolist() == [1, 2] and par.tolist() == [0, 0] and not fl.any()
    tok, par, _ = O.step(st, np.array([[0, 3, 3, 0], [3, 0, 0, 3]], np.float32))
    # beam 0 (score s) and beam 1 (score s, its second token) tie: beam 0's first token, then beam 0's token 2
    assert tok.tolist() == [1, 2] and par.tolist() == [0, 0]


# ---- the C ABI --------------------------------------------------------------------------------------------------------
def _params(**kw):
    p = _lib.BeamStepParams()
    p.logits, p.stride_row, p.B, p.K, p.V, p.dtype = 0x1000, 400, 2, 3, 389, _lib.PCV_BF16
    p.n_eos, p.eos[0], p.eos[1] = 2, 7, 9
    p.length_penalty, p.early_stopping, p.hist_len = 1.0, 0, 17
    base = 0x10000000
    for i, f in enumerate(("running_scores", "finished_scores", "finished_flags", "running_hist", "finished_hist",
                           "hist_scratch", "item_flags", "counters", "cand_scores", "cand_index", "next_tokens",
                           "parents")):
        setattr(p, f, base + i * 0x100000)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


BEAM_REFUSALS = [
    (dict(logits=None), b"pointer is NULL"),
    (dict(counters=None), b"pointer is NULL"),
    (dict(parents=None), b"pointer is NULL"),
    (dict(V=0), b"V=0 must be in [1, 32768]"),
    (dict(V=32769, stride_row=40000), b"V=32769 must be in [1, 32768]"),
    (dict(K=0), b"K=0 must be in [1, 8]"),
    (dict(K=9), b"K=9 must be in [1, 8]"),
    (dict(B=0), b"B=0 must be >= 1"),
    (dict(n_eos=5), b"n_eos=5 must be in [0, 4]"),
    (dict(V=2, stride_row=2, n_eos=0, K=1), None),   # K*V = 2 = beams_to_keep: taken
    (dict(V=2, stride_row=2, eos=(ctypes.c_int32 * 4)(0, 1, 0, 0), K=1), b"K*V=2 is below beams_to_keep=3"),
    (dict(eos=(ctypes.c_int32 * 4)(7, 389, 0, 0)), b"EOS id 389 is outside [0, V=389)"),
    (dict(eos=(ctypes.c_int32 * 4)(-1, 3, 0, 0)), b"EOS id -1 is outside"),
    (dict(stride_row=388), b"stride_row=388 is below V=389"),
    (dict(length_penalty=float("inf")), b"length_penalty must be finite"),
    (dict(length_penalty=float("nan")), b"length_penalty must be finite"),
    (dict(early_stopping=3), b"unknown early_stopping code 3"),
    (dict(dtype=_lib.PCV_E4M3), b"unknown dtype 3"),
    (dict(hist_len=0), b"hist_len=0 must be >= 1"),
    (dict(parents=0x10000000 + 10 * 0x100000), b"output buffers 10 and 11 overlap"),
    (dict(finished_scores=0x10000000 + 4), b"output buffers 0 and 1 overlap"),
]


@pytest.mark.parametrize("kw,reason", BEAM_REFUSALS, ids=[f"refuse{i}" for i in range(len(BEAM_REFUSALS))])
def test_beam_step_refusals_come_before_any_cuda_call(kw, reason):
    lib = _lib.lib()
    p = _params(**kw)
    if reason is None:
        assert lib.pcv_beam_step_supported(ctypes.byref(p)) == 1, lib.pcv_last_error()
        return
    assert lib.pcv_beam_step_supported(ctypes.byref(p)) == 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()
    assert lib.pcv_beam_step(ctypes.byref(p), None) != 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()


def test_beam_step_accepts_the_edges():
    lib = _lib.lib()
    for kw in (dict(), dict(K=8), dict(K=1, n_eos=0), dict(V=32768, stride_row=32768), dict(dtype=_lib.PCV_F32),
               dict(dtype=_lib.PCV_F16), dict(early_stopping=2), dict(length_penalty=-0.5),
               dict(n_eos=4, eos=(ctypes.c_int32 * 4)(0, 1, 2, 388))):
        assert lib.pcv_beam_step_supported(ctypes.byref(_params(**kw))) == 1, (kw, lib.pcv_last_error())
    assert lib.pcv_beam_step_supported(None) == 0 and b"params is NULL" in lib.pcv_last_error()
    assert lib.pcv_beam_step(None, None) != 0


def test_kv_gather_refusals_come_before_any_cuda_call():
    lib = _lib.lib()
    rows = _lib.DevRows(bounds=0x3000, capacity=12, bounds_stride_b=12)
    ok = dict(table=0x1000, n_entries=57, R=24, parents=0x2000)
    assert lib.pcv_kv_gather_rows_supported(ctypes.byref(_lib.KvGatherParams(**ok)), ctypes.byref(rows)) == 1
    for kw, reason in ((dict(table=None), b"pointer is NULL"), (dict(parents=None), b"pointer is NULL"),
                       (dict(n_entries=0), b"n_entries=0"), (dict(R=0), b"R=0"), (dict(R=70000), b"R=70000")):
        p = _lib.KvGatherParams(**{**ok, **kw})
        assert lib.pcv_kv_gather_rows_supported(ctypes.byref(p), ctypes.byref(rows)) == 0
        assert reason in lib.pcv_last_error()
        assert lib.pcv_kv_gather_rows(ctypes.byref(p), ctypes.byref(rows), None) != 0
    bad = _lib.DevRows(bounds=0x3000, capacity=12, bounds_stride_b=-1)
    assert lib.pcv_kv_gather_rows(ctypes.byref(_lib.KvGatherParams(**ok)), ctypes.byref(bad), None) != 0
    assert b"negative" in lib.pcv_last_error()
    assert lib.pcv_kv_gather_rows(None, ctypes.byref(rows), None) != 0


def _layout(tmp_path, name, cls):
    import subprocess

    header = os.path.join(ROOT, "include", "pcv_attn.h")
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void){",
             f'printf("size %zu\\n", sizeof({name}));']
    lines += [f'printf("{f} %zu\\n", offsetof({name}, {f}));' for f, _ in cls._fields_]
    lines.append("return 0;}")
    (tmp_path / f"{name}.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-o", str(tmp_path / name), str(tmp_path / f"{name}.c")])
    got = dict(l.split() for l in subprocess.check_output([str(tmp_path / name)]).decode().split("\n") if l)
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def test_the_length_penalty_travels_in_fp64():
    """🤗 raises the length to the Python (fp64) penalty: an fp32 field would round 0.6 first and move fp32(g ** lp)."""
    p = _params(length_penalty=0.6)
    assert p.length_penalty == 0.6
    moved = sum(O.divisor(g, 0.6)[0] != np.float32(float(g) ** float(np.float32(0.6))) for g in range(1, 257))
    assert moved > 100   # what an fp32 field would get wrong


def test_params_layout_matches_the_header(tmp_path):
    _layout(tmp_path, "pcv_beam_step_params", _lib.BeamStepParams)
    _layout(tmp_path, "pcv_kv_gather_entry", _lib.KvGatherEntry)
    _layout(tmp_path, "pcv_kv_gather_params", _lib.KvGatherParams)
    assert (_lib.BEAM_MAX_BEAMS, _lib.BEAM_MAX_EOS) == (O.MAX_BEAMS, O.MAX_EOS) == (8, 4)


def test_build_has_no_spills():
    log = os.path.join(ROOT, "build", "pcv_beam.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was not built in this tree")
    text = open(log).read()
    entries = text.split("Compiling entry function")[1:]
    names = ("beam_rows_kernel", "beam_item_kernel", "kv_gather_kernel")
    kernels = [e for e in entries if any(k in e.split("\n")[0] for k in names)]
    assert len(kernels) == 5, len(kernels)
    for e in kernels:
        own = next(line for line in e.split("\n") if "spill" in line)   # the kernel's own line, not a callee's
        assert "0 bytes spill stores, 0 bytes spill loads" in own, e[:300]
        regs = int(e.split("Used ")[1].split(" registers")[0])
        assert regs <= 64, e[:300]   # 512-thread CTAs: at most 128 registers, and these stay well below
    assert "C7515" not in text and "C7512" not in text


# ---- GraphedDecoder.beam_search: argument checks -----------------------------------------------------------------------
def _decoder(batch=6, T=20, vocab=97):
    from perceiver_io_b200.generation import GraphedDecoder

    dec = GraphedDecoder.__new__(GraphedDecoder)
    dec.batch, dec.max_new_tokens, dec.device = batch, T, torch.device("cpu")
    dec.model = types.SimpleNamespace(config=types.SimpleNamespace(vocab_size=vocab))
    dec.prefill = mock.Mock(side_effect=AssertionError("prefill ran"))
    return dec


BAD_ARGS = [
    (dict(num_beams=2), ValueError, "batch 6 must be batch \\* num_beams = 2 \\* 2"),
    (dict(num_beams=9), ValueError, "num_beams must be an integer in \\[1, 8\\]"),
    (dict(num_beams=0), ValueError, "num_beams"),
    (dict(n=0), ValueError, "n must be an integer in \\[1, max_new_tokens \\+ 1 = 21\\]"),
    (dict(n=22), ValueError, "n must be an integer"),
    (dict(n=2.0), ValueError, "n must be an integer"),
    (dict(num_return_sequences=4), ValueError, "num_return_sequences must be an integer in \\[1, num_beams=3\\]"),
    (dict(num_return_sequences=0), ValueError, "num_return_sequences"),
    (dict(check_every=0), ValueError, "check_every"),
    (dict(eos_token_id=97), ValueError, "each in \\[0, 97\\)"),
    (dict(eos_token_id=[1, 2, 3, 4, 5]), ValueError, "at most 4 EOS ids"),
    (dict(eos_token_id="x"), ValueError, "eos_token_id must be"),
    (dict(length_penalty=float("inf")), ValueError, "length_penalty must be finite"),
    (dict(early_stopping="always"), ValueError, "early_stopping must be False, True or 'never'"),
    (dict(early_stopping=1), ValueError, "early_stopping must be False, True or 'never'"),
    (dict(early_stopping="True"), ValueError, "early_stopping must be False, True or 'never'"),
    (dict(early_stopping="False"), ValueError, "early_stopping must be False, True or 'never'"),
]


@pytest.mark.parametrize("kw,exc,match", BAD_ARGS, ids=[f"bad{i}" for i in range(len(BAD_ARGS))])
def test_beam_search_refusals_come_before_any_work(kw, exc, match):
    dec = _decoder()
    args = dict(n=5, num_beams=3)
    args.update(kw)
    with pytest.raises(exc, match=match):
        dec.beam_search(torch.zeros(2, 4, dtype=torch.long), 0, **args)
    dec.prefill.assert_not_called()


def test_beam_search_refuses_a_vocabulary_above_the_limit_and_too_few_candidates():
    with pytest.raises(RuntimeError, match="vocabularies up to 32768, this model has 32769"):
        _decoder(vocab=32769).beam_search(torch.zeros(2, 4, dtype=torch.long), 0, 5, num_beams=3)
    with pytest.raises(ValueError, match="num_beams \\* vocab = 3 is below the 6 candidates"):
        _decoder(batch=3, vocab=1).beam_search(torch.zeros(1, 4, dtype=torch.long), 0, 5, num_beams=3)
