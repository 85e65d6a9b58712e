"""CPU checks of the logits processors (pcv_logits_process) and their wiring: the numpy oracle against 🤗's own
RepetitionPenaltyLogitsProcessor -> NoRepeatNGramLogitsProcessor -> MinNewTokensLengthLogitsProcessor, bit for bit on
fp32 rows, in the logits and the log-softmax mode; an oracle greedy loop against 🤗 ``generate()`` on a fake model;
every refusal of the C ABI before any CUDA call; the header layout; and the argument checks of ``set_sampling``,
``generate``, ``verify``, ``beam_search`` and ``contrastive_search``, which come before any CUDA work."""
import ctypes
import os
import types
from unittest import mock

import numpy as np
import pytest
import torch

import process_oracle as P
from conftest import ROOT
from oracle import beam_oracle
from perceiver_io_b200 import _lib

transformers = pytest.importorskip("transformers")
from transformers.generation import logits_process as LP  # noqa: E402


def _hf(ids, scores, theta, N, M, n0, eos):
    """🤗's processors, chained in _get_logits_processor's order."""
    procs = []
    if theta != 1.0:
        procs.append(LP.RepetitionPenaltyLogitsProcessor(penalty=float(theta)))
    if N > 0:
        procs.append(LP.NoRepeatNGramLogitsProcessor(N))
    if M > 0:
        procs.append(LP.MinNewTokensLengthLogitsProcessor(n0, M, eos, device="cpu"))
    return LP.LogitsProcessorList(procs)(ids, scores)


CASES = [(theta, N, M) for theta in (1.0, 1.2, 0.7, 3.0) for N in (0, 1, 2, 3, 5) for M in (0, 3)]


@pytest.mark.parametrize("log_softmax", [False, True])
@pytest.mark.parametrize("theta,N,M", CASES)
def test_oracle_equals_hf_processors(theta, N, M, log_softmax):
    rng = np.random.default_rng(int(theta * 10) * 100 + N * 10 + M)
    V, n0 = 61, 5
    for L in (0, 1, N - 1, N, N + 1, 4, 6, 7, 9, 24):
        if L < 1:   # 🤗 needs one id at least
            continue
        B = 3
        # small ids: duplicates and repeated n-grams; id 0 doubles as a pad id of the prompt
        ids = rng.integers(0, 4 if L > 6 else V, size=(B, L))
        ids[0, :2] = 0
        x = (rng.standard_normal((B, V)) * 4).astype(np.float32)
        x[1, :8] = -np.abs(x[1, :8])
        if log_softmax:
            x = np.stack([beam_oracle.log_softmax(r)[0] for r in x])
        eos = [7, 11]
        want = _hf(torch.from_numpy(ids), torch.from_numpy(x.copy()), theta, N, M, n0, eos).numpy()
        got = P.process_rows(x, ids, repetition_penalty=theta, no_repeat_ngram_size=N, min_new_tokens=M,
                             prompt_len=n0, eos=eos)
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg=f"L={L}")


def test_penalty_rounding_is_one_fp32_operation():
    """x * θ and x / θ as torch rounds them: one correctly rounded fp32 operation with fp32(θ)."""
    rng = np.random.default_rng(0)
    V = 4096
    x = (rng.standard_normal((1, V)) * 100).astype(np.float32)
    ids = torch.arange(V)[None]
    for theta in (1.1, 1.3, 0.9, 2.0 / 3.0, 1.7):
        want = LP.RepetitionPenaltyLogitsProcessor(theta)(ids, torch.from_numpy(x.copy())).numpy()[0]
        t32 = np.float32(theta)
        mine = np.where(x[0] < 0, x[0] * t32, x[0] / t32).astype(np.float32)
        np.testing.assert_array_equal(mine.view(np.uint32), want.view(np.uint32))
        np.testing.assert_array_equal(P.process(x[0], np.arange(V), repetition_penalty=theta).view(np.uint32),
                                      want.view(np.uint32))


def test_out_of_range_ids_match_but_are_never_written():
    x = np.zeros(8, np.float32)
    hist = [-1, 3, -1, 3, 9, -1]   # the n-gram (-1, 3) occurred; the suffix is (-1,)
    got = P.process(x, hist, no_repeat_ngram_size=2)
    assert np.isneginf(got[3]) and np.isfinite(np.delete(got, 3)).all()
    got = P.process(x, [1, 9, 1], no_repeat_ngram_size=2)   # bans 9, outside V: nothing is written
    assert np.isfinite(got).all()
    got = P.process(x + 1, [9, -1, 2, 2], repetition_penalty=2.0)
    assert got[2] == 0.5 and (np.delete(got, 2) == 1).all()


# ---- 🤗 generate() on a fake model against the oracle loops ----------------------------------------------------------
class _Cfg(transformers.PretrainedConfig):
    model_type = "pcv_toy_process"

    def __init__(self, vocab_size=17, **kw):
        super().__init__(**kw)
        self.vocab_size = vocab_size


class _Fake(transformers.PreTrainedModel, transformers.GenerationMixin):
    """Logits a fixed function of the last two ids, at every position."""
    config_class = _Cfg

    def __init__(self, V):
        super().__init__(_Cfg(vocab_size=V))
        self.dummy = torch.nn.Parameter(torch.zeros(1))
        g = torch.Generator().manual_seed(3)
        self.T = torch.randn(V, V, generator=g) * 3
        self.U = torch.randn(V, V, generator=g)

    def prepare_inputs_for_generation(self, input_ids, **kw):
        return {"input_ids": input_ids}

    def forward(self, input_ids, **kw):
        prev = input_ids[:, -2] if input_ids.shape[1] > 1 else input_ids[:, -1]
        logits = self.T[input_ids[:, -1]] + self.U[prev]
        return transformers.modeling_outputs.CausalLMOutput(logits=logits[:, None].expand(-1, input_ids.shape[1], -1))

    def logits(self, ids):
        with torch.no_grad():
            return self.forward(torch.as_tensor(ids)).logits[:, -1].numpy()


def _greedy_oracle(model, ids, n, theta, N, M, eos, pad):
    ids = [list(r) for r in ids.tolist()]
    n0 = len(ids[0])
    out = [[] for _ in ids]
    done = [False] * len(ids)
    for _ in range(n):
        x = model.logits(ids)
        for b in range(len(ids)):
            row = P.process(x[b], ids[b], repetition_penalty=theta, no_repeat_ngram_size=N, min_new_tokens=M,
                            prompt_len=n0, eos=eos)
            t = pad if done[b] else int(np.argmax(row))
            done[b] = done[b] or t in eos
            ids[b].append(t)
            out[b].append(t)
        if all(done):
            break
    return out


@pytest.mark.parametrize("theta,N,M,eos", [(1.3, 0, 0, None), (1.0, 2, 0, None), (1.5, 3, 4, [5]),
                                           (1.0, 0, 0, [2, 5]), (0.8, 1, 2, [5])])
def test_greedy_oracle_loop_equals_hf_generate(theta, N, M, eos):
    V = 17
    model = _Fake(V).eval()
    ids = torch.tensor([[1, 2, 3, 1], [4, 4, 0, 6]])
    kw = dict(max_new_tokens=10, do_sample=False, repetition_penalty=theta, no_repeat_ngram_size=N,
              min_new_tokens=M, pad_token_id=0, eos_token_id=eos, use_cache=False)
    hf = model.generate(ids, **kw)[:, ids.shape[1]:].tolist()
    got = _greedy_oracle(model, ids, 10, theta, N, M, eos or [], 0)
    for b in range(2):   # 🤗 stops when every row is done; the padded tail is the same
        assert got[b] == hf[b][:len(got[b])], (b, got[b], hf[b])


def _logprob_rows(x):
    """(fp32 log-softmax rows, ambiguous) of the beam step, the oracle's own log_softmax kept before any patch"""
    return _LOG_SOFTMAX(x)


_LOG_SOFTMAX = beam_oracle.log_softmax


@pytest.mark.parametrize("theta,N,M,eos", [(1.4, 2, 0, ()), (0.7, 0, 0, (3,)), (1.0, 3, 3, (3, 5)), (2.0, 1, 0, ())])
def test_beam_oracle_loop_with_processors_equals_hf_generate(theta, N, M, eos):
    """🤗 5.5's _beam_search runs the processors on the fp32 log-softmax with the prompt and the beam's own generated
    tokens as history (flat_running_sequences): the beam oracle fed those processed rows in place of its log-softmax
    (it is patched to the identity) returns 🤗's sequences and scores."""
    V, K, n, B = 13, 3, 7, 2
    model = _Fake(V).eval()
    ids = torch.tensor([[1, 2, 3, 1], [4, 4, 0, 6]])
    prompts = ids.tolist()
    hf = model.generate(ids, max_new_tokens=n, do_sample=False, num_beams=K, repetition_penalty=theta,
                        no_repeat_ngram_size=N, min_new_tokens=M, pad_token_id=0, eos_token_id=list(eos) or None,
                        num_return_sequences=K, output_scores=True, return_dict_in_generate=True, use_cache=False)

    def logits_fn(rows):   # rows: the B*K beams' generated tokens
        seqs = [prompts[i // K] + list(r) for i, r in enumerate(rows)]
        out = []
        for s_, x in zip(seqs, model.logits(seqs)):
            lp, _ = _logprob_rows(x)
            out.append(P.process(lp, s_, repetition_penalty=theta, no_repeat_ngram_size=N, min_new_tokens=M,
                                 prompt_len=4, eos=eos))
        return np.stack(out)

    with mock.patch.object(beam_oracle, "log_softmax", lambda x: (np.asarray(x, np.float32),
                                                                  np.zeros(np.shape(x), bool))):
        seqs, scores, flagged, _ = beam_oracle.beam_search(logits_fn, B, K, n, eos, 1.0, False, K, 0, tie_tol=1e-6)
    assert not np.any(flagged)
    got = hf.sequences[:, 4:].numpy().reshape(B, K, -1)
    want = np.full((B, K, n), beam_oracle.fill_value(eos, 0), np.int64)
    want[:, :, :got.shape[2]] = got
    np.testing.assert_array_equal(seqs, want)
    # 🤗's log_softmax is torch's fp32 one, the oracle's the fp64 one rounded once: scores agree to the last bits
    np.testing.assert_allclose(scores, hf.sequences_scores.numpy().reshape(B, K), rtol=1e-5, atol=1e-4)


# ---- the C ABI ---------------------------------------------------------------------------------------------------------
def _params(**kw):
    p = _lib.LogitsProcessParams(logits=0x10000000, stride_row=389, out=0x20000000, out_stride_row=389,
                                 prefix=0x30000000, prefix_stride=64, prefix_count=5, prefix_cap=64, R=4, V=389,
                                 dtype=_lib.PCV_BF16, row_group=1, rows_per_hist=1, repetition_penalty=1.2,
                                 no_repeat_ngram=3, min_new_tokens=2, prompt_len=5, n_eos=1)
    p.eos[0] = 7
    for k, v in kw.items():
        setattr(p, k, v)
    return p


REFUSALS = [
    (dict(logits=None), b"a pointer is NULL"), (dict(prefix=None), b"a pointer is NULL"),
    (dict(tail_len=0x4000), b"tail_len is set without a tail"), (dict(dtype=_lib.PCV_E4M3), b"unknown dtype 3"),
    (dict(V=0, stride_row=0, out_stride_row=0), b"V=0 must be in [1, 32768]"),
    (dict(V=32769, stride_row=32769, out_stride_row=32769), b"V=32769"), (dict(R=0), b"R=0 must be >= 1"),
    (dict(stride_row=388), b"stride_row=388"), (dict(out_stride_row=388), b"out_stride_row=388"),
    (dict(row_map=0x5000, row_group=0), b"row_group=0 must be >= 1"), (dict(rows_per_hist=0), b"rows_per_hist=0"),
    (dict(log_softmax=2), b"log_softmax=2"), (dict(prefix_cap=-1), b"must be >= 0"),
    (dict(repetition_penalty=0.0), b"repetition_penalty=0 must be finite and > 0"),
    (dict(repetition_penalty=float("inf")), b"must be finite"), (dict(repetition_penalty=float("nan")), b"finite"),
    (dict(no_repeat_ngram=9), b"no_repeat_ngram=9 must be in [0, 8]"), (dict(no_repeat_ngram=-1), b"[0, 8]"),
    (dict(min_new_tokens=-1), b"min_new_tokens=-1"), (dict(n_eos=5), b"n_eos=5 must be in [0, 4]"),
    (dict(n_eos=0), b"min_new_tokens=2 needs EOS ids"), (dict(eos=(ctypes.c_int32 * 4)(389)), b"EOS id 389"),
]


@pytest.mark.parametrize("kw,reason", REFUSALS, ids=[f"refuse{i}" for i in range(len(REFUSALS))])
def test_refusals_come_before_any_cuda_call(kw, reason):
    lib = _lib.lib()
    assert lib.pcv_logits_process_supported(ctypes.byref(_params())) == 1, lib.pcv_last_error()
    p = _params(**kw)
    assert lib.pcv_logits_process_supported(ctypes.byref(p)) == 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()
    assert lib.pcv_logits_process(ctypes.byref(p), None) != 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()


def test_edges_are_accepted_and_beam_logprobs_takes_fp32_only():
    lib = _lib.lib()
    for kw in (dict(no_repeat_ngram=8), dict(no_repeat_ngram=0), dict(min_new_tokens=0, n_eos=0),
               dict(V=32768, stride_row=32768, out_stride_row=32768), dict(dtype=_lib.PCV_F32), dict(log_softmax=1),
               dict(tail=0x6000, tail_len=0x7000), dict(row_map=0x5000, row_group=4)):
        assert lib.pcv_logits_process_supported(ctypes.byref(_params(**kw))) == 1, (kw, lib.pcv_last_error())
    assert lib.pcv_logits_process_supported(None) == 0 and b"params is NULL" in lib.pcv_last_error()
    b = _lib.BeamStepParams(logits=0x1000, stride_row=64, length_penalty=1.0, B=1, K=2, V=64, dtype=_lib.PCV_BF16,
                            hist_len=8)
    for i, f in enumerate(("running_scores", "finished_scores", "finished_flags", "running_hist", "finished_hist",
                           "hist_scratch", "item_flags", "counters", "cand_scores", "cand_index", "next_tokens",
                           "parents")):
        setattr(b, f, 0x10000000 * (i + 1))
    assert lib.pcv_beam_step_supported(ctypes.byref(b)) == 1, lib.pcv_last_error()
    assert lib.pcv_beam_step_logprobs_supported(ctypes.byref(b)) == 0
    assert b"must be fp32" in lib.pcv_last_error()
    b.dtype = _lib.PCV_F32
    assert lib.pcv_beam_step_logprobs_supported(ctypes.byref(b)) == 1, lib.pcv_last_error()


def test_params_layout_matches_the_header(tmp_path):
    import subprocess

    name, cls = "pcv_logits_process_params", _lib.LogitsProcessParams
    header = os.path.join(ROOT, "include", "pcv_attn.h")
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void){",
             f'printf("size %zu\\n", sizeof({name}));']
    lines += [f'printf("{f} %zu\\n", offsetof({name}, {f}));' for f, _ in cls._fields_]
    lines.append("return 0;}")
    (tmp_path / "l.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-o", str(tmp_path / "l"), str(tmp_path / "l.c")])
    got = dict(l.split() for l in subprocess.check_output([str(tmp_path / "l")]).decode().split("\n") if l)
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f
    assert (_lib.PROCESS_MAX_NGRAM, _lib.PROCESS_MAX_EOS) == (P.MAX_NGRAM, P.MAX_EOS) == (8, 4)


# ---- ops and GraphedDecoder: argument checks ---------------------------------------------------------------------------
def test_ops_refuse_bad_arguments_before_any_launch():
    from perceiver_io_b200 import ops

    with pytest.raises(RuntimeError, match="CUDA .* tensors only"):
        ops.process_logits(torch.zeros(2, 8), torch.zeros(2, 4, dtype=torch.long), 2)
    # past the CUDA check (CPU stand-ins): every history row read must exist, on the logits' device; nothing launches
    with mock.patch.object(ops, "_require_cuda", lambda *t: None), \
            mock.patch.object(ops._lib, "lib", side_effect=AssertionError("no library call")):
        x, h = torch.zeros(8, 16), torch.zeros(2, 4, dtype=torch.long)
        with pytest.raises(ValueError, match="prefix has 2 rows; 8 processed rows at 1 per history row read 8"):
            ops.process_logits(x, h, 2)
        with pytest.raises(ValueError, match="prefix has 2 rows; 8 processed rows at 3 per history row read 3"):
            ops.process_logits(x, h, 2, rows_per_hist=3)
        with pytest.raises(ValueError, match="tail has 2 rows; 4 processed rows"):
            ops.process_logits(x, torch.zeros(4, 4, dtype=torch.long), 2, tail=h,
                               tail_len=torch.zeros(1, dtype=torch.int32), row_map=torch.zeros(4, dtype=torch.int32))
        with pytest.raises(ValueError, match="prefix is on meta, the logits on cpu"):
            ops.process_logits(x, torch.zeros(8, 4, dtype=torch.long, device="meta"), 2)
        with pytest.raises(ValueError, match="prefix_len is on meta"):
            ops.process_logits(x, torch.zeros(8, 4, dtype=torch.long), torch.zeros(8, dtype=torch.int32, device="meta"))
        with pytest.raises(ValueError, match="row_map is on meta"):
            ops.process_logits(x, h, 2, row_map=torch.zeros(2, dtype=torch.int32, device="meta"))


def _decoder():
    from perceiver_io_b200 import generation as G

    dec = G.GraphedDecoder.__new__(G.GraphedDecoder)
    dec.batch, dec.max_new_tokens = 2, 8
    dec.model = types.SimpleNamespace(config=types.SimpleNamespace(vocab_size=100, num_channels=64))
    dec._sampling = (1.0, 0, 1.0)
    return G, dec


@pytest.mark.parametrize("kw,match", [
    (dict(repetition_penalty=0.0), "repetition_penalty must be a number > 0"),
    (dict(repetition_penalty=float("inf")), "repetition_penalty"), (dict(repetition_penalty=True), "repetition_penalty"),
    (dict(repetition_penalty=1e-50), "finite and > 0 in fp32"), (dict(repetition_penalty=1e39), "in fp32"),
    (dict(no_repeat_ngram_size=9), "no_repeat_ngram_size must be an integer in \\[0, 8\\]"),
    (dict(no_repeat_ngram_size=-1), "no_repeat_ngram_size"), (dict(no_repeat_ngram_size=1.5), "no_repeat_ngram_size"),
    (dict(min_new_tokens=-1), "min_new_tokens must be an integer >= 0"),
    (dict(min_new_tokens=3), "min_new_tokens=3 needs eos_token_id"),
    (dict(eos_token_id=[1, 2, 3, 4, 5]), "at most 4 EOS ids"), (dict(eos_token_id=100), "EOS id must be in"),
    (dict(eos_token_id=3, pad_token_id=100), "pad_token_id must be None or an id"),
    (dict(eos_token_id="x"), "eos_token_id must be None"),
])
def test_set_sampling_refuses_and_keeps_the_old_values(kw, match):
    G, dec = _decoder()
    dec.set_sampling(0.5, 3, 0.9, repetition_penalty=1.1, no_repeat_ngram_size=2)
    before = (dec._sampling, dec._process, dec._eos, dec._pad_token)
    with pytest.raises(ValueError, match=match):
        dec.set_sampling(**kw)
    assert (dec._sampling, dec._process, dec._eos, dec._pad_token) == before


def test_set_sampling_values_and_neutral_defaults():
    G, dec = _decoder()
    dec.set_sampling()
    assert dec._process == G._NO_PROCESS and dec._eos == () and dec._pad_token is None
    dec.set_sampling(repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=8, eos_token_id=[5, 9])
    assert dec._process == (1.2, 3, 8) and dec._eos == (5, 9) and dec._pad_token == 5
    dec.set_sampling(eos_token_id=5, pad_token_id=0)
    assert dec._process == G._NO_PROCESS and dec._pad_token == 0


def test_generate_verify_and_speculative_refuse_processors():
    G, dec = _decoder()
    dec._bounds, dec._seeded, dec._remaining = torch.zeros(2, 2, 6, dtype=torch.int32), True, 8
    dec.set_sampling(repetition_penalty=1.2)
    first = torch.zeros(2, 1, dtype=torch.long)
    with pytest.raises(ValueError, match="logits=True .* not covered with logits processors"):
        dec.generate(first, 2, logits=True)
    with pytest.raises(ValueError, match="check_every must be an integer >= 1"):
        dec.generate(first, 2, check_every=0)
    with pytest.raises(ValueError, match="speculative verification is not covered"):
        dec.verify(torch.zeros(2, 3, dtype=torch.long), torch.zeros(2, 2, 100), (1.0, 0, 1.0))
    _, draft = _decoder()
    draft._bounds, draft._process = dec._bounds, G._NO_PROCESS
    with pytest.raises(ValueError, match="not covered with logits processors"):
        G.speculative_generate(dec, draft, first, 4)


def test_beam_and_contrastive_refuse_bad_processor_values_before_any_work():
    G, dec = _decoder()
    dec.batch = 4
    ids = torch.zeros(2, 5, dtype=torch.long)
    with pytest.raises(ValueError, match="beam_search: no_repeat_ngram_size"):
        dec.beam_search(ids, 0, 4, num_beams=2, no_repeat_ngram_size=9)
    with pytest.raises(ValueError, match="beam_search: min_new_tokens=2 needs eos_token_id"):
        dec.beam_search(ids, 0, 4, num_beams=2, min_new_tokens=2)
    dec.model.config.num_channels = 64
    with pytest.raises(ValueError, match="contrastive_search: repetition_penalty"):
        dec.contrastive_search(ids, 0, 4, penalty_alpha=0.6, top_k=2, repetition_penalty=-1.0)
