"""CPU checks of prompt-lookup decoding: the oracle's lookup (oracle/lookup_oracle.py) against 🤗's own
PromptLookupCandidateGenerator.get_candidates on many random histories; the oracle's greedy round loop against 🤗
``generate(prompt_lookup_num_tokens=G, max_matching_ngram_size=N)`` on a toy causal model, token for token and round
for round; every refusal of the C ABI before any CUDA call; the header layout; no spills in the kernel; and
``prompt_lookup_generate``'s refusals and stated budget."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import lookup_oracle as LO
from perceiver_io_b200 import _lib

transformers = pytest.importorskip("transformers")
from transformers.generation.candidate_generator import PromptLookupCandidateGenerator  # noqa: E402


def _hf_lookup(history, G, N, eos):
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor(list(eos) or [-7]), num_output_tokens=G,
                                         max_matching_ngram_size=N, max_length=10 ** 9)
    ids = torch.tensor([history])
    out, _ = gen.get_candidates(ids)
    return out[0, len(history):].tolist()


@pytest.mark.parametrize("G,N", [(1, 1), (1, 16), (10, 2), (63, 2), (63, 16), (4, 3)])
def test_oracle_lookup_equals_hf(G, N):
    rng = np.random.default_rng(G * 31 + N)
    hits = 0
    for trial in range(300):
        vocab = int(rng.integers(2, 9))
        L = int(rng.integers(1, 90))
        h = [int(x) for x in rng.integers(0, vocab, L)]
        eos = [int(x) for x in rng.integers(0, vocab + 3, int(rng.integers(0, 3)))]
        want = _hf_lookup(h, G, N, eos)
        assert LO.lookup(h, G, N, eos) == want, (h, G, N, eos)
        hits += bool(want)
        for lim in (0, 1, G // 2):
            assert LO.lookup(h, G, N, eos, lim) == want[:lim]
    assert hits > 50


@pytest.mark.parametrize("h,G,N,eos,want", [
    ([1, 2, 3, 4], 5, 2, (), []),                           # no match
    ([3, 3], 5, 2, (), [3]),                                # the 1-gram (3,) at 0 continues with the suffix itself
    ([1, 2], 5, 2, (), []),                                 # only the suffix itself matches
    ([5], 5, 2, (), []),                                    # one id: nothing to match
    ([1, 2, 7, 8, 1, 2], 5, 2, (), [7, 8, 1, 2]),           # the continuation is cut by the history's end
    ([1, 2, 9, 8, 1, 2], 5, 2, (9,), []),                   # EOS first: empty, and no other window is tried
    ([1, 2, 3, 9, 4, 1, 2], 5, 2, (9,), [3]),               # EOS mid-draft
    ([1, 2, 3, 4, 5, 6, 1, 2], 1, 2, (), [3]),              # G = 1
    ([4, 1, 2, 9, 1, 2, 5, 2], 3, 2, (), [9, 1, 2]),        # the 2-gram fails, the 1-gram (2,) at 2 continues
])
def test_oracle_lookup_edges_equal_hf(h, G, N, eos, want):
    assert _hf_lookup(h, G, N, eos) == want
    assert LO.lookup(h, G, N, eos) == want


# ---- 🤗 generate() on a toy causal model against the oracle round loop ------------------------------------------------
class _Cfg(transformers.PretrainedConfig):
    model_type = "pcv_toy_lookup"

    def __init__(self, vocab_size=11, **kw):
        super().__init__(**kw)
        self.vocab_size = vocab_size


class _Toy(transformers.PreTrainedModel, transformers.GenerationMixin):
    """Causal logits: position t's row is a fixed function of ids t - 1 and t; no cache (every call sees every id)."""
    config_class = _Cfg

    def __init__(self, V, seed):
        super().__init__(_Cfg(vocab_size=V))
        self.dummy = torch.nn.Parameter(torch.zeros(1))
        g = torch.Generator().manual_seed(seed)
        self.T = torch.randn(V, V, generator=g) * 3
        self.U = torch.randn(V, V, generator=g)

    def prepare_inputs_for_generation(self, input_ids, **kw):
        return {"input_ids": input_ids}

    def forward(self, input_ids, **kw):
        prev = torch.cat([input_ids[:, :1], input_ids[:, :-1]], dim=1)
        logits = self.T[input_ids] + self.U[prev]
        return transformers.modeling_outputs.CausalLMOutputWithPast(logits=logits,
                                                                    past_key_values=transformers.DynamicCache())

    def greedy(self, seq):
        with torch.no_grad():
            return self.forward(torch.tensor([seq])).logits[0].argmax(-1).tolist()


# 🤗 5.5's prompt lookup fails without an EOS id (torch.isin on None): the runs without one use an id outside V
@pytest.mark.parametrize("seed,G,N,eos", [(1, 4, 2, [99]), (2, 10, 2, [99]), (3, 3, 1, [99]), (6, 6, 3, [5]),
                                          (5, 10, 2, [0, 3])])
def test_greedy_round_loop_equals_hf_generate(monkeypatch, seed, G, N, eos):
    V, n = 7, 30
    model = _Toy(V, seed).eval()
    prompt = [1, 2, 3, 1, 2, 4, 1, 2, 3]
    seen = []
    orig_get = PromptLookupCandidateGenerator.get_candidates

    def get(self, input_ids):
        out, lg = orig_get(self, input_ids)
        seen.append([out.shape[1] - input_ids.shape[1], None])
        return out, lg

    def update(self, input_ids, scores, num_matches):
        seen[-1][1] = int(num_matches)

    monkeypatch.setattr(PromptLookupCandidateGenerator, "get_candidates", get)
    monkeypatch.setattr(PromptLookupCandidateGenerator, "update_candidate_strategy", update)
    hf = model.generate(torch.tensor([prompt]), max_new_tokens=n, do_sample=False, prompt_lookup_num_tokens=G,
                        max_matching_ngram_size=N, eos_token_id=eos, pad_token_id=0, use_cache=True)
    hf = hf[0, len(prompt):].tolist()
    # 🤗's t_0 of its first round is the prompt's last id, as the loop's is
    got, rounds = LO.greedy_rounds(model.greedy, prompt, n, G, N, eos)
    assert got == hf[:len(got)], (got, hf)
    assert len(got) == n or got[-1] in eos
    # the limit rule caps a row's drafts at the tokens it has left minus one, so no round runs past n; 🤗 offers up to
    # G there and drops what passes max_length.  The rounds agree wherever the cap does not bind.
    emitted, compared = 0, 0
    for i, (offered, acc) in enumerate(rounds):
        if n - emitted - 1 >= G:
            assert tuple(seen[i]) == (offered, acc), (i, seen, rounds)
            compared += 1
        emitted += acc + 1
    assert compared >= 2 and any(a > 0 for _, a in rounds), rounds


# ---- the C ABI ----------------------------------------------------------------------------------------------------------
def _params(**kw):
    p = _lib.PromptLookupParams()
    p.ids, p.ids_stride, p.length, p.length_stride = 0x1000, 512, 0x2000, 1
    p.B, p.cap, p.G, p.N, p.n_eos, p.k = 3, 500, 10, 2, 1, 0
    p.eos[0] = 7
    p.drafts, p.drafts_stride, p.counts = 0x3000, 64, 0x4000
    for k, v in kw.items():
        setattr(p, k, v)
    return p


ROUND = dict(k=4, fed=0x5000, draws=0x6000, t0=0x7000, t0_stride=64, accepted=0x8000, unfinished=0x9000, left=0xa000)
REFUSALS = [(dict(**{f: None}), b"pointer is NULL") for f in ("ids", "length", "drafts", "counts")] + [
    (dict(B=0), b"B=0 must be >= 1"),
    (dict(cap=0), b"cap=0 must be >= 1"),
    (dict(ids_stride=499), b"ids_stride=499 is below cap=500"),
    (dict(length_stride=-1), b"length_stride=-1"),
    (dict(G=0), b"G=0 must be in [1, 63]"),
    (dict(G=64), b"G=64 must be in [1, 63]"),
    (dict(N=0), b"N=0 must be in [1, 16]"),
    (dict(N=17), b"N=17 must be in [1, 16]"),
    (dict(n_eos=5), b"n_eos=5 must be in [0, 4]"),
    (dict(drafts_stride=9), b"drafts_stride=9 is below G=10"),
    (dict(k=-1), b"k=-1 must be in [0, G+1=11]"),
    (dict(k=12, **{f: v for f, v in ROUND.items() if f != "k"}), b"k=12 must be in [0, G+1=11]"),
    (dict(k=3), b"needs fed, draws, t0, accepted, unfinished and left"),
    (dict(ROUND, left=None), b"needs fed, draws"),
    (dict(ROUND, t0_stride=0), b"t0_stride=0 must be >= 1"),
]


@pytest.mark.parametrize("kw,reason", REFUSALS, ids=[f"refuse{i}" for i in range(len(REFUSALS))])
def test_abi_refusals_come_before_any_cuda_call(kw, reason):
    lib = _lib.lib()
    p = _params(**kw)
    assert lib.pcv_prompt_lookup_supported(ctypes.byref(p)) == 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()
    assert lib.pcv_prompt_lookup(ctypes.byref(p), None) != 0
    assert reason in lib.pcv_last_error(), lib.pcv_last_error()


def test_abi_accepts_the_edges():
    lib = _lib.lib()
    for kw in (dict(), dict(G=1, drafts_stride=1), dict(G=63), dict(N=1), dict(N=16), dict(n_eos=4), dict(B=1, cap=1),
               dict(ROUND), dict(ROUND, k=1), dict(ROUND, k=11)):
        assert lib.pcv_prompt_lookup_supported(ctypes.byref(_params(**kw))) == 1, (kw, lib.pcv_last_error())
    assert lib.pcv_prompt_lookup_supported(None) == 0 and b"params is NULL" in lib.pcv_last_error()


def test_lookup_params_layout_matches_the_header(tmp_path):
    import subprocess

    header = os.path.join(ROOT, "include", "pcv_attn.h")
    S = _lib.PromptLookupParams
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void){",
             'printf("size %zu\\n", sizeof(pcv_prompt_lookup_params));',
             'printf("max_drafts %d\\n", PCV_LOOKUP_MAX_DRAFTS);', 'printf("max_ngram %d\\n", PCV_LOOKUP_MAX_NGRAM);',
             'printf("max_eos %d\\n", PCV_LOOKUP_MAX_EOS);']
    lines += [f'printf("{f} %zu\\n", offsetof(pcv_prompt_lookup_params, {f}));' for f, _ in S._fields_]
    lines.append("return 0;}")
    (tmp_path / "l.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-o", str(tmp_path / "l"), str(tmp_path / "l.c")])
    got = dict(l.split() for l in subprocess.check_output([str(tmp_path / "l")]).decode().split("\n") if l)
    assert int(got["size"]) == ctypes.sizeof(S)
    assert (int(got["max_drafts"]), int(got["max_ngram"]), int(got["max_eos"])) == (
        _lib.LOOKUP_MAX_DRAFTS, _lib.LOOKUP_MAX_NGRAM, _lib.LOOKUP_MAX_EOS) == (63, 16, 4)
    for f, _ in S._fields_:
        assert int(got[f]) == getattr(S, f).offset, f


def test_lookup_kernel_has_no_spills():
    log = os.path.join(ROOT, "build", "pcv_lookup.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was not built in this tree")
    entries = open(log).read().split("Compiling entry function")[1:]
    assert len(entries) == 1 and "lookup_kernel" in entries[0].split("\n")[0]
    assert "0 bytes spill stores, 0 bytes spill loads" in entries[0], entries[0][:300]


# ---- GraphedDecoder.prompt_lookup_generate: refusals and the stated budget ----------------------------------------------
def _decoder(B=3, T=40, V=11):
    from test_window_rows_cpu import _decoder as rows_decoder

    dec = rows_decoder(B, 30, 10, 40, 16, T)
    dec._graphs = {}
    dec._seeds, dec._seeded, dec._sampling = torch.zeros(B, dtype=torch.int64), True, (1.0, 0, 1.0)
    dec.model = types.SimpleNamespace(config=types.SimpleNamespace(vocab_size=V))
    return dec


def test_budget_is_stated_and_refused_before_any_work():
    from perceiver_io_b200.generation import prompt_lookup_budget

    assert prompt_lookup_budget(20, 10, 1) == 20
    assert prompt_lookup_budget(20, 10, 4) == 31
    assert prompt_lookup_budget(5, 10, 4) == 10     # a row never drafts past its n tokens: at most n - 1 drafts
    assert prompt_lookup_budget(1, 63, 2) == 2
    for B, T, n in ((1, 9, 10), (3, 30, 20)):
        dec = _decoder(B=B, T=T)
        before = (dec._bounds.clone(), dec._fed, dec._remaining, dec._tokens)
        with pytest.raises(RuntimeError, match=f"needs {prompt_lookup_budget(n, 10, B)}"):
            dec.prompt_lookup_generate(torch.zeros(B, 1, dtype=torch.long), n)
        assert torch.equal(dec._bounds, before[0]) and (dec._fed, dec._remaining) == before[1:3]
        assert dec._lookup_state == () and dec._graphs == {}


def test_refusals_leave_the_state_untouched():
    dec = _decoder()
    first = torch.zeros(3, 1, dtype=torch.long)
    for kw, exc, match in ((dict(num_output_tokens=0), ValueError, "num_output_tokens must be an integer in"),
                           (dict(num_output_tokens=64), ValueError, r"\[1, 63\]"),
                           (dict(num_output_tokens=True), ValueError, "num_output_tokens"),
                           (dict(max_matching_ngram_size=0), ValueError, "max_matching_ngram_size"),
                           (dict(max_matching_ngram_size=17), ValueError, r"\[1, 16\]"),
                           (dict(n=0), ValueError, "n must be an integer >= 1"),
                           (dict(first=torch.zeros(3, 2, dtype=torch.long)), ValueError, r"\(3, 1\) int64 first"),
                           (dict(first=torch.zeros(3, 1, dtype=torch.int32)), ValueError, "int64 first")):
        args = dict(first=first, n=4)
        args.update(kw)
        with pytest.raises(exc, match=match):
            dec.prompt_lookup_generate(**args)
    big = _decoder(V=_lib.SAMPLE_MAX_VOCAB + 1)
    with pytest.raises(RuntimeError, match="vocabularies up to"):
        big.prompt_lookup_generate(first, 4)
    fresh = _decoder()
    fresh._bounds = None
    with pytest.raises(RuntimeError, match="prefill"):
        fresh.prompt_lookup_generate(first, 4)
    assert dec._lookup_state == () and dec._graphs == {} and dec._fed == 0
