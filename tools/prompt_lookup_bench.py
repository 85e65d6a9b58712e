"""Prompt-lookup decoding (GraphedDecoder.prompt_lookup_generate) against plain GraphedDecoder.generate, measured in one
run on one GPU.

Model: the GiantMIDI config of tools/fp8_kv_bench.py (C = 768, H = 8, 18 self-attention layers, vocabulary 389) with a
full 6144-token context, at batch 1 and 16, bf16 and FP8 arenas, greedy and top_k = 10.  Prompts: a random one (few
n-gram matches: it measures the overhead of the lookup rounds) and a repetitive one (a 37-token motif repeated, where
drafts are found).  The weights are random, so the acceptance rate measures the machinery; speed on a trained
checkpoint is not measured.  The arms alternate call by call: "plain" is generate(first, T); "lookup_G" (G = 4, 10;
N = 2) is prompt_lookup_generate(first, T, G).  Every call starts from the prompt (a rewind of everything fed) under a
new seed and is timed from a synchronise to its return and a synchronise.  It reports ms per emitted token (per batch
row), median (min-max), the acceptance rate, tokens per round and rounds per call.  The read cost per round is the
one device-to-host read of a round's (3, B) counts plus a per-row rewind, timed alone on an idle stream.  Kernel leg:
ops.prompt_lookup on (B, 6144 + 256) histories at B = 1 and 16, CUDA events around 50 launches.  Prints one JSON line
(also written to --out) with the card's name and power limit."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import perceiver_io_b200 as P  # noqa: E402
from perceiver_io_b200 import ops  # noqa: E402
from fp8_kv_bench import GIANTMIDI, card, stats  # noqa: E402

GS = (4, 10)
NGRAM = 2
SAMPLINGS = {"greedy": (0.0, 0, 1.0), "top_k10": (1.0, 10, 1.0)}


def prompts(batch, n, vocab):
    gen = torch.Generator().manual_seed(batch)
    motif = torch.randint(0, vocab, (37,), generator=gen)
    return {"random": torch.randint(0, vocab, (batch, n), generator=gen),
            "repetitive": motif.repeat(n // 37 + 1)[:n].repeat(batch, 1)}


def run(model, cfg, batch, kind, tokens, reps):
    n, prefix = cfg.max_seq_len, cfg.max_seq_len - cfg.max_latents
    out = {}
    for pname, prompt in prompts(batch, n, cfg.vocab_size).items():
        dec = P.GraphedDecoder(model, batch=batch, max_new_tokens=tokens + max(GS) + 1, kv_cache=kind)
        with torch.no_grad():
            logits = dec.prefill(prompt.cuda(), prefix).clone()
        for sname, vals in SAMPLINGS.items():
            dec.set_sampling(*vals)
            arms = ["plain"] + [f"lookup_{g}" for g in GS]
            rec = {a: {"ms_per_token": [], "rounds": [], "accepted": 0, "proposed": 0, "emitted": 0} for a in arms}

            def one(arm, r):
                dec.set_seed(1000 + r)
                first = dec.draw(logits)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if arm == "plain":
                    dec.generate(first, tokens)
                    st = None
                else:
                    _, st = dec.prompt_lookup_generate(first, tokens, num_output_tokens=int(arm.split("_")[1]),
                                                       max_matching_ngram_size=NGRAM)
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3
                dec.rewind([dec._fed - (dec._lag[b] if dec._lag else 0) for b in range(batch)])
                return ms, st

            with torch.no_grad():
                for r in range(2):   # warm-up: records every graph these calls use
                    for arm in arms:
                        one(arm, r)
                for r in range(reps):
                    for arm in arms:
                        ms, st = one(arm, 100 + r)
                        rec[arm]["ms_per_token"].append(ms / tokens)
                        if st is not None:
                            rec[arm]["rounds"].append(st["rounds"])
                            rec[arm]["accepted"] += sum(st["accepted"])
                            rec[arm]["proposed"] += sum(st["proposed"])
                            rec[arm]["emitted"] += tokens * batch
            res = {}
            for a, st in rec.items():
                o = {"ms_per_token": stats(st["ms_per_token"])}
                if a != "plain":
                    o["acceptance"] = round(st["accepted"] / max(st["proposed"], 1), 4)
                    o["rounds_per_call"] = round(statistics.mean(st["rounds"]), 2)
                    o["tokens_per_round"] = round(tokens / statistics.mean(st["rounds"]), 3)
                res[a] = o
            out[f"{pname}_{sname}"] = res
        out[f"{pname}_read_ms_per_round"] = stats(read_cost(dec, batch))
        del dec
    return out


def read_cost(dec, batch, reps=50):
    """One device-to-host read of a (3, B) int32 and a per-row rewind (host bookkeeping of a round), on an idle stream."""
    state = torch.zeros(3, batch, dtype=torch.int32, device="cuda")
    first = torch.zeros(batch, 1, dtype=torch.long, device="cuda")
    times = []
    for _ in range(reps):
        dec.extend(first)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        state.to("cpu").tolist()
        dec.rewind([1] * batch)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return times


def kernel_leg(batch, launches=50, reps=5):
    gen = torch.Generator(device="cuda").manual_seed(batch)
    cap = 6144 + 256
    ids = torch.randint(0, 389, (batch, cap), device="cuda", generator=gen)
    lengths = torch.full((batch,), cap, dtype=torch.int32, device="cuda")
    ops.prompt_lookup(ids, lengths, 10, NGRAM)
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            ops.prompt_lookup(ids, lengths, 10, NGRAM)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / launches)
    return {"us": stats(times)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--kinds", default="bf16,fp8")
    ap.add_argument("--tokens", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = {"card": card(), "note": "random weights: acceptance measures the machinery; speed on a trained checkpoint "
                                   "is not measured", "tokens_per_call": a.tokens, "ngram": NGRAM, "model": {},
           "kernel": {}}
    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    for b in [int(x) for x in a.batches.split(",")]:
        for kind in a.kinds.split(","):
            res["model"][f"B{b}_{kind}"] = run(model, cfg, b, kind, a.tokens, a.reps)
            print(f"# B={b} {kind}: {json.dumps(res['model'][f'B{b}_{kind}'])}", flush=True)
    for b in (1, 16):
        res["kernel"][f"B{b}"] = kernel_leg(b)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
