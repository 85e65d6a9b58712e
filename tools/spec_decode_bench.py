"""Speculative sampling with a draft model (generation.speculative_generate's round) against plain
GraphedDecoder.generate, measured in one run on one GPU.

Target: the GiantMIDI config of tools/graph_decode_bench.py (C = 768, H = 8, 18 self-attention layers, vocabulary 389)
with a full 6144-token context; draft: the same width with 2 self-attention layers.  Both have random weights, so the
acceptance rate — and any speed-up — measures the machinery, not a trained draft / target pair.  At batch 1 and 16, bf16
and FP8 arenas, top_k = 10 for both models, the arms alternate round by round: "plain" is target.generate of 8 tokens;
"spec_G" (G = 2, 4, 8) is one speculative round: draft.generate(t_0, G+1, logits=True), target.verify, the one
device-to-host read of the accept counts, and both rewinds.  Every round starts from the prompt (a rewind of everything
fed) under a new seed.  A round is timed from a synchronise to the end of its rewinds and a synchronise (host work
included); CUDA events split the draft replays and the verify replay, the rest is the read and the rewinds.  It reports
ms per emitted token (per batch row), median (min-max), the measured acceptance rate and tokens per round.  Kernel leg:
ops.spec_verify (B = 16, G = 4) against ops.sample_tokens on the same (16, 5, V) rows at V = 389 and 32000, alternated,
CUDA events around 50 launches.  Prints one JSON line (also written to --out) with the card's name and power limit."""
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

GS = (2, 4, 8)
PLAIN = 8
VALS = (1.0, 10, 1.0)


def run(batch, kind, rounds):
    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    target = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    draft = P.CausalSequenceModel(P.CausalSequenceModelConfig(**dict(GIANTMIDI, num_self_attention_layers=2)))
    draft = draft.cuda().bfloat16().eval()
    n, prefix = cfg.max_seq_len, cfg.max_seq_len - cfg.max_latents
    prompt = torch.randint(0, cfg.vocab_size, (batch, n), device="cuda")
    budget = 2 * (max(GS) + 1) + PLAIN
    tgt = P.GraphedDecoder(target, batch=batch, max_new_tokens=budget, kv_cache=kind)
    dft = P.GraphedDecoder(draft, batch=batch, max_new_tokens=budget, kv_cache=kind)
    with torch.no_grad():
        logits = tgt.prefill(prompt, prefix)
        dft.prefill(prompt, prefix)
    for d in (tgt, dft):
        d.set_sampling(*VALS)
    arms = ["plain"] + [f"spec_{g}" for g in GS]
    rec = {a: {"ms_per_token": [], "draft_ms": [], "verify_ms": [], "sync_rewind_ms": [], "tokens": [],
               "accepted": 0, "proposed": 0} for a in arms}

    def reset():
        for d in (tgt, dft):
            fed = [d._fed - (d._lag[b] if d._lag else 0) for b in range(batch)]
            d.rewind(fed)

    def one(arm, r):
        for d in (tgt, dft):
            d.set_seed(1000 + r)
        first = tgt.draw(logits)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if arm == "plain":
            tgt.generate(first, PLAIN)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            rec[arm]["ms_per_token"].append(ms / PLAIN)
            rec[arm]["tokens"].append(PLAIN)
            reset()
            return
        g = int(arm.split("_")[1])
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        drafts, q = dft.generate(first, g + 1, logits=True)
        e[1].record()
        _, acc = tgt.verify(torch.cat([first, drafts[:, :g]], dim=1), q[:, :g], draft_sampling=VALS)
        e[2].record()
        counts = acc.to("cpu").tolist()
        back = [g - c for c in counts]
        tgt.rewind(back)
        dft.rewind(back)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        per_row = sum(c + 1 for c in counts) / batch
        st = rec[arm]
        st["ms_per_token"].append(ms / per_row)
        st["draft_ms"].append(e[0].elapsed_time(e[1]))
        st["verify_ms"].append(e[1].elapsed_time(e[2]))
        st["sync_rewind_ms"].append(ms - e[0].elapsed_time(e[2]))
        st["tokens"].append(per_row)
        st["accepted"] += sum(counts)
        st["proposed"] += g * batch
        reset()

    with torch.no_grad():
        for r in range(2):          # warm-up: records every graph
            for arm in arms:
                one(arm, r)
        for a in arms:
            rec[a] = {k: ([] if isinstance(v, list) else 0) for k, v in rec[a].items()}
        for r in range(rounds):
            for arm in arms:
                one(arm, 100 + r)
    out = {}
    for a, st in rec.items():
        o = {"ms_per_token": stats(st["ms_per_token"]), "tokens_per_round": round(statistics.mean(st["tokens"]), 3)}
        if a != "plain":
            o["acceptance"] = round(st["accepted"] / st["proposed"], 4)
            for k in ("draft_ms", "verify_ms", "sync_rewind_ms"):
                o[k] = stats(st[k])
        out[a] = o
    return out


def kernel_leg(V, launches=50, reps=5):
    gen = torch.Generator(device="cuda").manual_seed(V)
    B, G = 16, 4
    tgt = torch.randn(B, G + 1, V, device="cuda", generator=gen).bfloat16()
    dft = (tgt[:, :G].float() + torch.randn(B, G, V, device="cuda", generator=gen)).bfloat16()
    seeds = torch.arange(B, device="cuda", dtype=torch.long)
    pos = torch.arange(G + 1, device="cuda", dtype=torch.int32).repeat(B, 1)
    toks = torch.randint(0, V, (B, G + 1), device="cuda", generator=gen)
    calls = {"spec_verify": lambda: ops.spec_verify(tgt, dft, toks, seeds, pos, VALS, VALS),
             "sample_tokens": lambda: ops.sample_tokens(tgt, seeds, pos, *VALS)}
    times = {k: [] for k in calls}
    for f in calls.values():
        f()
    for _ in range(reps):
        for k, f in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                f()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e3 / launches)
    return {k: {"us": stats(v)} for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = {"card": card(), "note": "random weights: the acceptance rate and speed-up measure the machinery, not a "
                                   "trained draft / target pair", "model": {}, "kernel": {}}
    for b in [int(x) for x in a.batches.split(",")]:
        for kind in ("bf16", "fp8"):
            res["model"][f"B{b}_{kind}"] = run(b, kind, a.rounds)
            print(f"# B={b} {kind}: {json.dumps(res['model'][f'B{b}_{kind}'])}", flush=True)
    for V in (389, 32000):
        res["kernel"][f"V{V}"] = kernel_leg(V)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
