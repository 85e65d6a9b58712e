"""Beam search per generated token: ``GraphedDecoder.beam_search`` (one graph replay per token: step, device beam step,
KV gather of the generated rows) against the loop a caller writes without it (``step``, 🤗's beam bookkeeping in eager
torch, and the whole-arena ``reorder``).

A CausalSequenceModel at the GiantMIDI config of tools/fp8_kv_bench.py (C = 768, 18 self-attention layers, max_seq_len
6144, max_latents 2048, vocab 389), random bf16 weights, a full 6144-token prompt, bf16 and FP8 arenas, K = 3 and 8
beams, batch 1 and 4, n = 32 and 256 generated tokens, EOS id 0 (random weights rarely emit it, so runs go to n).  The
two arms alternate call by call; each timing covers the n - 1 replays / (reorder, step, bookkeeping) rounds after the
prefill's first token, from the first replay / reorder to the end (CUDA events, ending in a synchronise).  Prints one
JSON line (also written to --out) with ms per generated token, median (min-max), and the card's name and power limit
read in the same run.  --profile instead traces one call of each arm
with torch.profiler and reports the device time of the beam-step kernels, the gather and the eager ``reorder`` (one JSON
line, also written to --out)."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import perceiver_io_b200 as P  # noqa: E402
from perceiver_io_b200 import generation  # noqa: E402
from fp8_kv_bench import GIANTMIDI, card, stats  # noqa: E402

EOS = (0,)


def eager_beam_search(dec, ids, prefix, n, K, eos=EOS, lp=1.0, on_first=None):
    """The loop without the device beam step: 🤗's _beam_search bookkeeping in eager torch, ``step`` and ``reorder``."""
    B = ids.shape[0]
    dev = ids.device
    logits = dec.prefill(ids[:, None].expand(B, K, ids.shape[1]).reshape(B * K, -1), prefix)
    V = logits.shape[-1]
    keep = max(2, len(eos) + 1) * K
    eos_t = torch.tensor(eos, device=dev)
    running = torch.full((B, K), -1e9, device=dev)
    running[:, 0] = 0
    fin = torch.full((B, K), -1e9, device=dev)
    fin_flag = torch.zeros(B, K, dtype=torch.bool, device=dev)
    run_seq = torch.full((B, K, n), eos[0], dtype=torch.long, device=dev)
    fin_seq = run_seq.clone()
    unsat = torch.ones(B, 1, dtype=torch.bool, device=dev)
    first_k = torch.arange(keep, device=dev) < K
    offs = (torch.arange(B, device=dev) * K)[:, None]
    for t in range(n):
        lp_ = torch.log_softmax(logits.float(), -1).view(B, K, V) + running[:, :, None]
        top, idx = lp_.view(B, K * V).topk(keep)
        par, tok = idx // V, idx % V
        seq = run_seq.gather(1, par[:, :, None].expand(B, keep, n)).clone()
        seq[:, :, t] = tok
        hit = torch.isin(tok, eos_t) | (t + 1 >= n)
        trun = top + hit.float() * -1e9
        sel = trun.topk(K)[1]
        running = trun.gather(1, sel)
        run_seq = seq.gather(1, sel[:, :, None].expand(B, K, n))
        s = top / ((t + 1) ** lp)
        s = s + (~unsat).float() * -1e9 + (~(hit & first_k)).float() * -1e9
        merged = torch.cat([fin, s], 1)
        msel = merged.topk(K)[1]
        fin = merged.gather(1, msel)
        fin_flag = torch.cat([fin_flag, hit & first_k], 1).gather(1, msel)
        fin_seq = torch.cat([fin_seq, seq], 1).gather(1, msel[:, :, None].expand(B, K, n))
        best = running[:, :1] / ((t + 1) ** lp)
        worst = torch.where(fin_flag, fin.min(1, keepdim=True)[0], -1e9)
        unsat = unsat & (best > worst).any(-1, keepdim=True)
        if t == n - 1:
            break
        if t == 0 and on_first is not None:   # the graph arm's window starts at its first replay: the same point
            on_first()
        dec.reorder((par.gather(1, sel) + offs).flatten())
        logits = dec.step(tok.gather(1, sel).reshape(B * K, 1))
    return fin_seq, fin


def timed(fn, n):
    """ms per token of the n - 1 tokens after the first: events from the first replay / step to the end."""
    marks = {}

    def first():
        marks["e0"] = torch.cuda.Event(enable_timing=True)
        marks["e0"].record()

    e1 = torch.cuda.Event(enable_timing=True)
    fn(first)
    e1.record()
    torch.cuda.synchronize()
    return marks["e0"].elapsed_time(e1) / (n - 1)


def graph_arm(dec, ids, prefix, n, K):
    def run(on_first):
        orig = generation.GraphedForward.__call__
        fired = []

        def call(self, *a):
            if not fired:
                fired.append(1)
                on_first()
            return orig(self, *a)

        generation.GraphedForward.__call__ = call
        try:
            dec.beam_search(ids, prefix, n, num_beams=K, eos_token_id=list(EOS), check_every=n)
        finally:
            generation.GraphedForward.__call__ = orig
    return run


def run(kind, K, batch, n, reps):
    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    prefix = cfg.max_seq_len - cfg.max_latents
    ids = torch.randint(1, cfg.vocab_size, (batch, cfg.max_seq_len), device="cuda")
    dec = P.GraphedDecoder(model, batch=batch * K, max_new_tokens=n, kv_cache=kind)
    arms = {"graph": graph_arm(dec, ids, prefix, n, K),
            "eager": lambda f: eager_beam_search(dec, ids, prefix, n, K, on_first=f)}
    times = {a: [] for a in arms}
    with torch.no_grad():
        for a, fn in arms.items():   # warm-up
            timed(fn, n)
        for _ in range(reps):
            for a, fn in arms.items():
                times[a].append(timed(fn, n))
        g = dec.beam_search(ids, prefix, n, num_beams=K, eos_token_id=list(EOS))
        e_seq, e_sc = eager_beam_search(dec, ids, prefix, n, K)
    res = {"cache": kind, "K": K, "batch": batch, "n": n, "graph_ms_per_token": stats(times["graph"]),
           "eager_ms_per_token": stats(times["eager"]),
           "speedup": round(statistics.median(times["eager"]) / statistics.median(times["graph"]), 3),
           "best_sequence_equal": bool(torch.equal(g.sequences[:, 0], e_seq[:, 0]))}
    del dec, model
    torch.cuda.empty_cache()
    return res


def profile(kind, K, batch, n):
    from torch.profiler import ProfilerActivity, profile as prof, record_function

    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    prefix = cfg.max_seq_len - cfg.max_latents
    ids = torch.randint(1, cfg.vocab_size, (batch, cfg.max_seq_len), device="cuda")
    dec = P.GraphedDecoder(model, batch=batch * K, max_new_tokens=n, kv_cache=kind)
    orig_reorder = dec.reorder

    def reorder(idx):
        with record_function("eager_reorder"):
            orig_reorder(idx)

    dec.reorder = reorder
    with torch.no_grad():
        dec.beam_search(ids, prefix, n, num_beams=K, eos_token_id=list(EOS))
        eager_beam_search(dec, ids, prefix, n, K)
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            dec.beam_search(ids, prefix, n, num_beams=K, eos_token_id=list(EOS))
            eager_beam_search(dec, ids, prefix, n, K)
            torch.cuda.synchronize()
    # kernels: device time per launch; the eager reorder: its range's device time (the largest of the CPU range and
    # its GPU annotation, which both carry the name), n - 1 calls
    per = {}
    for name, per_token in (("beam_rows_kernel", 1), ("beam_item_kernel", 1), ("kv_gather_kernel", 2)):
        evs = [ev for ev in p.key_averages() if name in ev.key]
        total = sum(getattr(ev, "device_time_total", 0.0) for ev in evs) / 1000.0
        count = sum(ev.count for ev in evs)
        per[name] = {"device_ms_per_launch": round(total / max(1, count), 4), "launches": count,
                     "device_ms_per_token": round(per_token * total / max(1, count), 4)}
    total = max([getattr(ev, "device_time_total", 0.0) for ev in p.key_averages() if ev.key == "eager_reorder"] + [0.0])
    per["eager_reorder"] = {"device_ms_per_token": round(total / 1000.0 / (n - 1), 4), "calls": n - 1}
    return {"cache": kind, "K": K, "batch": batch, "n": n, "profile": per}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ns", default="32,256")
    ap.add_argument("--ks", default="3,8")
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--caches", default="bf16,fp8")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("beam_bench needs a CUDA device (there is no CPU measurement)")
    results = []
    ks, batches, ns, caches = ([int(x) for x in a.ks.split(",")], [int(x) for x in a.batches.split(",")],
                               [int(x) for x in a.ns.split(",")], a.caches.split(","))
    for kind in caches:
        for K in ks:
            for batch in batches:
                if a.profile:
                    results.append(profile(kind, K, batch, ns[0]))
                    continue
                for n in ns:
                    results.append(run(kind, K, batch, n, a.reps))
                    print(json.dumps(results[-1]), file=sys.stderr, flush=True)
    line = json.dumps({"bench": "beam_search", "card": card(), "results": results})
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
