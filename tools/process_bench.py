"""Cost of the device logits processors (``ops.process_logits``) on an H100: per-token time of ``generate``,
``beam_search`` (K=4) and ``contrastive_search`` (K=4, α=0.6) with the processors off and on (repetition_penalty=1.2,
no_repeat_ngram_size=3, min_new_tokens=8), the processor kernel alone, and the plain ``step`` replay with and without
the token-arena scatter.  Both arms of the on / off comparison pass the same EOS id (min_new_tokens needs one), and
their runs alternate in one process.  B in {1, 8}, V = 32768, a 1024-token prompt, 256 new tokens, random weights (the times
depend on shapes only).  The card's name and power limit are read in the same run.  Writes one JSON object to the
path given by ``--out`` and prints it."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PROMPT, NEW, V = 1024, 256, 32768
ON = dict(repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=8)
OFF = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().split("\n")[0]
    name, limit = (s.strip() for s in q.split(","))
    return {"gpu": name, "power_limit": limit}


def model():
    import perceiver_io_b200 as P

    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(vocab_size=V, max_seq_len=PROMPT + NEW, max_latents=512, num_channels=512,
                                      num_heads=8, num_self_attention_layers=6, num_self_attention_rotary_layers=-1,
                                      cross_attention_dropout=0.0, output_norm=True, init_scale=0.02)
    return P.CausalSequenceModel(cfg).cuda().bfloat16().eval()


def _elapsed_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def arm(m, B, kind, kw):
    """One per-token sample (ms) of ``kind`` with processor values ``kw``: the replays alone, the prefill outside the
    events (beam and contrastive search prefill inside the call: the same call's prefill alone is timed and
    subtracted).  Both arms pass the same EOS id, so they differ only in the processors."""
    import perceiver_io_b200 as P

    K = 1 if kind == "generate" else 4
    ids = torch.randint(0, V, (B, PROMPT), generator=torch.Generator().manual_seed(1)).cuda()
    dec = P.GraphedDecoder(m, batch=B * K, max_new_tokens=NEW + 1, kv_cache="bf16")
    eos = [V - 1]
    if kind == "generate":
        def sample():
            logits = dec.prefill(ids, PROMPT // 2)
            dec.set_sampling(0.0, eos_token_id=eos, **kw)
            first = dec.draw(logits)
            return _elapsed_ms(lambda: dec.generate(first, NEW, check_every=NEW)) / NEW
    else:
        if kind == "beam":
            run = lambda: dec.beam_search(ids, PROMPT // 2, NEW, num_beams=K, eos_token_id=eos, check_every=NEW, **kw)
        else:
            run = lambda: dec.contrastive_search(ids, PROMPT // 2, NEW, penalty_alpha=0.6, top_k=K, eos_token_id=eos,
                                                 check_every=NEW, **kw)

        def sample():
            whole = _elapsed_ms(run)
            pre = _elapsed_ms(lambda: dec.prefill(ids.repeat_interleave(K, 0), PROMPT // 2))
            return (whole - pre) / NEW
    sample()   # records the graphs
    return sample


def per_token(m, B, kind, rounds=5):
    """off / on samples alternated in one process: median, min and max per arm, and the median overhead."""
    fns = {"off": arm(m, B, kind, OFF), "on": arm(m, B, kind, ON)}
    got = {"off": [], "on": []}
    for _ in range(rounds):
        for name, fn in fns.items():
            got[name].append(fn())
    med = {k: sorted(v)[rounds // 2] for k, v in got.items()}
    return {"off": med["off"], "on": med["on"], "overhead_ms": med["on"] - med["off"],
            "off_range": [min(got["off"]), max(got["off"])], "on_range": [min(got["on"]), max(got["on"])]}


def kernel_alone(B, n=200):
    """µs per launch of the processor kernel alone: n launches captured in one CUDA graph, timed by events around its
    replay, so the host wrapper is outside the window."""
    from perceiver_io_b200 import ops

    x = torch.randn(B, V, device="cuda").bfloat16()
    hist = torch.randint(0, V, (B, PROMPT + NEW), device="cuda")
    pos = torch.full((B,), PROMPT + NEW - 1, dtype=torch.int32, device="cuda")
    out = torch.empty(B, V, device="cuda")
    fn = lambda: ops.process_logits(x, hist, pos, out=out, prompt_len=PROMPT, eos=(V - 1,), **ON)
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    times = sorted(_elapsed_ms(g.replay) / n * 1000.0 for _ in range(5))
    return {"median_us": times[2], "range_us": [times[0], times[-1]]}


class _NoWrite:
    """A token arena whose scatter does nothing: the step graph without the write (its index math stays)."""

    def __init__(self, t):
        self.shape = t.shape

    def scatter_(self, *a):
        return None


def step_with_without_write(m, B, rounds=6, n=200):
    import perceiver_io_b200 as P

    ids = torch.randint(0, V, (B, PROMPT), generator=torch.Generator().manual_seed(2)).cuda()
    decs = []
    for write in (True, False):
        d = P.GraphedDecoder(m, batch=B, max_new_tokens=rounds * n + 8, kv_cache="bf16")
        d.prefill(ids, PROMPT // 2)
        if not write:
            d._tokens = _NoWrite(d._tokens)
        tok = torch.zeros(B, 1, dtype=torch.long, device="cuda")
        d.step(tok)
        decs.append((d, tok))
    res = {True: [], False: []}
    for r in range(rounds):   # alternated in one process
        for write, (d, tok) in zip((True, False), decs):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(n // rounds):
                d.step(tok)
            b.record()
            torch.cuda.synchronize()
            res[write].append(a.elapsed_time(b) / (n // rounds) * 1000.0)
    return {"with_write_us": sorted(res[True])[rounds // 2], "without_write_us": sorted(res[False])[rounds // 2],
            "with_write_all_us": res[True], "without_write_all_us": res[False]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("process_bench needs a CUDA device")
    out = {"card": card(), "prompt": PROMPT, "new_tokens": NEW, "vocab": V, "processors_on": ON, "eos_both_arms": [V - 1],
           "per_token_ms": {}, "kernel_in_graph": {}, "step_arena_write": {}}
    m = model()
    for B in (1, 8):
        for kind in ("generate", "beam", "contrastive"):
            out["per_token_ms"][f"{kind}_B{B}"] = per_token(m, B, kind)
        out["kernel_in_graph"][f"rows{B}"] = kernel_alone(B)
        out["kernel_in_graph"][f"rows{4 * B}"] = kernel_alone(4 * B)
        out["step_arena_write"][f"B{B}"] = step_with_without_write(m, B)
    out["card_after"] = card()
    text = json.dumps(out)
    with open(args.out, "w") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
