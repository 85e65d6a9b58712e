"""Graph-replayed decoding (generation.GraphedDecoder) against the eager cached step, measured in one run on one GPU.

A CausalSequenceModel at the GiantMIDI config of tools/fp8_kv_bench.py (C = 768, H = 8, 18 self-attention layers,
max_latents 2048, max_seq_len 6144) with random weights and a full 6144-token context, at batch 1 and 16.  Four arms,
alternating step by step: the eager cached step with bf16 and with FP8 (e4m3) caches (every token slides both windows by
one), and GraphedDecoder with each cache.  Each step is timed with CUDA events around the call and a synchronise, so the
wall time of a step includes its host work.  Prints one JSON line (also written to --out) with the card's name and
power limit; ms per token as median (min-max).  --profile traces the steps with torch.profiler instead (a run of its
own) and reports device time per step (the sum of kernel times) and kernels per step."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import perceiver_io_b200 as P  # noqa: E402
from perceiver_io_b200 import modules  # noqa: E402
from fp8_kv_bench import GIANTMIDI, card, stats  # noqa: E402

ARMS = ("eager_bf16", "eager_fp8", "graph_bf16", "graph_fp8")


def run(batch, steps, profile=False):
    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    n, prefix = cfg.max_seq_len, cfg.max_seq_len - cfg.max_latents
    warm = 3
    tokens = torch.randint(0, cfg.vocab_size, (batch, n + warm + steps + 1), device="cuda")
    state = {}
    with torch.no_grad():
        for arm in ARMS:
            kind = arm.split("_")[1]
            if arm.startswith("eager"):
                modules.fp8_config["kv_cache"] = kind == "fp8"
                try:
                    o = model(tokens[:, :n], prefix_len=prefix, kv_cache=[])
                finally:
                    modules.fp8_config["kv_cache"] = False
                state[arm] = {"cache": o.kv_cache, "times": [], "logits": o.logits[:, -1]}
            else:
                dec = P.GraphedDecoder(model, batch=batch, max_new_tokens=warm + steps, kv_cache=kind)
                state[arm] = {"dec": dec, "times": [], "logits": dec.prefill(tokens[:, :n], prefix)}

        def step(arm, s):
            st = state[arm]
            tok = tokens[:, n + s:n + s + 1]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            if arm.startswith("eager"):
                cache = st["cache"]
                # full context: every new token slides both windows by one
                cache = [(cache[0][0][:, 1:], cache[0][1][:, 1:])] + [(k[:, 1:], v[:, 1:]) for k, v in cache[1:]]
                e0.record()
                o = model(tok, prefix_len=prefix, kv_cache=cache)
                e1.record()
                st["cache"], st["logits"] = o.kv_cache, o.logits[:, -1]
            else:
                e0.record()
                st["logits"] = st["dec"].step(tok)
                e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1)

        for s in range(warm):   # every shape warmed up; the graphs are recorded at their first step
            for arm in ARMS:
                step(arm, s)
        res = {"batch": batch, "context": n}
        if profile:
            from torch.profiler import ProfilerActivity, profile as trace

            for arm in ARMS:
                with trace(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    for s in range(warm, warm + steps):
                        step(arm, s)
                kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                res[f"{arm}_kernel_ms_per_token"] = round(sum(e.time_range.elapsed_us() for e in kern) / steps / 1e3, 4)
                res[f"{arm}_kernels_per_token"] = round(len(kern) / steps, 1)
        else:
            for s in range(warm, warm + steps):
                for arm in ARMS:
                    state[arm]["times"].append(step(arm, s))
            for arm in ARMS:
                res[f"{arm}_ms_per_token"] = stats(state[arm]["times"])
            for kind in ("bf16", "fp8"):
                res[f"speedup_{kind}"] = round(statistics.median(state[f"eager_{kind}"]["times"])
                                               / statistics.median(state[f"graph_{kind}"]["times"]), 2)
                # the graph and the eager step computed the same next-token logits (up to kernel choice and rounding)
                a, b = state[f"graph_{kind}"]["logits"].float(), state[f"eager_{kind}"]["logits"].float()
                res[f"max_rel_logit_diff_{kind}"] = round(((a - b).abs().max() / b.abs().max()).item(), 5)
    del state, model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true", help="trace the steps instead of timing them")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "graph_decode_bench measures on a GPU"
    res = {"card": card(), ("step_profile" if a.profile else "step"):
           [run(int(b), a.steps, a.profile) for b in a.batches.split(",")]}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
