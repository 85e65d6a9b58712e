"""Graph-replayed decoding (generation.GraphedDecoder) against the eager cached step, measured in one run on one GPU.

A CausalSequenceModel at the GiantMIDI config of tools/fp8_kv_bench.py (C = 768, H = 8, 18 self-attention layers,
max_latents 2048, max_seq_len 6144) with random weights and a full 6144-token context, at batch 1 and 16.  Four arms,
alternating step by step: the eager cached step with bf16 and with FP8 (e4m3) caches (every token slides both windows by
one), and GraphedDecoder with each cache.  Each step is timed with CUDA events around the call and a synchronise, so the
wall time of a step includes its host work.  Prints one JSON line (also written to --out) with the card's name and
power limit; ms per token as median (min-max).  --profile traces the steps with torch.profiler instead (a run of its
own) and reports device time per step (the sum of kernel times) and kernels per step.

--step-tokens 1,4,8,16,64 measures multi-token replays instead (GraphedDecoder.extend): at each batch and for bf16 and
FP8 arenas, one replay of k tokens on the full context, then rewind(k) so that every replay sees the same windows; the
(cache, k) arms alternate replay by replay.  It reports ms per replay and ms per token, median (min-max); with --profile,
device time and kernels per replay from a trace.  --kernel-leg times the attention kernels alone at the decode-core
shape (B = 8, 16384 cached tokens, C = 1024, H = 8) for k = 2, 4, 5, 16, 64 query rows: ops.attention_window on bf16
and e4m3 arenas, pcv_attn_decode_window (k <= 4), ops.attention_decode_fp8 (pcv_attn_cached_fp8 above 4 rows) and
ops.attention on a bf16 cache, alternated, CUDA events around 20 launches.

--spec-rows 4,8 measures a batched speculative loop at each batch (bf16 arenas): every round feeds k draft tokens per
row in one extend(k) replay; each draft is accepted with probability --accept until the row's first rejection (seeded
per row).  Two arms, alternated round by round: "per_row" rewinds every row by its own rejected count; "refeed" is the
loop without per-row rewinds: it rewinds every row to the smallest accepted count, and a row's other accepted tokens
lead its next replay again (in place of drafts).  A token counts as accepted once it is kept by its row for good.  It
reports ms per accepted token (replay and rewind, CUDA events and a synchronise around each round; over all rows) and
replays per accepted token of one row, median (min-max) over --reps blocks of --steps rounds; every block starts from
the prompt (a per-row rewind of everything fed).

--sample measures sampling.  Model leg: at each batch, bf16 and FP8 arenas, and the sampling values top_k=10 /
top_p=0.5 / greedy, two arms alternate token by token: "eager" is GraphedDecoder.step followed by the eager 🤗-equivalent
warper chain (divide, topk + masked_fill, sort + softmax + cumsum + scatter, softmax + multinomial; argmax when greedy),
what a caller writes without the device sampler; "generate" is one GraphedDecoder.generate replay.  Each token is timed
with CUDA events around the call and a synchronise (host work included); ms per token, median (min-max).  Kernel leg:
ops.sample_tokens against the eager chain alone at V = 389 and 32000 and R = 1, 16 and 1024 rows, alternated, CUDA
events around 50 launches."""
import argparse
import json
import os
import random
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


def run_tokens(batch, ks, reps, profile=False):
    """ms per replay of GraphedDecoder.extend(k) on the full context, each replay followed by rewind(k)."""
    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    n, prefix = cfg.max_seq_len, cfg.max_seq_len - cfg.max_latents
    tokens = torch.randint(0, cfg.vocab_size, (batch, n + max(ks)), device="cuda")
    arms = [(kind, k) for kind in ("bf16", "fp8") for k in ks]
    decs, times = {}, {a: [] for a in arms}
    with torch.no_grad():
        for kind in ("bf16", "fp8"):
            decs[kind] = P.GraphedDecoder(model, batch=batch, max_new_tokens=max(ks), kv_cache=kind)
            decs[kind].prefill(tokens[:, :n], prefix)

        def replay(kind, k):
            dec = decs[kind]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dec.extend(tokens[:, n:n + k])
            e1.record()
            dec.rewind(k)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1)

        for _ in range(2):       # every graph recorded and warmed up
            for a in arms:
                replay(*a)
        res = {"batch": batch, "context": n}
        if profile:
            from torch.profiler import ProfilerActivity, profile as trace

            for a in arms:
                with trace(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    for _ in range(reps):
                        replay(*a)
                kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                res[f"{a[0]}_k{a[1]}_kernel_ms_per_replay"] = round(
                    sum(e.time_range.elapsed_us() for e in kern) / reps / 1e3, 4)
                res[f"{a[0]}_k{a[1]}_kernels_per_replay"] = round(len(kern) / reps, 1)
        else:
            for _ in range(reps):
                for a in arms:
                    times[a].append(replay(*a))
            for kind, k in arms:
                res[f"{kind}_k{k}_ms_per_replay"] = stats(times[(kind, k)])
                res[f"{kind}_k{k}_ms_per_token"] = stats([t / k for t in times[(kind, k)]])
    del decs, model
    torch.cuda.empty_cache()
    return res


def run_spec(batch, k, rounds, reps, accept):
    """The batched speculative loop with per-row rewinds against the smallest-count rewind and refeed."""
    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    n, prefix = cfg.max_seq_len, cfg.max_seq_len - cfg.max_latents
    tokens = torch.randint(0, cfg.vocab_size, (batch, n + k), device="cuda")
    feed = tokens[:, n:n + k]          # the token values do not change the work of a replay
    arms = ("per_row", "refeed")
    with torch.no_grad():
        decs = {a: P.GraphedDecoder(model, batch=batch, max_new_tokens=(rounds + 1) * k) for a in arms}
        for dec in decs.values():
            dec.prefill(tokens[:, :n], prefix)
            dec.extend(feed)           # the graph recorded and warmed up
            dec.rewind(k)
        torch.cuda.synchronize()

        def accepted(rng, m):          # drafts kept before the first rejection, at most m
            a = 0
            while a < m and rng.random() < accept:
                a += 1
            return a

        res = {"batch": batch, "k": k, "context": n, "accept": accept, "rounds_per_block": rounds}
        blocks = {a: {"ms": [], "replays": []} for a in arms}
        for rep in range(reps):
            # the same seeded draws per row in both arms
            rngs = {a: [random.Random(1000 * rep + b) for b in range(batch)] for a in arms}
            fed = {a: [0] * batch for a in arms}
            carry = [0] * batch        # refeed: accepted tokens a row has to feed again
            ms = {a: 0.0 for a in arms}
            for _ in range(rounds):
                for a in arms:
                    dec = decs[a]
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    dec.extend(feed)
                    if a == "per_row":
                        acc = [accepted(r, k) for r in rngs[a]]
                        dec.rewind([k - x for x in acc])
                        fed[a] = [f + x for f, x in zip(fed[a], acc)]
                    else:
                        known = [min(c, k) for c in carry]
                        got = [kn + accepted(r, k - kn) for kn, r in zip(known, rngs[a])]
                        m = min(got)
                        dec.rewind(k - m)
                        carry = [c - kn + g - m for c, kn, g in zip(carry, known, got)]
                        fed[a] = [f + m for f in fed[a]]
                    e1.record()
                    torch.cuda.synchronize()
                    ms[a] += e0.elapsed_time(e1)
            for a in arms:
                kept = sum(fed[a])
                blocks[a]["ms"].append(ms[a] / max(kept, 1))
                blocks[a]["replays"].append(rounds * batch / max(kept, 1))
                res.setdefault(f"{a}_accepted_per_row_per_round", []).append(round(kept / batch / rounds, 3))
                decs[a].rewind(fed[a])   # back to the prompt for the next block
        for a in arms:
            res[f"{a}_ms_per_accepted_token"] = stats(blocks[a]["ms"])
            res[f"{a}_replays_per_accepted_token"] = stats(blocks[a]["replays"])
        res["speedup"] = round(statistics.median(blocks["refeed"]["ms"]) / statistics.median(blocks["per_row"]["ms"]), 2)
    del decs, model
    torch.cuda.empty_cache()
    return res


def kernel_leg(ks=(2, 4, 5, 16, 64), reps=7, iters=20):
    """The attention kernels alone at the decode-core shape: ms per call, median (min-max) of `reps` alternated
    rounds of `iters` launches."""
    from perceiver_io_b200 import ops

    B, M, C, H = 8, 16384, 1024, 8
    g = torch.Generator(device="cuda").manual_seed(0)
    k = torch.randn(B, M, C, device="cuda", generator=g).bfloat16()
    v = torch.randn(B, M, C, device="cuda", generator=g).bfloat16()
    kd = (k.float().abs().reshape(-1, H, C // H).amax(dim=(0, 2)) / 448.0).contiguous()
    vd = (v.float().abs().reshape(-1, H, C // H).amax(dim=0) / 448.0).contiguous()
    k8, v8 = ops.fp8_quantize(k, kd, H), ops.fp8_quantize(v, vd, H)
    bounds = torch.tensor([0, M], dtype=torch.int32, device="cuda")
    scale = (C // H) ** -0.5
    out = {"shape": {"B": B, "cached": M, "C": C, "H": H}}
    for n in ks:
        q = torch.randn(B, n, C, device="cuda", generator=g).bfloat16()
        arms = {
            "window_bf16": lambda: ops.attention_window(q, k, v, bounds, H, scale, causal=True),
            "window_fp8": lambda: ops.attention_window(q, k8, v8, bounds, H, scale, causal=True, k_descale=kd,
                                                       v_descale=vd),
            "decode_fp8" if n <= 4 else "cached_fp8": lambda: ops.attention_decode_fp8(q, k8, v8, kd, vd, H, scale,
                                                                                        causal=True),
            "attention_bf16": lambda: ops.attention(q, k, v, H, scale, causal=True),
        }
        if n <= 4:
            arms["decode_window_bf16"] = lambda: ops.attention_decode_window(q, k, v, bounds, H, scale, causal=True)
            arms["decode_window_fp8"] = lambda: ops.attention_decode_window(q, k8, v8, bounds, H, scale, causal=True,
                                                                            k_descale=kd, v_descale=vd)
        times = {a: [] for a in arms}
        for fn in arms.values():
            fn()
        torch.cuda.synchronize()
        for _ in range(reps):
            for a, fn in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[a].append(e0.elapsed_time(e1) / iters)
        out[f"k{n}"] = {a: stats(t) for a, t in times.items()}
    return out


SAMPLE_CONFIGS = {"top_k=10": (1.0, 10, 1.0), "top_p=0.5": (1.0, 0, 0.5), "greedy": (0.0, 0, 1.0)}


def eager_sample(logits, temperature, top_k, top_p):
    """The 🤗 warper chain and multinomial in eager torch: (B, V) logits -> (B, 1) tokens."""
    if temperature == 0:
        return logits.argmax(-1, keepdim=True)
    s = logits.float() / temperature
    if top_k:
        s = s.masked_fill(s < torch.topk(s, top_k)[0][..., -1:], float("-inf"))
    if top_p < 1:
        srt, idx = torch.sort(s, descending=False)
        remove = srt.softmax(-1).cumsum(-1) <= 1 - top_p
        remove[..., -1:] = False
        s = s.masked_fill(remove.scatter(-1, idx, remove), float("-inf"))
    return torch.multinomial(s.softmax(-1), 1)


def run_sample(batch, steps):
    """ms per token: step + the eager chain against one generate replay, per cache kind and sampling config."""
    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    n, prefix = cfg.max_seq_len, cfg.max_seq_len - cfg.max_latents
    warm = 3
    tokens = torch.randint(0, cfg.vocab_size, (batch, n), device="cuda")
    out = []
    with torch.no_grad():
        for kind in ("bf16", "fp8"):
            decs = {}
            for arm in ("eager", "generate"):
                decs[arm] = P.GraphedDecoder(model, batch=batch, max_new_tokens=warm + steps, kv_cache=kind)
                decs[arm].set_seed(1)
            for name, vals in SAMPLE_CONFIGS.items():
                state = {}
                for arm, dec in decs.items():
                    dec.set_sampling(*vals)
                    state[arm] = {"tok": dec.draw(dec.prefill(tokens, prefix)), "times": []}

                def one(arm):
                    st, dec = state[arm], decs[arm]
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    if arm == "eager":
                        st["tok"] = eager_sample(dec.step(st["tok"]), *vals)
                    else:
                        st["tok"] = dec.generate(st["tok"], 1)
                    e1.record()
                    torch.cuda.synchronize()
                    return e0.elapsed_time(e1)

                for _ in range(warm):
                    for arm in decs:
                        one(arm)
                for _ in range(steps):
                    for arm in decs:
                        state[arm]["times"].append(one(arm))
                res = {"batch": batch, "cache": kind, "sampling": name,
                       "eager_ms_per_token": stats(state["eager"]["times"]),
                       "generate_ms_per_token": stats(state["generate"]["times"])}
                res["speedup"] = round(statistics.median(state["eager"]["times"])
                                       / statistics.median(state["generate"]["times"]), 3)
                out.append(res)
    del decs, model
    torch.cuda.empty_cache()
    return out


def sample_kernel_leg(reps=7, iters=50):
    """ms per call of ops.sample_tokens and of the eager chain, median (min-max) over reps blocks of iters calls."""
    from perceiver_io_b200 import ops

    out = []
    for V in (389, 32000):
        for R in (1, 16, 1024):
            logits = torch.randn(R, V, device="cuda").bfloat16() * 3
            seeds = torch.arange(R, device="cuda")
            pos = torch.zeros(R, dtype=torch.int32, device="cuda")
            for name, vals in SAMPLE_CONFIGS.items():
                arms = {"kernel": lambda: ops.sample_tokens(logits, seeds, pos, *vals),
                        "eager": lambda: eager_sample(logits, *vals)}
                times = {a: [] for a in arms}
                for a, f in arms.items():
                    f()
                torch.cuda.synchronize()
                for _ in range(reps):
                    for a, f in arms.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(iters):
                            f()
                        e1.record()
                        torch.cuda.synchronize()
                        times[a].append(e0.elapsed_time(e1) / iters)
                out.append({"V": V, "R": R, "sampling": name, "kernel_ms": stats(times["kernel"]),
                            "eager_ms": stats(times["eager"])})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true", help="trace the steps instead of timing them")
    ap.add_argument("--step-tokens", default=None, help="e.g. 1,4,8,16,64: time k-token replays (extend + rewind)")
    ap.add_argument("--kernel-leg", action="store_true", help="time the attention kernels at the decode-core shape")
    ap.add_argument("--spec-rows", default=None, help="e.g. 4,8: a batched speculative loop of k-token drafts, "
                                                     "per-row rewind against the smallest-count rewind and refeed")
    ap.add_argument("--accept", type=float, default=0.7, help="--spec-rows: acceptance probability of a draft token")
    ap.add_argument("--reps", type=int, default=5, help="--spec-rows: blocks of --steps rounds")
    ap.add_argument("--sample", action="store_true", help="step + the eager warper chain against generate, and the "
                                                          "sampler kernel against the eager chain")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "graph_decode_bench measures on a GPU"
    res = {"card": card()}
    if a.sample:
        res["sample_kernel"] = sample_kernel_leg()
        res["sample"] = [r for b in a.batches.split(",") for r in run_sample(int(b), a.steps)]
    elif a.kernel_leg:
        res["kernel_leg"] = kernel_leg()
    elif a.spec_rows:
        res["spec_rows"] = [run_spec(int(b), int(k), a.steps, a.reps, a.accept) for b in a.batches.split(",")
                            for k in a.spec_rows.split(",")]
    elif a.step_tokens:
        ks = [int(k) for k in a.step_tokens.split(",")]
        res["tokens_profile" if a.profile else "tokens"] = [run_tokens(int(b), ks, a.steps, a.profile)
                                                            for b in a.batches.split(",")]
    else:
        res["step_profile" if a.profile else "step"] = [run(int(b), a.steps, a.profile) for b in a.batches.split(",")]
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
