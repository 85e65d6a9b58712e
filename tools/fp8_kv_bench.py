"""FP8 (e4m3) KV cache against the bf16 cache, measured in one run on one GPU.

(1) Decode core at the tools/decode_bench.py shape (B = 8, 16 k cached tokens, C = 1024, H = 8, one new token): the bf16
    streaming decode kernel against the e4m3 one, alternating call by call over four caches per arm so that L2 does not
    hold them.  Achieved GB/s from the algorithmic bytes B*M*(Dqk + Dv) x 2 bytes (bf16) or x 1 byte (e4m3).
(2) Multi-row cached steps at the same shape (--rows, default 5,8,16,32,64,65 new query rows, causal): the new route
    (ops.attention_decode_fp8: the tensor-core kernel of pcv_attn_cached_fp8 up to 64 rows), the dequantising route as
    modules._attend_kv8 runs it above 64 rows (ops.fp8_dequantize of K and V, then ops.attention), and the bf16 cache
    through ops.attention, alternating call by call over four caches per arm.  At 65 rows the new route does not apply.
    Median (min-max) time, algorithmic GB/s (B*M*(Dqk + Dv)*H bytes x the cache's byte width) and the peak extra device
    memory of one call (torch.cuda.max_memory_allocated above what was allocated before it).
(3) Per-token step latency of a CausalSequenceModel at the GiantMIDI config (C = 768, H = 8, 18 self-attention layers,
    max_latents 2048, max_seq_len 6144, rotary over all channels) with random weights and a full context, bf16 and FP8
    caches alternating step by step, at batch 1 and 16, and the bytes each arm's caches hold (arenas + rotated shadows);
    and the same for one cached step of 16 new tokens.

Prints one JSON line (also written to --out); medians with min-max.  --profile traces the model steps with torch.profiler
instead (in a run of its own) and reports device time per step: all kernels, the decode kernels, the FP8 append and
rotary kernels.  --dry-run prints the plan and the byte counts only (no GPU)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import perceiver_io_b200 as P  # noqa: E402
from perceiver_io_b200 import modules, ops  # noqa: E402

B, L, C, H = 8, 16384, 1024, 8
GIANTMIDI = dict(vocab_size=389, max_seq_len=6144, max_latents=2048, num_channels=768, num_heads=8,
                 num_self_attention_layers=18, num_self_attention_rotary_layers=1, cross_attention_dropout=0.0,
                 abs_pos_emb=False, output_norm=True)


def stats(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else q.stderr.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi failed: {e}"


def core(rounds, per_round):
    bytes16, bytes8 = B * L * 2 * C * 2, B * L * 2 * C
    d = C // H
    scale = d ** -0.5
    q = torch.randn(B, 1, C, device="cuda").bfloat16()
    caches16, caches8 = [], []
    for _ in range(4):
        k, v = torch.randn(B, L, C, device="cuda").bfloat16(), torch.randn(B, L, C, device="cuda").bfloat16()
        kd = k.float().abs().reshape(-1, H, d).amax(dim=(0, 2)) / 448.0
        vd = v.float().abs().reshape(-1, H, d).amax(dim=0) / 448.0
        caches16.append((k, v))
        caches8.append((ops.fp8_quantize(k, kd, H), ops.fp8_quantize(v, vd, H), kd, vd))
    arms = {
        "bf16": lambda i: ops.attention(q, *caches16[i % 4], H, scale, causal=True, impl="decode"),
        "fp8": lambda i: ops.attention_decode_fp8(q, caches8[i % 4][0], caches8[i % 4][1], caches8[i % 4][2],
                                                  caches8[i % 4][3], H, scale, causal=True),
    }
    # the two kernels compute the same attention up to the e4m3 rounding of K and V
    o16, o8 = arms["bf16"](0).float(), arms["fp8"](0).float()
    rel = ((o8 - o16).abs().max() / o16.abs().max()).item()
    times = {a: [] for a in arms}
    for a in arms:  # warm-up
        for i in range(8):
            arms[a](i)
    torch.cuda.synchronize()
    for r in range(rounds):
        for a, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(per_round):
                fn(i)
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1) / per_round)
    res = {"shape": {"B": B, "cached_tokens": L, "C": C, "H": H, "new_tokens": 1}, "max_rel_diff_fp8_vs_bf16": rel}
    for a, b in (("bf16", bytes16), ("fp8", bytes8)):
        res[f"{a}_ms"] = stats(times[a])
        res[f"{a}_gbs"] = round(b / statistics.median(times[a]) / 1e6, 1)
    res["speedup"] = round(statistics.median(times["bf16"]) / statistics.median(times["fp8"]), 3)
    del caches16, caches8
    torch.cuda.empty_cache()
    return res


def multirow(rows, rounds, per_round):
    d = C // H
    scale = d ** -0.5
    caches16, caches8 = [], []
    for _ in range(4):
        k, v = torch.randn(B, L, C, device="cuda").bfloat16(), torch.randn(B, L, C, device="cuda").bfloat16()
        kd = k.float().abs().reshape(-1, H, d).amax(dim=(0, 2)) / 448.0
        vd = v.float().abs().reshape(-1, H, d).amax(dim=0) / 448.0
        caches16.append((k, v))
        caches8.append((ops.fp8_quantize(k, kd, H), ops.fp8_quantize(v, vd, H), kd, vd))
        del k, v
    out = []
    for n in rows:
        q = torch.randn(B, n, C, device="cuda").bfloat16()
        arms = {
            "cached": lambda i: ops.attention_decode_fp8(q, *caches8[i % 4], H, scale, causal=True),
            "dequant": lambda i: ops.attention(q, ops.fp8_dequantize(caches8[i % 4][0], caches8[i % 4][2], H, q.dtype),
                                               ops.fp8_dequantize(caches8[i % 4][1], caches8[i % 4][3], H, q.dtype),
                                               H, scale, causal=True),
            "bf16": lambda i: ops.attention(q, *caches16[i % 4], H, scale, causal=True),
        }
        if n > modules.KV8_MAX_ROWS:
            del arms["cached"]
        res = {"rows": n}
        if "cached" in arms:   # same codes, same attention: the two routes differ by the P rounding only
            oc, od = arms["cached"](0).float(), arms["dequant"](0).float()
            res["max_rel_diff_cached_vs_dequant"] = ((oc - od).abs().max() / od.abs().max()).item()
        for a, fn in arms.items():   # warm-up, then the peak extra memory of one call
            for i in range(4):
                fn(i)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            fn(0)
            torch.cuda.synchronize()
            res[f"{a}_peak_extra_mib"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        times = {a: [] for a in arms}
        for r in range(rounds):
            for a, fn in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(per_round):
                    fn(i)
                e1.record()
                torch.cuda.synchronize()
                times[a].append(e0.elapsed_time(e1) / per_round)
        for a in arms:
            width = 2 if a == "bf16" else 1
            res[f"{a}_ms"] = stats(times[a])
            res[f"{a}_gbs"] = round(B * L * 2 * C * width / statistics.median(times[a]) / 1e6, 1)
        if "cached" in arms:
            res["speedup_vs_dequant"] = round(statistics.median(times["dequant"]) / statistics.median(times["cached"]), 3)
        out.append(res)
    del caches16, caches8
    torch.cuda.empty_cache()
    return out


def cache_bytes(cache):
    total = 0
    for kv in cache:
        for t in kv:
            root = t._base if t._base is not None else t
            total += root.untyped_storage().nbytes()
            arena = getattr(root, "_pcv_kv_arena", None)
            if arena is not None and arena.rot is not None:
                total += arena.rot["buf"].untyped_storage().nbytes()
    return total


def step_latency(batch, steps, profile=False, new_tokens=1):
    """Timed steps of ``new_tokens`` tokens each, bf16 and FP8 alternating; with ``profile``, instead a torch.profiler trace of ``steps`` steps per
    arm (in a run of its own: tracing slows the host) summed into device time per step: all kernels, the decode
    attention kernels, and the FP8 route's append / rotary kernels."""
    torch.manual_seed(0)
    cfg = P.CausalSequenceModelConfig(**GIANTMIDI)
    model = P.CausalSequenceModel(cfg).cuda().bfloat16().eval()
    n, prefix = cfg.max_seq_len, cfg.max_seq_len - cfg.max_latents
    w = new_tokens
    tokens = torch.randint(0, cfg.vocab_size, (batch, n + (steps + 3) * w + 8), device="cuda")
    state = {}
    with torch.no_grad():
        for arm in ("bf16", "fp8"):
            modules.fp8_config["kv_cache"] = arm == "fp8"
            o = model(tokens[:, :n], prefix_len=prefix, kv_cache=[])
            state[arm] = {"cache": o.kv_cache, "plen": prefix, "times": []}
        modules.fp8_config["kv_cache"] = False

        def step(arm, s):
            st = state[arm]
            cache = st["cache"]
            # full context: every new token slides the window by one (the oldest prefix token and latent leave)
            cache = [(cache[0][0][:, w:], cache[0][1][:, w:])] + [(k[:, w:], v[:, w:]) for k, v in cache[1:]]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            o = model(tokens[:, n + s * w:n + (s + 1) * w], prefix_len=st["plen"], kv_cache=cache)
            e1.record()
            torch.cuda.synchronize()
            st["cache"] = o.kv_cache
            return e0.elapsed_time(e1)

        for s in range(3):   # the first steps warm up every shape
            for arm in ("bf16", "fp8"):
                step(arm, s)
        res = {"batch": batch, "context": n, "new_tokens": w}
        if profile:
            from torch.profiler import ProfilerActivity, profile as trace

            for arm in ("bf16", "fp8"):
                with trace(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    for s in range(3, 3 + steps):
                        step(arm, s)
                kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                us = lambda evs: sum(e.time_range.elapsed_us() for e in evs) / steps / 1000.0  # noqa: E731
                res[f"{arm}_kernel_ms_per_token"] = round(us(kern), 4)
                res[f"{arm}_decode_kernel_ms_per_token"] = round(us([e for e in kern if "attn_decode" in e.name]), 4)
                res[f"{arm}_append_rotary_kernel_ms_per_token"] = round(
                    us([e for e in kern if "kv_append" in e.name or "rotary" in e.name]), 4)
                res[f"{arm}_kernels_per_token"] = round(len(kern) / steps, 1)
        else:
            for s in range(3, 3 + steps):
                for arm in ("bf16", "fp8"):
                    state[arm]["times"].append(step(arm, s))
            for arm in ("bf16", "fp8"):
                res[f"{arm}_ms_per_token" if w == 1 else f"{arm}_ms_per_step"] = stats(state[arm]["times"])
                res[f"{arm}_cache_mib"] = round(cache_bytes(state[arm]["cache"]) / 2 ** 20, 1)
            res["speedup"] = round(statistics.median(state["bf16"]["times"]) / statistics.median(state["fp8"]["times"]),
                                   3)
    del state, model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--per-round", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--rows", default="5,8,16,32,64,65", help="query rows of the multi-row leg ('' to skip it)")
    ap.add_argument("--rows-rounds", type=int, default=10)
    ap.add_argument("--rows-per-round", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dry-run", action="store_true")
    ap.add_argument("--profile", action="store_true", help="trace the model steps instead of timing them")
    a = ap.parse_args()
    if a.dry_run:
        c = GIANTMIDI["num_channels"]
        per_seq = (GIANTMIDI["max_seq_len"] + GIANTMIDI["max_latents"] * GIANTMIDI["num_self_attention_layers"]) * 2 * c
        print(json.dumps({"core_bytes_bf16": B * L * 2 * C * 2, "core_bytes_fp8": B * L * 2 * C,
                          "giantmidi_cache_bytes_per_sequence_bf16": per_seq * 2,
                          "giantmidi_cache_bytes_per_sequence_fp8": per_seq, "batches": a.batches,
                          "multirow_rows": [int(r) for r in a.rows.split(",") if r],
                          "multirow_bytes_bf16": B * L * 2 * C * 2, "multirow_bytes_fp8": B * L * 2 * C,
                          "multirow_route": {r: ("pcv_attn_cached_fp8" if 4 < int(r) <= modules.KV8_MAX_ROWS
                                                 else "dequantise" if int(r) > modules.KV8_MAX_ROWS
                                                 else "pcv_attn_decode_fp8") for r in a.rows.split(",") if r},
                          "model_steps": {"new_tokens": [1, 16]}}))
        return
    assert torch.cuda.is_available(), "fp8_kv_bench measures on a GPU"
    if a.profile:
        res = {"card": card(), "step_profile": [step_latency(int(b), a.steps, True) for b in a.batches.split(",")]}
    else:
        rows = [int(r) for r in a.rows.split(",") if r]
        res = {"card": card(), "core": core(a.rounds, a.per_round),
               "multirow": multirow(rows, a.rows_rounds, a.rows_per_round) if rows else [],
               "step": [step_latency(int(b), a.steps) for b in a.batches.split(",")],
               "step16": [step_latency(int(b), a.steps, new_tokens=16) for b in a.batches.split(",")]}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
