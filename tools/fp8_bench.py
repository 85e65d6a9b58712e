"""Times the FP8 attention forward (ops.attention_fp8) against the bf16 one (ops.attention) on one GPU, operands
resident, the two alternating step by step; prints one JSON line with the card, its power limit, per-shape medians and
spread, TFLOP/s and the error of each against exact fp64 attention on the unquantised operands (a few query rows).

usage: python tools/fp8_bench.py [--steps 20] [--warmup 3]"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import perceiver_io_b200 as P  # noqa: E402
from perceiver_io_b200 import modules, ops  # noqa: E402


def amax_descale(x, H, per_channel=False):
    a = x.float().abs().reshape(-1, H, x.shape[-1] // H).amax(dim=0)
    return ((a if per_channel else a.amax(dim=1)) / ops.E4M3_MAX).clamp_min(1e-12)

SHAPES = {
    # name: (B, Bq, N, M, H, dqk, dv); the north-star core has one q per batch row, as bench.py's core leg
    "north_star_core": (8, 8, 512, 65536, 8, 128, 128),
    "mlm_encoder_cross": (64, 1, 256, 2048, 8, 32, 160),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        pl, clk = (float(x) for x in out.split(","))
    except Exception:  # noqa: BLE001 - the card name still identifies the run
        pl, clk = None, None
    return {"name": name, "power_limit_w": pl, "max_sm_clock_mhz": clk}


def exact_rows(q, k, v, H, scale, rows):
    """fp64 attention of query rows `rows` (q batch 1) for every batch and head: (B, len(rows), H*dv)."""
    B, M, _ = k.shape
    dqk, dv = q.shape[2] // H, v.shape[2] // H
    out = []
    for b in range(B):
        qh = q[b if q.shape[0] > 1 else 0, rows].double().view(len(rows), H, dqk).transpose(0, 1)  # (H, r, dqk)
        kh = k[b].double().view(M, H, dqk).transpose(0, 1)
        vh = v[b].double().view(M, H, dv).transpose(0, 1)
        p = torch.softmax((qh @ kh.transpose(-1, -2)) * scale, dim=-1)
        out.append((p @ vh).transpose(0, 1).reshape(len(rows), H * dv))
    return torch.stack(out)


def run_shape(B, Bq, N, M, H, dqk, dv, steps, warmup, peaked):
    g = torch.Generator(device="cuda").manual_seed(0)
    amp = 4.0 if peaked else 1.0
    q = (torch.randn(Bq, N, H * dqk, device="cuda", generator=g) * amp).bfloat16()
    k = (torch.randn(B, M, H * dqk, device="cuda", generator=g) * amp).bfloat16()
    v = torch.randn(B, M, H * dv, device="cuda", generator=g).bfloat16()
    qd, kd, vd = amax_descale(q, H), amax_descale(k, H), amax_descale(v, H, per_channel=True)
    q8, k8 = ops.fp8_quantize(q, qd, H), ops.fp8_quantize(k, kd, H)
    vt8 = ops.fp8_transpose_v(ops.fp8_quantize(v, vd, H), H)
    scale = dqk ** -0.5
    calls = {"bf16": lambda: ops.attention(q, k, v, H, scale),
             "fp8": lambda: ops.attention_fp8(q8, k8, vt8, qd, kd, vd, H, scale)}
    times = {name: [] for name in calls}
    with torch.no_grad():
        for _ in range(warmup):
            for fn in calls.values():
                fn()
        for _ in range(steps):
            for name, fn in calls.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                b.synchronize()
                times[name].append(a.elapsed_time(b))
        rows = torch.linspace(0, N - 1, 8).long().tolist()
        ref = exact_rows(q, k, v, H, scale, rows)
        errs = {}
        for name, fn in calls.items():
            out = fn()[:, rows].double()
            errs[name] = (out - ref).abs().max().item() / ref.abs().max().item()
    flops = 2.0 * B * H * N * M * (dqk + dv)
    res = {}
    for name, t in times.items():
        t = sorted(t)
        med = t[len(t) // 2]
        res[name] = {"median_ms": round(med, 4), "min_ms": round(t[0], 4), "max_ms": round(t[-1], 4),
                     "tflops": round(flops / med / 1e9, 1), "max_err_rel": float(f"{errs[name]:.3e}")}
    res["speedup"] = round(res["bf16"]["median_ms"] / res["fp8"]["median_ms"], 3)
    return res


def run_module(steps, warmup):
    """The north-star CrossAttention.forward (B=8, M=65536, N=512, d=1024, H=8, batch-1 latents, device-resident,
    no_grad), bf16 route against modules.fp8_config["enabled"], alternating; error of each against the fp64 module."""
    B, N, M, D, H = 8, 512, 65536, 1024, 8
    torch.manual_seed(0)
    layer = P.CrossAttention(num_heads=H, num_q_input_channels=D, num_kv_input_channels=D).cuda().bfloat16().eval()
    x_q = torch.randn(1, N, D, device="cuda").bfloat16()
    x_kv = torch.randn(B, M, D, device="cuda").bfloat16()
    def call(fp8):
        modules.fp8_config["enabled"] = fp8
        try:
            return layer(x_q, x_kv).last_hidden_state
        finally:
            modules.fp8_config["enabled"] = False
    times = {"bf16": [], "fp8": []}
    with torch.no_grad():
        for _ in range(warmup):
            call(False), call(True)
        for _ in range(steps):
            for name in times:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                call(name == "fp8")
                b.record()
                b.synchronize()
                times[name].append(a.elapsed_time(b))
        outs = {name: call(name == "fp8")[:1, ::64].double() for name in times}
        # fp64 module on batch row 0, every 64th query
        lay64 = P.CrossAttention(num_heads=H, num_q_input_channels=D, num_kv_input_channels=D).cuda().double().eval()
        lay64.load_state_dict({k: v.double() for k, v in layer.state_dict().items()})
        modules.kv_producer_config["enabled"] = False
        q = lay64.attention.q_proj(lay64.q_norm(x_q.double()))[:, ::64]
        kv = lay64.kv_norm(x_kv[:1].double())
        k, v = lay64.attention.k_proj(kv), lay64.attention.v_proj(kv)
        modules.kv_producer_config["enabled"] = True
        sp = lambda t: t.view(t.shape[0], t.shape[1], H, -1).transpose(1, 2)
        p = torch.softmax(sp(q) @ sp(k).transpose(-1, -2) * lay64.attention.dp_scale, dim=-1)
        ref = lay64.attention.o_proj((p @ sp(v)).transpose(1, 2).reshape(1, q.shape[1], D))
    res = {}
    for name, t in times.items():
        t = sorted(t)
        res[name] = {"median_ms": round(t[len(t) // 2], 3), "min_ms": round(t[0], 3), "max_ms": round(t[-1], 3),
                     "max_err_rel": float(f"{((outs[name] - ref).abs().max() / ref.abs().max()).item():.3e}")}
    res["speedup"] = round(res["bf16"]["median_ms"] / res["fp8"]["median_ms"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fp8_bench needs a GPU"
    result = {"card": card(), "steps": args.steps, "shapes": {}}
    for name, shp in SHAPES.items():
        for peaked in (False, True):
            result["shapes"][f"{name}{'_peaked' if peaked else ''}"] = {
                "B,Bq,N,M,H,dqk,dv": list(shp), **run_shape(*shp, args.steps, args.warmup, peaked)}
            torch.cuda.empty_cache()
    result["north_star_cross_attention_forward"] = run_module(args.steps, args.warmup)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
