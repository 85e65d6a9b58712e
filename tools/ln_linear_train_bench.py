"""Training cost of the LayerNorm -> Linear chain: the fused route (ops.ln_linear: pcv_ln_stats + the fused producer
forward, pcv_ln_linear_bwd backward) against ATen (nn.LayerNorm + two nn.Linear), alternating step by step.

For each shape it times (CUDA events, medians over --steps alternating steps after --warmup):
  - the chain alone, forward + backward (grad of x, W, b, gamma, beta);
  - one CrossAttention training step (forward + backward) with ``kv_producer_config["training"]`` on and off;
and reports the peak ``max_memory_allocated`` of each, per-kernel device times of one fused chain step
(torch.profiler, a separate pass), and the card name and power limit read in the same run.  One JSON line.

usage: python tools/ln_linear_train_bench.py [--steps 10] [--warmup 3] [--shapes north_star,mlm]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import perceiver_io_b200 as P  # noqa: E402
from perceiver_io_b200 import modules, ops  # noqa: E402

SHAPES = {  # (B, M, C, n_k, n_v, latents N)
    "north_star": (8, 65536, 1024, 1024, 1024, 512),
    "mlm": (64, 2048, 768, 256, 1280, 256),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, pl = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit_w": float(pl)}


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), torch.cuda.max_memory_allocated() - base


def alternate(fns, steps, warmup):
    res = {k: ([], []) for k in fns}
    for i in range(warmup + steps):
        for k, fn in fns.items():
            ms, mem = timed(fn)
            if i >= warmup:
                res[k][0].append(ms)
                res[k][1].append(mem)
    return {k: {"ms": round(statistics.median(v[0]), 3), "peak_mib": round(max(v[1]) / 2 ** 20, 1)} for k, v in res.items()}


def kernel_times(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t > 0:
            out[e.key[:60]] = round(t / 1000.0, 3)
    return dict(sorted(out.items(), key=lambda kv: -kv[1])[:12])


def chain_case(B, M, C, n_k, n_v):
    dt, dev = torch.bfloat16, "cuda"
    x = torch.randn(B * M, C, device=dev, dtype=dt)
    norm = torch.nn.LayerNorm(C).to(dev, dt)
    k_proj, v_proj = torch.nn.Linear(C, n_k).to(dev, dt), torch.nn.Linear(C, n_v).to(dev, dt)
    gk = torch.randn(B * M, n_k, device=dev, dtype=dt)
    gv = torch.randn(B * M, n_v, device=dev, dtype=dt)
    params = list(norm.parameters()) + list(k_proj.parameters()) + list(v_proj.parameters())

    def fused():
        xx = x.requires_grad_()
        k, v = ops.ln_linear(xx, norm.weight, norm.bias, [k_proj.weight, v_proj.weight], [k_proj.bias, v_proj.bias],
                             n_k, n_v, norm.eps)
        torch.autograd.backward([k, v], [gk, gv])
        for p in params + [xx]:
            p.grad = None

    def aten():
        xx = x.requires_grad_()
        y = norm(xx)
        torch.autograd.backward([k_proj(y), v_proj(y)], [gk, gv])
        for p in params + [xx]:
            p.grad = None

    return {"fused": fused, "aten": aten}


def module_case(B, M, C, N):
    dt, dev = torch.bfloat16, "cuda"
    layer = P.CrossAttention(num_heads=8, num_q_input_channels=C, num_kv_input_channels=C).to(dev, dt).train()
    x_q = torch.randn(1, N, C, device=dev, dtype=dt, requires_grad=True)
    x_kv = torch.randn(B, M, C, device=dev, dtype=dt, requires_grad=True)

    def step(on):
        def run():
            modules.kv_producer_config["training"] = on
            try:
                layer(x_q, x_kv).last_hidden_state.float().square().mean().backward()
            finally:
                modules.kv_producer_config["training"] = False
            layer.zero_grad(set_to_none=True)
            x_q.grad = x_kv.grad = None
        return run

    return {"fused": step(True), "aten": step(False)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default="north_star,mlm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ln_linear_train_bench needs a GPU")
    out = {"card": card(), "steps": args.steps, "cases": {}}
    for name in args.shapes.split(","):
        B, M, C, n_k, n_v, N = SHAPES[name]
        rows = B * M
        fns = chain_case(B, M, C, n_k, n_v)
        chain = alternate(fns, args.steps, args.warmup)
        flop = 3 * 2 * rows * C * (n_k + n_v)  # forward, dX and dW GEMMs
        for v in chain.values():
            v["gemm_tflops"] = round(flop / (v["ms"] * 1e-3) / 1e12, 1)
        chain["fused_kernels_ms"] = kernel_times(fns["fused"])
        chain["aten_kernels_ms"] = kernel_times(fns["aten"])
        del fns
        torch.cuda.empty_cache()
        mod = alternate(module_case(B, M, C, N), args.steps, args.warmup)
        torch.cuda.empty_cache()
        out["cases"][name] = {"shape": {"B": B, "M": M, "C": C, "n_k": n_k, "n_v": n_v, "rows": rows, "latents": N},
                              "chain_fwd_bwd": chain, "cross_attention_step": mod}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
