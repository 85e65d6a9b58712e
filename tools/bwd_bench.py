"""Times the attention backward at the north-star shape: tcgen05 kernels (pcv_attn_bwd) vs the torch shim.
Run on the GPU box: python tools/bwd_bench.py [--shim] [--M 65536]

--compare times the backward alone, kernels against the shim, alternating the two step by step (median of --steps
after warm-up), at any head dims (--dqk / --dv, odd ones padded as in training) and with attention dropout
(--dropout p); it prints the card's name and power limit and the per-kernel times of one kernel backward.
  python tools/bwd_bench.py --compare --B 64 --N 256 --M 2048 --H 8 --dqk 32 --dv 160 --steps 20"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from perceiver_io_b200 import _lib, ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--N", type=int, default=512)
    ap.add_argument("--M", type=int, default=65536)
    ap.add_argument("--H", type=int, default=8)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--dqk", type=int, default=None, help="qk head dim (--compare; default --d)")
    ap.add_argument("--dv", type=int, default=None, help="v head dim (--compare; default --d)")
    ap.add_argument("--dropout", type=float, default=0.0, help="attention dropout p (--compare)")
    ap.add_argument("--compare", action="store_true", help="backward only: kernels vs shim, alternating")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--shim", action="store_true", help="also time the torch shim (slow)")
    ap.add_argument("--per-batch-q", action="store_true", help="q of shape (B, N, C) instead of one latent array shared by the batch")
    ap.add_argument("--no-flush", action="store_true", help="back-to-back calls, no L2 flush in between")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.compare:
        return compare(a)
    B, N, M, H, d = a.B, a.N, a.M, a.H, a.d
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(B if a.per_batch_q else 1, N, H * d, device="cuda", generator=g).to(torch.bfloat16)
    k = torch.randn(B, M, H * d, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn(B, M, H * d, device="cuda", generator=g).to(torch.bfloat16)
    go = torch.randn(B, N, H * d, device="cuda", generator=g).to(torch.bfloat16)
    scale = d ** -0.5
    po, pm, pl = ops.attention_partial(q, k, v, H, scale)
    out = ops.combine_partials(po[None], pm[None], pl[None], q.dtype)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def timed(fn, steps):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(steps):
            if not a.no_flush:
                flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts) // 2]

    flops_fwd = 4.0 * B * N * M * H * d
    res = {"shape": {"B": B, "N": N, "M": M, "H": H, "d": d}, "flops_fwd": flops_fwd, "flops_bwd": 2.5 * flops_fwd}
    res["fwd_ms"] = timed(lambda: ops.attention_partial(q, k, v, H, scale), a.steps)
    n0 = _lib.launch_count()
    res["bwd_kernel_ms"] = timed(lambda: ops.attention_backward(q, k, v, out, go, pm, pl, H, scale), a.steps)
    res["bwd_launches_per_call"] = (_lib.launch_count() - n0) / (a.steps + 3)
    res["bwd_kernel_tflops_algorithmic"] = 2.5 * flops_fwd / res["bwd_kernel_ms"] * 1e-9
    res["bwd_kernel_tflops_executed"] = 3.5 * flops_fwd / res["bwd_kernel_ms"] * 1e-9
    # training step with attention dropout 0.1: the dropout forward, the backward regenerating the mask
    res["fwd_dropout_pass_ms"] = timed(
        lambda: ops.attention_dropout_forward(q, k, v, pm, pl, H, scale, 0.1, 1234), a.steps)
    res["bwd_dropout_kernel_ms"] = timed(
        lambda: ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, dropout_p=0.1, dropout_seed=1234), a.steps)
    if a.shim:
        qq, kk, vv = (t.detach().clone().requires_grad_() for t in (q, k, v))

        def shim():
            ops.backward_config["impl"] = "shim"
            try:
                o = ops.attention(qq, kk, vv, H, scale)
                o.backward(go)
            finally:
                ops.backward_config["impl"] = "auto"
            qq.grad = kk.grad = vv.grad = None

        res["fwd_plus_shim_bwd_ms"] = timed(shim, 3)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


class _Ctx:
    """The saved state of an ``ops._FusedAttention`` forward, to run its backward alone."""


def compare(a):
    from dropout_bench import card_info

    dqk, dv = a.dqk or a.d, a.dv or a.d
    B, N, M, H, p = a.B, a.N, a.M, a.H, a.dropout
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(B if a.per_batch_q else 1, N, H * dqk, device="cuda", generator=g).to(torch.bfloat16)
    k = torch.randn(B, M, H * dqk, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn(B, M, H * dv, device="cuda", generator=g).to(torch.bfloat16)
    go = torch.randn(B, N, H * dv, device="cuda", generator=g).to(torch.bfloat16)
    scale = dqk ** -0.5
    qq, kk, vv = (t.detach().clone().requires_grad_() for t in (q, k, v))
    # the forward of a training step; its saved tensors feed both backward paths
    fn = ops._FusedAttention
    ctx = _Ctx()
    with torch.no_grad():
        ctx.save_for_backward = lambda *t: setattr(ctx, "saved_tensors", t)
        fn.forward(ctx, qq, kk, vv, H, scale, None, False, "auto", p, 1234)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def backward(mode):
        ops.backward_config["impl"] = mode
        try:
            fn.backward(ctx, go)
        finally:
            ops.backward_config["impl"] = "auto"

    def one(mode):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        backward(mode)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for _ in range(3):
        backward("kernel")
        backward("shim")
    ts = {"kernel": [], "shim": []}
    for i in range(a.steps):
        for mode in (("kernel", "shim") if i % 2 == 0 else ("shim", "kernel")):
            ts[mode].append(one(mode))
    med = {m: sorted(t)[len(t) // 2] for m, t in ts.items()}
    flops = 4.0 * B * N * M * H * (dqk + dv) / 2  # forward QK^T + PV: 2*N*M*(dqk + dv) per (b, h)
    res = {"card": card_info(), "shape": {"B": B, "N": N, "M": M, "H": H, "dqk": dqk, "dv": dv, "q_batch": q.shape[0],
           "dropout": p}, "steps": a.steps, "bwd_kernel_ms": med["kernel"], "bwd_shim_ms": med["shim"],
           "speedup": med["shim"] / med["kernel"],
           "bwd_kernel_tflops_algorithmic": 2.5 * flops / med["kernel"] * 1e-9,
           "kernel_ms_range": [min(ts["kernel"]), max(ts["kernel"])], "shim_ms_range": [min(ts["shim"]), max(ts["shim"])]}
    # per-kernel device time of one kernel backward (the dK/dV passes, the dQ kernel, the prep and sum kernels)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        backward("kernel")
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "bwd" in ev.name:
            short = ev.name.replace("(anonymous namespace)::", "").split("(")[0].split("::")[-1]
            per[short] = per.get(short, 0.0) + ev.device_time / 1000.0
    res["kernel_ms_by_name"] = per
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
