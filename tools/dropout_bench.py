"""Times the attention-dropout training paths and prints one JSON line (with the card's name and power limit):

- north-star shape (B=8, N=512, M=65536, H=8, head dim 128): the dropout-free partial forward, the dropout forward
  (attention_partial with dropout_p) and the dropout backward on the tensor-core kernels;
- the masked-LM recipe's encoder cross-attention (B=64, N=256, M=2048, H=8, head dims 32 / 160): the dropout-free
  partial forward, the dropout forward and the backward under autograd.

Run on the GPU box: python tools/dropout_bench.py [--steps 20] [--p 0.1]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from perceiver_io_b200 import ops  # noqa: E402


def timed(fn, steps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def card_info():
    """Name and power limit of the card: a timing means little without them."""
    info = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        info["power_limit_w"] = float(out.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def operands(Bq, B, N, M, H, dqk, dv, seed, grad=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(Bq, N, H * dqk, device="cuda", generator=g).bfloat16()
    k = torch.randn(B, M, H * dqk, device="cuda", generator=g).bfloat16()
    v = torch.randn(B, M, H * dv, device="cuda", generator=g).bfloat16()
    go = torch.randn(B, N, H * dv, device="cuda", generator=g).bfloat16()
    if grad:
        q, k, v = (t.requires_grad_() for t in (q, k, v))
    return q, k, v, go


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--p", type=float, default=0.1)
    a = ap.parse_args()
    p, seed = a.p, 1234
    res = {"card": card_info(), "dropout_p": p}

    B, N, M, H, d = 8, 512, 65536, 8, 128
    q, k, v, go = operands(B, B, N, M, H, d, d, 0)
    scale = d ** -0.5
    po, pm, pl = ops.attention_partial(q, k, v, H, scale)
    out = ops.combine_partials(po[None], pm[None], pl[None], torch.bfloat16)
    del po
    res["north_star"] = {
        "shape": {"B": B, "N": N, "M": M, "H": H, "dqk": d, "dv": d},
        "partial_forward_ms": timed(lambda: ops.attention_partial(q, k, v, H, scale), a.steps),
        "dropout_forward_ms": timed(lambda: ops.attention_partial(q, k, v, H, scale, dropout_p=p, dropout_seed=seed),
                                    a.steps),
        "backward_kernels_ms": timed(lambda: ops.attention_backward(q, k, v, out, go, pm, pl, H, scale, dropout_p=p,
                                                                    dropout_seed=seed), a.steps),
    }
    del q, k, v, go, out, pm, pl

    B, N, M, H, dqk, dv = 64, 256, 2048, 8, 32, 160
    q, k, v, go = operands(1, B, N, M, H, dqk, dv, 3, grad=True)
    scale = dqk ** -0.5
    with torch.no_grad():
        ms_part = timed(lambda: ops.attention_partial(q, k, v, H, scale), a.steps)
        ms_drop = timed(lambda: ops.attention_partial(q, k, v, H, scale, dropout_p=p, dropout_seed=seed), a.steps)
    out = ops.attention(q, k, v, H, scale, dropout_p=p, dropout_seed=seed)
    res["mlm_encoder_cross_attention"] = {
        "shape": {"B": B, "N": N, "M": M, "H": H, "dqk": dqk, "dv": dv},
        "partial_forward_ms": ms_part, "dropout_forward_ms": ms_drop,
        "backward_ms": timed(lambda: out.backward(go, retain_graph=True), a.steps),
    }
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
