"""Times the key-shard backward (pcv_attn_bwd_shard) on one GPU against the unsharded backward (pcv_attn_bwd) and prints
one JSON line with the card's name and power limit.

For G in {2, 4, 8} the G shard backwards run one after another from the merged statistics, as the G ranks of a
key-sharded training step would run them in parallel; the sum of their times against the unsharded time is the cost of
sharding (per-shard statistics preparation, the dQ split into fp32 contributions).  Shapes: B=1, N=512, H=8, head dim
128, M in {65536, 262144} (bf16).  The unsharded and the sharded backward alternate step by step; medians of --steps.
Also reported: the bytes of the one dQ all-reduce per rank (fp32 (Bq, N, H*dqk)).  Multi-GPU wall time is not measured
here.

Run on the GPU box: python tools/shard_bwd_bench.py [--steps 20]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from perceiver_io_b200 import ops  # noqa: E402
from perceiver_io_b200.dist import shard_bounds  # noqa: E402
from tools.dropout_bench import card_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--M", type=int, nargs="*", default=[65536, 262144])
    ap.add_argument("--G", type=int, nargs="*", default=[2, 4, 8])
    a = ap.parse_args()
    B, N, H, d = 1, 512, 8, 128
    scale = d ** -0.5
    res = {"card": card_info(), "shape": {"B": B, "N": N, "H": H, "d": d, "dtype": "bf16"}, "cases": []}
    for M in a.M:
        g = torch.Generator(device="cuda").manual_seed(M)
        q = torch.randn(B, N, H * d, device="cuda", generator=g).bfloat16()
        k = torch.randn(B, M, H * d, device="cuda", generator=g).bfloat16()
        v = torch.randn(B, M, H * d, device="cuda", generator=g).bfloat16()
        go = torch.randn(B, N, H * d, device="cuda", generator=g).bfloat16()
        po, m, l = ops.attention_partial(q, k, v, H, scale)
        out = ops.combine_partials(po[None], m[None], l[None], q.dtype)
        del po

        def full():
            ops.attention_backward(q, k, v, out, go, m, l, H, scale)

        def sharded(G):
            def run():
                gq = torch.zeros(B, N, H * d, device="cuda")
                for r in range(G):
                    b, e = shard_bounds(M, G, r)
                    g32, _, _ = ops.attention_backward_shard(q, k[:, b:e], v[:, b:e], out, go, m, l, H, scale, M, b)
                    gq += g32  # stands in for the all-reduce
            return run

        fns = {"unsharded": full, **{f"G{G}": sharded(G) for G in a.G}}
        for fn in fns.values():  # warm-up of every shape
            fn()
            fn()
        torch.cuda.synchronize()
        times = {name: [] for name in fns}
        for _ in range(a.steps):
            for name, fn in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1))
        base = statistics.median(times["unsharded"])
        case = {"M": M, "unsharded_ms": round(base, 3), "dq_allreduce_bytes": 4 * B * N * H * d, "shards": {}}
        for G in a.G:
            t = statistics.median(times[f"G{G}"])
            case["shards"][G] = {"sum_of_shards_ms": round(t, 3), "overhead_pct": round(100.0 * (t / base - 1.0), 1),
                                 "per_shard_ms": round(t / G, 3)}
        res["cases"].append(case)
        del q, k, v, go, out
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
