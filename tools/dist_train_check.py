"""Multi-GPU training check (run under torchrun, one rank per GPU, NCCL): a cross_attention_sharded training step with
attention dropout, then reduce_shard_grads, gives every CrossAttention parameter the gradient of the one-GPU
CrossAttention step.

- Key shards over all ranks (B = 1 latent batch row against B = 2 inputs: plan_grid(1, world) = (1, world)).
- With 4 or more ranks also the rank grid of plan_grid(2, world): 2 batch groups, each sharding the keys over its own
  process sub-group (m_shard_group); each group is compared with the one-GPU step on its own batch row.
The seed is drawn on the group's first rank and broadcast; every rank's one-GPU reference draws the same seed from the
same CPU generator state.  Exercises the seed broadcast, the fp32 dQ all-reduce, the per-parameter all-reduces of
reduce_shard_grads and the grid sub-groups on NCCL.
  torchrun --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29535 tools/dist_train_check.py"""
import copy
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import perceiver_io_b200 as P  # noqa: E402
from perceiver_io_b200.dist import (cross_attention_sharded, grid_position, m_shard_group, plan_grid,  # noqa: E402
                                    reduce_shard_grads, shard_bounds)

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
H, D, C, N, M = 8, 512, 256, 128, 8192


def shard_params(mod):
    a = mod.attention
    return [*mod.kv_norm.parameters(), *a.k_proj.parameters(), *a.v_proj.parameters()]


def step(mod, x_q, x_kv, pad, go, sharded, group=None, m_shards=1, shard=0):
    mod.zero_grad(set_to_none=True)
    torch.manual_seed(1234)  # the dropout seed: drawn on the group's first rank (sharded) or locally (reference)
    if sharded:
        m0, m1 = shard_bounds(M, m_shards, shard)
        out = cross_attention_sharded(mod, x_q, x_kv[:, m0:m1], M, m0, pad[:, m0:m1], group=group).last_hidden_state
    else:
        out = mod(x_q, x_kv, pad_mask=pad).last_hidden_state
    out.backward(go)
    if sharded:
        reduce_shard_grads(shard_params(mod), group)
    return out.detach().float(), {n: p.grad.float() if p.grad is not None else None for n, p in mod.named_parameters()}


def compare(what, a, b):
    """-> (ok, worst err / bound).  bf16 parameters and gradients, keys summed in a different order: 3e-2 of max|ref|.
    k_proj.bias has an exact gradient of 0 (a key bias shifts each row's scores by a constant): it is held to the scale
    of the k_proj weight gradient."""
    out_a, g_a = a
    out_b, g_b = b
    worst = (out_a - out_b).abs().max().item() / (3e-2 * out_b.abs().max().item())
    for name, ref in g_b.items():
        got = g_a[name]
        if got is None:
            print(f"rank {rank} {what}: {name} has no gradient")
            return False, float("inf")
        scale = g_b["attention.k_proj.weight"] if name == "attention.k_proj.bias" else ref
        worst = max(worst, (got - ref).abs().max().item() / (3e-2 * scale.abs().max().item() + 1e-6))
    return worst <= 1.0, worst


torch.manual_seed(0)
mod = P.CrossAttention(num_heads=H, num_q_input_channels=D, num_kv_input_channels=C, dropout=0.1)
mod = mod.to(dev).bfloat16().train()
ref_mod = copy.deepcopy(mod)
g = torch.Generator().manual_seed(3)
x_q = torch.randn(1, N, D, generator=g).bfloat16().to(dev)
x_kv = torch.randn(2, M, C, generator=g).bfloat16().to(dev)
go = torch.randn(2, N, D, generator=g).bfloat16().to(dev)
pad = torch.zeros(2, M, dtype=torch.bool)
pad[1, 6000:] = True
pad = pad.to(dev)
ok = True

# key shards over every rank
bg, mg = plan_grid(1, world)
res = step(mod, x_q, x_kv, pad, go, True, m_shard_group(bg, mg), mg, grid_position(rank, bg, mg)[1])
good, worst = compare("key shards", res, step(ref_mod, x_q, x_kv, pad, go, False))
flags = torch.tensor([1.0 if good else 0.0, worst], device=dev)
dist.all_reduce(flags[:1], op=dist.ReduceOp.MIN)
dist.all_reduce(flags[1:], op=dist.ReduceOp.MAX)
if rank == 0:
    print(f"{world} key shards: every parameter gradient within the gate on all ranks: {bool(flags[0])}, worst "
          f"err/bound {flags[1].item():.3f}")
ok = ok and bool(flags[0])

# the rank grid: 2 batch groups x (world / 2) key shards, each group on its own sub-group
if world >= 4:
    bg, mg = plan_grid(2, world)
    gb, gm = grid_position(rank, bg, mg)
    group = m_shard_group(bg, mg)
    rows = slice(gb, gb + 1)
    res = step(mod, x_q, x_kv[rows], pad[rows], go[rows], True, group, mg, gm)
    good, worst = compare("grid", res, step(ref_mod, x_q, x_kv[rows], pad[rows], go[rows], False))
    flags = torch.tensor([1.0 if good else 0.0, worst], device=dev)
    dist.all_reduce(flags[:1], op=dist.ReduceOp.MIN)
    dist.all_reduce(flags[1:], op=dist.ReduceOp.MAX)
    if rank == 0:
        print(f"grid {bg} batch groups x {mg} key shards: every parameter gradient within the gate on all ranks: "
              f"{bool(flags[0])}, worst err/bound {flags[1].item():.3f}")
    ok = ok and bool(flags[0])

dist.barrier()
if rank == 0:
    print("DIST_TRAIN_CHECK", "OK" if ok else "FAILED")
dist.destroy_process_group()
sys.exit(0 if ok else 1)
