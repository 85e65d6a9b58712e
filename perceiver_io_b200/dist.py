"""M-sharded latent cross-attention across the GPUs of one box (SURVEY.md §8(e)).

The key/value axis M is the only axis that shards naturally when N << M: rank g holds keys
[m_offset, m_offset + M_g) of ``m_total`` (and the matching slice of ``pad_mask``), computes the
partial softmax state of ALL B*H*N query rows over its keys with the fused kernel
(``pcv_attn_fwd`` with ``write_partial``), and the ranks merge:

    m  = max_g m_g                               all_reduce(MAX) on (B,H,N) floats        131 KB
    Õ_g, l_g *= 2^(m_g - m)                      pcv_partial_rescale (in place)
    [Õ ‖ l] = sum_g [Õ_g ‖ l_g]                  ONE all_reduce(SUM) over NVLink/NVSwitch  ~17 MB
    out = Õ / l                                  pcv_attn_combine (num_parts = 1)

Q, the projection weights and everything after the merge (o_proj, MLP, the latent self-attention
stack) are replicated: no further communication.  The reference has no counterpart (its only
multi-GPU modes are DDP/FSDP replicas, SURVEY.md §2.1).

Two merge transports exist.  ``merge="nccl"`` is the protocol above on ``torch.distributed`` collectives.
``merge="peer"`` (default on GPUs when symmetric memory can be set up) keeps NCCL off the data path: every rank
writes its partial state into a symmetric-memory buffer (``torch.distributed._symmetric_memory``: cuMem
allocations mapped into every peer over NVLink/NVSwitch), a signal-pad barrier publishes them, and ONE kernel
per rank (``pcv_attn_combine_peers``) loads the rows it owns from all peers through their mapped pointers,
merges them exactly, and stores the normalised rows into EVERY rank's output buffer; a second barrier publishes
the result.  Per rank that is (G-1)/G * 17 MB of NVLink reads and (G-1)/G * 8 MB of NVLink writes, versus two
NCCL collectives plus two extra kernels.

The communication backend is whatever ``torch.distributed`` group is passed (NCCL on GPUs).  The
device math is injectable (``ShardKernels``) so the host-side protocol is testable with ``gloo`` on
CPU boxes (tests/test_dist_cpu.py injects the oracle's math); the default is the CUDA path and
nothing else.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Optional, Tuple

import torch
import torch.distributed as dist


def plan_grid(batch: int, world_size: int) -> Tuple[int, int]:
    """(batch_groups, m_shards) with batch_groups * m_shards == world_size: ranks are spent on the batch axis first.

    Batch rows are independent — sharding them needs no exchange at all — while every extra M shard adds a partial
    softmax state to merge (17 MB per rank at the north-star shape).  So the batch axis takes the largest divisor of
    ``world_size`` that also divides ``batch``; only the remaining factor shards the key axis.  B=8 on 8 GPUs is
    (8, 1): one batch row per GPU, no collective; B=1 on 8 GPUs is (1, 8): the pure M-shard layout of SURVEY.md §8(e)."""
    if batch < 1 or world_size < 1:
        raise ValueError("batch and world_size must be positive")
    bg = 1
    for cand in range(1, world_size + 1):
        if world_size % cand == 0 and batch % cand == 0:
            bg = cand
    return bg, world_size // bg


def grid_position(rank: int, batch_groups: int, m_shards: int) -> Tuple[int, int]:
    """(batch group, M shard) of ``rank``: the ranks of one batch group are consecutive (they merge with each other)."""
    if not 0 <= rank < batch_groups * m_shards:
        raise ValueError("rank outside the grid")
    return rank // m_shards, rank % m_shards


def m_shard_group(batch_groups: int, m_shards: int):
    """The calling rank's process sub-group for the M-shard merge of its batch group (``None`` when there is nothing to
    merge or the whole world is one group).  Collective: every rank must call it (``dist.new_group`` semantics)."""
    if m_shards == 1 or not dist.is_initialized():
        return None
    if batch_groups == 1:
        return dist.group.WORLD
    mine = None
    rank = dist.get_rank()
    for gb in range(batch_groups):
        ranks = list(range(gb * m_shards, (gb + 1) * m_shards))
        g = dist.new_group(ranks)
        if rank in ranks:
            mine = g
    return mine


def shard_bounds(m_total: int, world_size: int, rank: int, align: int = 128) -> Tuple[int, int]:
    """Contiguous [begin, end) slice of the key axis owned by ``rank``: equal counts of ``align``-key
    tiles, remainder tiles to the lowest ranks, the ragged tail to the last non-empty rank."""
    tiles = (m_total + align - 1) // align
    base, extra = divmod(tiles, world_size)
    first_tile = rank * base + min(rank, extra)
    n_tiles = base + (1 if rank < extra else 0)
    begin = min(first_tile * align, m_total)
    end = min((first_tile + n_tiles) * align, m_total)
    return begin, end


def _cuda_partial(q, k, v, num_heads, scale, pad_mask, causal, m_total, m_offset, out):
    from . import ops

    return ops.attention_partial(q, k, v, num_heads, scale, pad_mask=pad_mask, causal=causal, m_total=m_total,
                                 m_offset=m_offset, out=out)


def _cuda_rescale(po, pm, pl, new_m):
    from . import ops

    ops.rescale_partial_(po, pm, pl, new_m)


def _cuda_finalize(po, pl, out_dtype):
    from . import ops

    return ops.combine_partials(po[None], torch.zeros_like(pl)[None], pl[None], out_dtype)


def _cuda_partial_dropout(q, k, v, num_heads, scale, pad_mask, causal, m_total, m_offset, out, dropout_p, dropout_seed):
    """The one-pass dropout forward on the local keys (global key indices in the mask).  Head dims that are not
    multiples of 8 are zero-padded as in ``ops._prep``, and the caller's buffers get the true head dim back."""
    from . import ops

    q, k, v, dims = ops._prep(q, k, v, num_heads=num_heads, pad=True)
    state = ops.attention_partial(q, k, v, num_heads, scale, pad_mask=pad_mask, causal=causal, m_total=m_total,
                                  m_offset=m_offset, out=None if dims else out, dropout_p=dropout_p,
                                  dropout_seed=dropout_seed)
    if dims is not None:
        po, pm, pl = state
        for dst, src in zip(out, (ops._unpad_heads(po, num_heads, dims[1]), pm, pl)):
            dst.copy_(src)


def _cuda_backward(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal, m_total, m_offset,
                   dropout_p, dropout_seed):
    """-> (grad_q32, grad_k, grad_v) of one key shard: the backward kernels where they cover the call, else (head dims
    above 192, 4-D operands) the torch shim with the key offset, as ``ops.backward_config["impl"]`` selects."""
    from . import ops

    return ops._attention_grads(q, k, v, out, grad_out, stat_m, stat_l, num_heads, scale, pad_mask, causal, dropout_p,
                                dropout_seed, shard=(m_total, m_offset))


@dataclass
class ShardKernels:
    """Device math of the sharded path; the defaults are the sm_90a kernels.

    ``partial_dropout`` is ``partial`` with two more arguments (dropout_p, dropout_seed); ``backward`` maps (q, k_shard,
    v_shard, out, grad_out, m_glob, l_glob, num_heads, scale, pad_mask_shard, causal, m_total, m_offset, dropout_p,
    dropout_seed) to (grad_q32, grad_k, grad_v), grad_q32 being the shard's fp32 contribution to grad_q."""
    partial: Callable = _cuda_partial
    rescale_: Callable = _cuda_rescale
    finalize: Callable = _cuda_finalize
    partial_dropout: Callable = _cuda_partial_dropout
    backward: Callable = _cuda_backward


class PeerMerger:
    """Symmetric-memory state of the peer-to-peer merge for one (group, shape): the partial-state buffer
    [Õ | m | l] and the output buffer, both mapped into every rank of the group."""

    _cache = {}
    disabled = False  # set when symmetric memory could not be set up; "auto" then stays on NCCL

    def __init__(self, B, H, N, dv, dtype, device, group):
        import torch.distributed._symmetric_memory as symm_mem

        self.B, self.H, self.N, self.dv, self.dtype = B, H, N, dv, dtype
        rows = B * H * N
        self.rows = rows
        group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        if self.world > 8:
            raise RuntimeError("peer merge supports up to 8 ranks (one NVSwitch domain)")
        self.part = symm_mem.empty(rows * dv + 2 * rows, dtype=torch.float32, device=device)
        self.part_hdl = symm_mem.rendezvous(self.part, group)
        self.out = symm_mem.empty(B * N * H * dv, dtype=dtype, device=device)
        self.out_hdl = symm_mem.rendezvous(self.out, group)
        self.po = self.part[: rows * dv].view(B, H, N, dv)
        self.pm = self.part[rows * dv: rows * dv + rows].view(B, H, N)
        self.pl = self.part[rows * dv + rows:].view(B, H, N)
        self.part_ptrs = [int(p) for p in self.part_hdl.buffer_ptrs]
        self.out_ptrs = [int(p) for p in self.out_hdl.buffer_ptrs]
        # flag block of the fused kernel-tail merge (pcv_attn_fwd_sharded): epochs, never reset
        self.flags = symm_mem.empty(64, dtype=torch.int32, device=device)
        self.flags.zero_()
        self.flags_hdl = symm_mem.rendezvous(self.flags, group)
        self.flag_ptrs = [int(p) for p in self.flags_hdl.buffer_ptrs]
        torch.cuda.synchronize(device)
        self.flags_hdl.barrier(channel=2)  # every rank's flags are zero before anybody's first kernel can write them
        self.epoch = 0
        # contiguous, equal row slices: rank r merges rows [r*R/G, (r+1)*R/G)
        self.row_begin = rows * self.rank // self.world
        self.row_end = rows * (self.rank + 1) // self.world

    @classmethod
    def get(cls, B, H, N, dv, dtype, device, group, tag=None):
        """``tag`` separates states whose kernels run with different grids (the fused tail counts CTA arrivals)."""
        key = (id(group), B, H, N, dv, dtype, str(device), tag)
        if key not in cls._cache:
            cls._cache[key] = cls(B, H, N, dv, dtype, device, group)
        return cls._cache[key]

    def fused_attention(self, q, k_shard, v_shard, num_heads, scale, m_total, m_offset, pad_mask_shard=None,
                        causal=False) -> torch.Tensor:
        """ONE kernel launch on this rank: partial state of the local key shard, then — in the same kernel — publish
        it, merge the rows this rank owns from all ranks over NVLink-mapped memory and push the normalised rows into
        every rank's output buffer.  Returns this rank's (complete) output buffer, valid until the next call."""
        from . import _lib, ops

        self.epoch += 1
        f = _lib.ShardFuse()
        for g in range(self.world):
            f.part[g], f.out[g], f.flags[g] = self.part_ptrs[g], self.out_ptrs[g], self.flag_ptrs[g]
        f.o_stride_b, f.o_stride_n, f.o_stride_h = self.N * self.H * self.dv, self.H * self.dv, self.dv
        f.num_peers, f.rank, f.epoch = self.world, self.rank, self.epoch
        ops.attention_sharded_fused(q, k_shard, v_shard, num_heads, scale, f, pad_mask=pad_mask_shard, causal=causal,
                                    m_total=m_total, m_offset=m_offset)
        return self.out.view(self.B, self.N, self.H * self.dv)

    def merge(self) -> torch.Tensor:
        """Partials (written into self.po/pm/pl by the local kernel) -> full normalised output on every rank."""
        import ctypes as C

        from . import _lib
        from .ops import _pcv_dtype, _stream

        self.part_hdl.barrier(channel=0)  # every rank's partial state is complete and visible
        p = _lib.PeerCombineParams()
        esz = 4
        for g in range(self.world):
            base = self.part_ptrs[g]
            p.part_o[g] = base
            p.part_m[g] = base + self.rows * self.dv * esz
            p.part_l[g] = base + (self.rows * self.dv + self.rows) * esz
            p.out[g] = self.out_ptrs[g]
        p.o_stride_b, p.o_stride_n, p.o_stride_h = self.N * self.H * self.dv, self.H * self.dv, self.dv
        p.row_begin, p.row_end = self.row_begin, self.row_end
        p.num_peers, p.rank = self.world, self.rank
        p.B, p.H, p.N, p.dv = self.B, self.H, self.N, self.dv
        p.dtype = _pcv_dtype(self.dtype)
        _lib.check(_lib.lib().pcv_attn_combine_peers(C.byref(p), _stream()), "pcv_attn_combine_peers")
        self.out_hdl.barrier(channel=1)   # every rank's output buffer has received all row slices
        return self.out.view(self.B, self.N, self.H * self.dv)


_warned = set()


def _warn_once(msg: str) -> None:
    if msg not in _warned:
        _warned.add(msg)
        import warnings

        warnings.warn(msg)


def _peer_merge_possible(t: torch.Tensor, world: int) -> bool:
    if not t.is_cuda or world < 2 or world > 8:
        return False
    try:
        import torch.distributed._symmetric_memory  # noqa: F401
    except Exception:  # noqa: BLE001
        return False
    return True


def _shared_dropout_seed(group, device) -> int:
    """A fresh dropout seed drawn on the group's first rank and broadcast (8 bytes), so that every shard drops with
    the same mask."""
    from . import ops

    seed = torch.tensor([ops.new_dropout_seed()], dtype=torch.int64, device=device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        g = group if group is not None else dist.group.WORLD
        dist.broadcast(seed, src=dist.get_global_rank(g, 0), group=g)
    return int(seed.item())


def _exact_merge(q, k_shard, v_shard, num_heads, scale, m_total, m_offset, pad_mask_shard, causal, group, kernels,
                 dropout_p, dropout_seed):
    """The exact merge over torch.distributed collectives: the local partial state, MAX all-reduce of the row maxima,
    rescale, ONE packed SUM all-reduce of [numerator | denominator].  -> (out, m_glob, l_glob): the normalised output
    and the row statistics over all m_total keys, on every rank."""
    B, M_local = k_shard.shape[0], k_shard.shape[1]
    N = q.shape[1]
    dv = v_shard.shape[2] // num_heads if v_shard.dim() == 3 else v_shard.shape[3]
    rows = B * num_heads * N
    if M_local == 0:
        raise ValueError("every rank must own at least one key (shard_bounds guarantees it for M >= world*align)")
    # one allocation so that numerator and denominator ride the same all-reduce
    flat = torch.empty(rows * dv + rows, dtype=torch.float32, device=k_shard.device)
    po = flat[: rows * dv].view(B, num_heads, N, dv)
    pl = flat[rows * dv:].view(B, num_heads, N)
    pm = torch.empty(B, num_heads, N, dtype=torch.float32, device=k_shard.device)
    if dropout_p > 0.0:
        kernels.partial_dropout(q, k_shard, v_shard, num_heads, scale, pad_mask_shard, causal, m_total, m_offset,
                                (po, pm, pl), dropout_p, dropout_seed)
    else:
        kernels.partial(q, k_shard, v_shard, num_heads, scale, pad_mask_shard, causal, m_total, m_offset, (po, pm, pl))
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    m_glob = pm
    if world > 1:
        m_glob = pm.clone()
        dist.all_reduce(m_glob, op=dist.ReduceOp.MAX, group=group)
        kernels.rescale_(po, pm, pl, m_glob)
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    return kernels.finalize(po, pl, q.dtype), m_glob, pl


class _ShardedAttention(torch.autograd.Function):
    """Training through the key-sharded attention.  Forward: the exact merge (``_exact_merge``), keeping the merged row
    statistics.  Backward: the shard backward from those statistics (``ShardKernels.backward``) — dK / dV of the local
    keys are complete — and ONE all_reduce(SUM) of the fp32 dQ contributions over the group."""

    @staticmethod
    def forward(ctx, q, k_shard, v_shard, num_heads, scale, m_total, m_offset, pad_mask_shard, causal, group, kernels,
                dropout_p, dropout_seed):
        out, m_glob, l_glob = _exact_merge(q, k_shard, v_shard, num_heads, scale, m_total, m_offset, pad_mask_shard,
                                           causal, group, kernels, dropout_p, dropout_seed)
        ctx.save_for_backward(q, k_shard, v_shard, pad_mask_shard, out, m_glob, l_glob)
        ctx.meta = (num_heads, scale, m_total, m_offset, causal, group, kernels, dropout_p, dropout_seed)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        q, k, v, pad, out, m_glob, l_glob = ctx.saved_tensors
        H, scale, m_total, m_offset, causal, group, kernels, dropout_p, dropout_seed = ctx.meta
        gq, gk, gv = kernels.backward(q, k, v, out, grad_out, m_glob, l_glob, H, scale, pad, causal, m_total, m_offset,
                                      dropout_p, dropout_seed)
        gq = gq.float().contiguous()
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(gq, op=dist.ReduceOp.SUM, group=group)
        return (gq.to(q.dtype), gk.to(k.dtype), gv.to(v.dtype)) + (None,) * 10


def sharded_attention(q: torch.Tensor, k_shard: torch.Tensor, v_shard: torch.Tensor, num_heads: int, scale: float,
                      m_total: int, m_offset: int, pad_mask_shard: Optional[torch.Tensor] = None,
                      causal: bool = False, group=None, kernels: Optional[ShardKernels] = None,
                      merge: str = "auto", copy_out: bool = True, dropout_p: float = 0.0,
                      dropout_seed: Optional[int] = None) -> torch.Tensor:
    """softmax(QK^T)V with K/V sharded along M over ``group``; every rank returns the full (B,N,H*dv).

    ``merge``: "fused" (ONE launch per rank: the merge runs in the attention kernel's tail over NVLink-mapped
    symmetric memory, no host-launched barrier, no NCCL), "peer" (partial-state kernel, signal-pad barrier, separate
    merge kernel, barrier), "nccl" (two all-reduces) or "auto" (fused when the kernel family covers the shapes and all
    shards are equally long, else peer, else nccl).  With the fused / peer merge the result lives in a reused symmetric
    buffer; ``copy_out=False`` returns that buffer itself (valid until the next call).

    Training: under autograd (grad enabled and q, k_shard or v_shard requiring grad) the call is differentiable.  Only
    the "nccl" merge leaves the merged row statistics on every rank, so "auto" selects it and "fused" / "peer" raise.
    An inference call made with grad enabled on operands that require grad (e.g. projected by parameters that require
    grad) is such a training call: run inference under ``torch.no_grad()`` to keep the fused merge.
    The backward computes dK / dV of the local keys locally and sums the dQ contributions with ONE fp32 all-reduce
    (B or 1, N, H*dqk floats) over the group — no other communication.  Every rank of the group must pass the SAME
    ``grad_out``: true when everything downstream is replicated, as after ``cross_attention_sharded``.

    ``dropout_p`` > 0 applies the attention-probability dropout (reference modules.py:161) with the mask of the
    unsharded call over global key indices (``m_offset`` must be even; ``shard_bounds`` gives 128-aligned offsets).  The
    seed must be identical on every rank of the group, else the gradients are silently wrong: ``dropout_seed=None``
    draws one on the group's first rank and broadcasts it (one 8-byte collective and one host read per call); a
    given seed is used as is."""
    world_now = dist.get_world_size(group) if dist.is_initialized() else 1
    train = torch.is_grad_enabled() and (q.requires_grad or k_shard.requires_grad or v_shard.requires_grad)
    if train or dropout_p > 0.0:
        if dropout_p > 0.0 and not 0.0 < dropout_p < 1.0:
            raise ValueError(f"dropout_p must be in [0, 1), got {dropout_p}")
        if merge not in ("auto", "nccl"):
            raise RuntimeError(f"sharded_attention: merge={merge!r} cannot be used for training or dropout: only the "
                               "'nccl' merge leaves the merged row statistics (and the dropout forward) on every rank")
        kernels = kernels or ShardKernels()
        seed = 0
        if dropout_p > 0.0:
            seed = _shared_dropout_seed(group, k_shard.device) if dropout_seed is None else int(dropout_seed)
        if train:
            return _ShardedAttention.apply(q, k_shard, v_shard, num_heads, scale, m_total, m_offset, pad_mask_shard,
                                           causal, group, kernels, float(dropout_p), seed)
        return _exact_merge(q, k_shard, v_shard, num_heads, scale, m_total, m_offset, pad_mask_shard, causal, group,
                            kernels, float(dropout_p), seed)[0]
    merge_requested = merge
    if merge == "auto":
        merge = "fused" if (kernels is None and not PeerMerger.disabled and _peer_merge_possible(k_shard, world_now)) else "nccl"
        if merge == "fused" and q.shape[1] <= 4:
            # decode step (a handful of query rows against a sharded cache): the streaming decode kernel produces the
            # partial state, the 33 KB-per-rank merge goes through the peer kernel
            merge = "peer"
    if merge in ("peer", "fused") and world_now > 1:
        from . import ops

        H = num_heads
        B, N = k_shard.shape[0], q.shape[1]
        dv = (v_shard.shape[2] // H) if v_shard.dim() == 3 else v_shard.shape[3]
        cdt = q.dtype if q.dtype in (torch.bfloat16, torch.float16) else torch.bfloat16
        try:
            pm = PeerMerger.get(B, H, N, dv, cdt, k_shard.device, group)
        except Exception as exc:  # noqa: BLE001 — symmetric memory cannot be set up on this system
            if merge_requested == "peer":
                raise
            _warn_once(f"perceiver_io_b200.dist: peer-memory merge unavailable ({type(exc).__name__}: {exc}); "
                       "using the NCCL all-reduce merge")
            PeerMerger.disabled = True
            pm = None
        if pm is None:
            return sharded_attention(q, k_shard, v_shard, num_heads, scale, m_total, m_offset, pad_mask_shard, causal,
                                     group, kernels, merge="nccl")
        if merge == "fused":
            # every rank must take the same path: equal shard lengths (identical work plans, hence identical grids) and
            # shapes the kernel family with the built-in tail covers; the decision depends on shapes only
            M_local = k_shard.shape[1]
            even = (m_total % world_now == 0) and (M_local * world_now == m_total)
            ok = even and ops.attention_sharded_fused(q, k_shard, v_shard, H, scale, None, pad_mask=pad_mask_shard,
                                                      causal=causal, m_total=m_total, m_offset=m_offset, check_only=True)
            if ok:
                pmf = PeerMerger.get(B, H, N, dv, cdt, k_shard.device, group, tag=("fused", M_local))
                out = pmf.fused_attention(q, k_shard, v_shard, H, scale, m_total, m_offset, pad_mask_shard, causal)
                out = out.clone() if copy_out else out
                return out if out.dtype == q.dtype else out.to(q.dtype)
            if merge_requested == "fused":
                raise RuntimeError("fused merge requested but the shapes are not covered (uneven shards or big-head kernel)")
        ops.attention_partial(q, k_shard, v_shard, H, scale, pad_mask=pad_mask_shard, causal=causal,
                              m_total=m_total, m_offset=m_offset, out=(pm.po, pm.pm, pm.pl))
        out = pm.merge()
        out = out.clone() if copy_out else out
        return out if out.dtype == q.dtype else out.to(q.dtype)
    return _exact_merge(q, k_shard, v_shard, num_heads, scale, m_total, m_offset, pad_mask_shard, causal, group,
                        kernels or ShardKernels(), 0.0, 0)[0]


def cross_attention_sharded(module, x_q: torch.Tensor, x_kv_shard: torch.Tensor, m_total: int, m_offset: int,
                            pad_mask_shard: Optional[torch.Tensor] = None, group=None,
                            kernels: Optional[ShardKernels] = None, merge: str = "auto"):
    """``CrossAttention.forward`` (reference modules.py:204-230) with ``x_kv`` sharded along M.

    ``module`` is a CrossAttention (this package's or a patched reference one).  LayerNorm and the K/V
    projections run on the local shard only — they are 2/3 of the module's FLOPs and shard perfectly —
    then the attention core is merged across ranks and ``o_proj`` is applied replicated.

    Training: in training mode the module's attention dropout is applied (one seed per call, broadcast from the group's
    first rank), and the call is differentiable (``sharded_attention``).  After ``loss.backward()`` the q-side and
    replicated parameters hold their full gradient on every rank; the parameters that saw only the local shard
    (kv_norm, k_proj, v_proj and whatever produced ``x_kv_shard``) hold the local share: sum it with
    ``reduce_shard_grads``."""
    from .utils import ModuleOutput

    from .modules import fused_linear, project_kv

    attn = module.attention
    q = fused_linear(module, "_pcv_q_fold", module.q_norm, attn.q_proj, x_q)
    k, v = project_kv(module, x_kv_shard)  # fused LayerNorm + K/V producer on the local shard
    drop_p = float(attn.dropout.p) if module.training else 0.0
    o = sharded_attention(q, k, v, attn.num_heads, attn.dp_scale, m_total, m_offset, pad_mask_shard,
                          attn.causal_attention, group, kernels, merge=merge, dropout_p=drop_p)
    return ModuleOutput(last_hidden_state=fused_linear(attn, "_pcv_o_fold", None, attn.o_proj, o), kv_cache=None)


def reduce_shard_grads(parameters, group=None) -> None:
    """Sum in place, over ``group``, the ``.grad`` of parameters whose forward saw only the local key shard:
    kv_norm / k_proj / v_proj of a ``cross_attention_sharded`` module and an input adapter run on the shard.  The
    q-side and replicated parameters already hold the full gradient on every rank and must NOT be passed.  Every rank
    must pass the same parameters in the same order (one all-reduce each; parameters without a gradient are skipped on
    every rank alike).  Wiring into DDP / FSDP (which would average over the batch groups too) is left to the caller."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    for p in parameters:
        if p.grad is not None:
            dist.all_reduce(p.grad, op=dist.ReduceOp.SUM, group=group)
