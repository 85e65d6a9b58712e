"""-m gpu: training through the key-sharded attention on one H100.

- Sequential shards: the shard partial states (with dropout: pcv_attn_fwd_partial_dropout_shard) merged on the device,
  each shard's backward (pcv_attn_bwd_shard, or the shim with a key offset above head dim 192) from the merged
  statistics, grad_q32 summed and grad_k / grad_v concatenated, against fp64 autograd on the globally exported mask
  with the gates of test_gpu_bwd.py (gpu_util.assert_grads).
- dK / dV of 128-aligned shards equal the unsharded backward's rows bit for bit (same key tiles, same arithmetic).
- The sharded dropout forward applies dropout_keep_mask over the global key range and leaves part_m / part_l alone.
- Two processes on cuda:0 with a gloo group: a cross_attention_sharded training step plus reduce_shard_grads gives every
  parameter the gradient of the one-process CrossAttention step."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

from gpu_util import GRAD_FLOOR, assert_grad_set, derived_bound, grad_magnitudes
from perceiver_io_b200 import _lib, dist as pdist, ops
from test_gpu_bwd import _case
from test_gpu_dropout import _drop_ref, _rp

pytestmark = pytest.mark.gpu

SEED = 0x5EED_5A4D_0001
_DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
B, N, M, H = 2, 130, 700, 2


def _bounds(G):
    return [pdist.shard_bounds(M, G, r) for r in range(G)]


def _sharded(q, k, v, go, H, pad, causal, G, p):
    """-> (out, grad_q, grad_k, grad_v) of the sharded protocol, shard after shard on one device."""
    scale = (q.shape[-1] // H) ** -0.5
    kern = pdist.ShardKernels()
    dv = v.shape[-1] // H
    parts = []
    for b, e in _bounds(G):
        pd = None if pad is None else pad[:, b:e]
        out = (torch.empty(B, H, N, dv, device="cuda"), torch.empty(B, H, N, device="cuda"),
               torch.empty(B, H, N, device="cuda"))
        if p > 0:
            kern.partial_dropout(q, k[:, b:e], v[:, b:e], H, scale, pd, causal, M, b, out, p, SEED)
        else:
            # odd head dims: the partial forward takes zero-padded operands, as the dropout forward does
            qp, kp, vp = q, k[:, b:e], v[:, b:e]
            if (q.shape[-1] // H) % 8 or dv % 8:
                qp, kp, vp = (ops._pad_heads_to8(t, H) for t in (qp, kp, vp))
            po, pm, pl = ops.attention_partial(qp, kp, vp, H, scale, pad_mask=pd, causal=causal, m_total=M, m_offset=b)
            out[0].copy_(po[..., :dv])
            out[1].copy_(pm)
            out[2].copy_(pl)
        parts.append(out)
    po, m, l = ops.merge_partials(*(torch.stack([x[i] for x in parts]) for i in range(3)))
    o = ops.combine_partials(po[None], m[None], l[None], q.dtype)
    gq = torch.zeros(q.shape, dtype=torch.float32, device="cuda")
    gks, gvs = [], []
    for b, e in _bounds(G):
        pd = None if pad is None else pad[:, b:e]
        g32, gk, gv = kern.backward(q, k[:, b:e], v[:, b:e], o, go, m, l, H, scale, pd, causal, M, b, p, SEED)
        assert g32.dtype == torch.float32 and g32.shape == q.shape
        gq += g32
        gks.append(gk.to(q.dtype))
        gvs.append(gv.to(q.dtype))
    return o, gq, torch.cat(gks, 1), torch.cat(gvs, 1)


CASES = [  # G, dqk, dv, bcast, dtype, pad kind, causal, p
    (2, 32, 160, True, "bf16", "row_full", False, 0.1),
    (3, 64, 64, False, "fp16", "ragged", True, 0.0),
    (3, 64, 64, False, "bf16", "row_full", True, 0.1),
    (4, 128, 128, False, "bf16", "row_full", True, 0.1),
    (4, 128, 128, True, "fp16", None, False, 0.0),
    (3, 131, 131, True, "bf16", "row_full", False, 0.1),
    (2, 160, 32, False, "bf16", "ragged", True, 0.0),
    (4, 192, 192, True, "fp16", "row_full", True, 0.1),
    (3, 192, 192, False, "bf16", None, True, 0.0),
    (2, 256, 256, False, "bf16", "row_full", True, 0.1),   # above 192: the shim with the key offset
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"G{c[0]}-d{c[1]}x{c[2]}{'-bcast' if c[3] else ''}-{c[4]}-"
                                                      f"{c[5] or 'nopad'}{'-causal' if c[6] else ''}-p{c[7]}")
def test_sequential_shards_match_autograd(case):
    G, dqk, dv, bcast, dt, pad_kind, causal, p = case
    dtype = _DTYPES[dt]
    q, k, v, go, pad = _case(B, N, M, H, dqk, dv, pad_kind, causal, bcast, dtype=dtype, seed=dqk + dv + G)
    if pad_kind == "row_full":
        assert pad[0].all() and pad[1, 256:].all()  # uniform row 0; shards past key 256 wholly padded for row 1
    scale = dqk ** -0.5
    out, *got = _sharded(q, k, v, go, H, pad, causal, G, p)
    keep = ops.dropout_keep_mask(B, H, N, M, p, SEED) if p > 0 else torch.ones(B, H, N, M, dtype=torch.bool,
                                                                                device="cuda")
    rp = _rp(p)[1] if p > 0 else 1.0

    r64, eager = (_drop_ref(q, k, v, go, H, scale, pad, causal, dt_, keep, rp) for dt_ in (torch.float64, dtype))
    assert out.shape == r64[0].shape and torch.isfinite(out).all()
    bound, eager_err, ref_max = derived_bound(r64[0], eager[0])
    bound = max(bound, GRAD_FLOOR * ref_max)
    err = (out.double() - r64[0]).abs().max().item()
    print(f"[shard train] {case} out: err {err:.3e} bound {bound:.3e} (eager {eager_err:.3e})")
    assert err <= bound, f"out: err {err:.3e} > bound {bound:.3e}"
    mags = grad_magnitudes(q, k, v, go, H, scale, pad, causal, keep if p > 0 else None, rp)
    assert_grad_set(got, r64[1:], eager[1:], mags, dtype, f"shard train {case}")


@pytest.mark.parametrize("dims, p, causal, pad_kind", [
    ((64, 64), 0.0, True, "ragged"), ((128, 128), 0.1, True, "row_full"), ((32, 160), 0.1, False, "ragged"),
    ((192, 192), 0.1, True, None), ((136, 136), 0.0, False, "row_full"),
], ids=["d64-causal", "d128-drop-causal", "d32x160-drop", "d192-drop-causal", "d136"])
def test_shard_dkdv_equal_the_unsharded_rows_bitwise(dims, p, causal, pad_kind):
    """The same (m, l, out) into pcv_attn_bwd and into pcv_attn_bwd_shard of 128-aligned shards: a shard's key tiles
    are the unsharded call's tiles, so grad_k / grad_v match bit for bit — an off-by-offset in the causal diagonal or
    the dropout key would not."""
    dqk, dv = dims
    q, k, v, go, pad = _case(B, N, M, H, dqk, dv, pad_kind, causal, True, seed=5)
    scale = dqk ** -0.5
    po, m, l = ops.attention_partial(q, k, v, H, scale, pad_mask=pad, causal=causal)
    out = ops.combine_partials(po[None], m[None], l[None], q.dtype)
    _, gk, gv = ops.attention_backward(q, k, v, out, go, m, l, H, scale, pad_mask=pad, causal=causal, dropout_p=p,
                                       dropout_seed=SEED)
    for b, e in _bounds(3):
        pd = None if pad is None else pad[:, b:e]
        _, sk, sv = ops.attention_backward_shard(q, k[:, b:e], v[:, b:e], out, go, m, l, H, scale, M, b, pad_mask=pd,
                                                 causal=causal, dropout_p=p, dropout_seed=SEED)
        assert torch.equal(sk, gk[:, b:e]), (b, (sk.float() - gk[:, b:e].float()).abs().max().item())
        assert torch.equal(sv, gv[:, b:e]), (b, (sv.float() - gv[:, b:e].float()).abs().max().item())


@pytest.mark.parametrize("dqk, dv, dt", [(64, 64, "bf16"), (136, 120, "bf16"), (32, 160, "fp16"), (72, 512, "bf16")])
def test_sharded_dropout_forward_applies_the_global_mask(dqk, dv, dt):
    """q = 0: every score is 0.  v = e_(j mod dv) over GLOBAL key j: part_o counts the kept keys of the shard per
    channel, as dropout_keep_mask over [m_offset, m_offset + M_shard) exports them.  part_m / part_l are those of the
    dropout-free partial call, bit for bit."""
    dtype = _DTYPES[dt]
    p = 0.25
    q = torch.zeros(1, N, H * dqk, device="cuda", dtype=dtype)
    k = torch.randn(B, M, H * dqk, device="cuda", dtype=dtype)
    j = torch.arange(M, device="cuda")
    v = torch.nn.functional.one_hot(j % dv, dv).to(dtype)[None, :, None, :].expand(B, M, H, dv).reshape(B, M, H * dv)
    v = v.contiguous()
    rp = torch.tensor(_rp(p)[1], dtype=torch.float32)
    for b, e in _bounds(3):
        po, pm, pl = ops.attention_partial(q, k[:, b:e], v[:, b:e], H, dqk ** -0.5, m_total=M, m_offset=b, dropout_p=p,
                                           dropout_seed=SEED)
        _, pm0, pl0 = ops.attention_partial(q, k[:, b:e], v[:, b:e], H, dqk ** -0.5, m_total=M, m_offset=b,
                                            impl="tcgen05")
        assert torch.equal(pm, pm0) and torch.equal(pl, pl0)
        keep = ops.dropout_keep_mask(B, H, N, M, p, SEED, key_begin=b, key_end=e).float()
        onehot = torch.nn.functional.one_hot(j[b:e] % dv, dv).float()
        want = (keep @ onehot) * rp
        assert (po[want == 0] == 0).all()
        rel = ((po - want).abs() / want.clamp_min(1)).max().item()
        assert rel <= 1e-6, (b, rel)


# ---- two processes on one GPU ---------------------------------------------------------------------------------------
def _train_worker(rank, world, port, queue):
    import torch.distributed as dist

    from perceiver_io_b200 import CrossAttention
    from perceiver_io_b200.dist import cross_attention_sharded, reduce_shard_grads, shard_bounds

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.manual_seed(0)
        Hh, Dq, Ckv, Nq, Mk = 8, 512, 256, 128, 4096
        mod = CrossAttention(num_heads=Hh, num_q_input_channels=Dq, num_kv_input_channels=Ckv, dropout=0.1)
        mod = mod.cuda().to(torch.bfloat16).train()
        g = torch.Generator(device="cuda").manual_seed(3)
        x_q = torch.randn(1, Nq, Dq, device="cuda", generator=g).bfloat16()
        x_kv = torch.randn(2, Mk, Ckv, device="cuda", generator=g).bfloat16()
        go = torch.randn(2, Nq, Dq, device="cuda", generator=g).bfloat16()
        pad = torch.zeros(2, Mk, dtype=torch.bool, device="cuda")
        pad[1, 3000:] = True
        b, e = shard_bounds(Mk, world, rank)
        out = cross_attention_sharded(mod, x_q, x_kv[:, b:e], Mk, b, pad[:, b:e]).last_hidden_state
        out.backward(go)
        attn = mod.attention
        reduce_shard_grads(list(mod.kv_norm.parameters()) + list(attn.k_proj.parameters())
                           + list(attn.v_proj.parameters()))
        torch.cuda.synchronize()
        # numpy arrays: a tensor would be passed by a file descriptor that dies with this process
        queue.put((rank, {n: p.grad.float().cpu().numpy() if p.grad is not None else None
                          for n, p in mod.named_parameters()}, out.detach().float().cpu().numpy()))
    finally:
        dist.destroy_process_group()


def test_two_ranks_on_one_gpu_train_like_one_process():
    """Both ranks' every parameter gradient (after reduce_shard_grads) matches the one-process CrossAttention step with
    the same dropout seed, within 3e-2 of max|grad| (bf16 parameters: the gradients are rounded to bf16, and the two
    steps sum the keys' contributions in different orders)."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    queue = ctx.Queue()
    procs = [ctx.Process(target=_train_worker, args=(r, 2, port, queue)) for r in range(2)]
    for p_ in procs:
        p_.start()
    try:
        results = [queue.get(timeout=300) for _ in procs]
    finally:
        for p_ in procs:
            p_.join(timeout=60)
            if p_.is_alive():
                p_.kill()
    assert all(p_.exitcode == 0 for p_ in procs)

    from perceiver_io_b200 import CrossAttention

    torch.manual_seed(0)
    Hh, Dq, Ckv, Nq, Mk = 8, 512, 256, 128, 4096
    mod = CrossAttention(num_heads=Hh, num_q_input_channels=Dq, num_kv_input_channels=Ckv, dropout=0.1)
    mod = mod.cuda().to(torch.bfloat16).train()
    g = torch.Generator(device="cuda").manual_seed(3)
    x_q = torch.randn(1, Nq, Dq, device="cuda", generator=g).bfloat16()
    x_kv = torch.randn(2, Mk, Ckv, device="cuda", generator=g).bfloat16()
    go = torch.randn(2, Nq, Dq, device="cuda", generator=g).bfloat16()
    pad = torch.zeros(2, Mk, dtype=torch.bool, device="cuda")
    pad[1, 3000:] = True
    # the dropout seed comes from the CPU generator in the state the group's first rank drew it in
    out = mod(x_q, x_kv, pad_mask=pad).last_hidden_state
    out.backward(go)
    ref = {n: p.grad.float().cpu() for n, p in mod.named_parameters()}
    for rank, grads, out_r in results:
        err = (torch.from_numpy(out_r) - out.detach().float().cpu()).abs().max().item()
        assert err <= 3e-2 * out.detach().float().abs().max().item(), (rank, "out", err)
        for name, r in ref.items():
            assert grads[name] is not None, (rank, name, "no gradient")
            got = torch.from_numpy(grads[name])
            err = (got - r).abs().max().item()
            print(f"[2 ranks] rank {rank} {name}: err {err:.3e} max|ref| {r.abs().max().item():.3e}")
            # k_proj.bias: its exact gradient is 0 (a key bias shifts every row's scores by a constant), so both steps
            # give rounding noise; it is held to the scale of the k_proj weight gradient
            scale = ref["attention.k_proj.weight"] if name == "attention.k_proj.bias" else r
            assert err <= 3e-2 * scale.abs().max().item() + 1e-6, (rank, name, err)


def test_zz_watchdog_record_is_clear():
    """No barrier wait of any kernel timed out during this module (runs last in it)."""
    torch.cuda.synchronize()
    assert _lib.debug_read()[0] == 0, _lib.debug_read()
