"""CPU checks of training through the key-sharded attention: the C entry points of the shard forward with dropout and
the shard backward (symbols, struct layout, argument checks before any CUDA call, workspace size without a device),
the backward shim with a key offset against fp64 autograd, and the autograd protocol of ``dist.sharded_attention`` /
``cross_attention_sharded`` / ``reduce_shard_grads`` on gloo with injected fp64 math."""
import copy
import ctypes
import os
import socket
import subprocess

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT
from oracle import dropout_oracle as D
from oracle import mha_oracle as O
from perceiver_io_b200 import _lib, ops

NEW_SYMBOLS = ("pcv_attn_fwd_partial_dropout_shard_supported", "pcv_attn_fwd_partial_dropout_shard",
               "pcv_attn_bwd_shard_supported", "pcv_attn_bwd_shard_workspace_bytes", "pcv_attn_bwd_shard")
FLT_MAX = torch.finfo(torch.float32).max


def test_new_symbols_are_declared_and_exported():
    lib = _lib.lib()
    header = open(os.path.join(ROOT, "include", "pcv_attn.h")).read()
    for name in NEW_SYMBOLS:
        assert name in _lib.EXPORTS and hasattr(lib, name) and f"{name}(" in header, name


def test_key_shard_layout_matches_header(tmp_path):
    cls = _lib.KeyShard
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "pcv_attn.h")}"',
             "int main(void){", 'printf("size %zu\\n", sizeof(pcv_key_shard));']
    lines += [f'printf("{f} %zu\\n", offsetof(pcv_key_shard, {f}));' for f, _ in cls._fields_]
    lines.append("return 0;}")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-o", str(tmp_path / "layout"), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(tmp_path / "layout")]).decode().split("\n") if l)
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def _bwd_params(**kw):
    """A backward call that passes every argument check (fake, never dereferenced pointers): keys [1024, 2048) of
    4096."""
    p = _lib.AttnBwdParams()
    p.q = p.k = p.v = p.out = p.grad_out = p.stat_m = p.stat_l = p.grad_k = p.grad_v = 1 << 20
    p.B, p.H, p.N, p.M, p.dqk, p.dv = 2, 4, 200, 1024, 64, 64
    p.q_stride_b, p.q_stride_n, p.q_stride_h = 0, 256, 64
    for pre in ("k", "v", "gk", "gv"):
        setattr(p, f"{pre}_stride_b", 1024 * 256)
        setattr(p, f"{pre}_stride_m", 256)
        setattr(p, f"{pre}_stride_h", 64)
    p.o_stride_b = p.go_stride_b = 200 * 256
    p.o_stride_n = p.go_stride_n = 256
    p.o_stride_h = p.go_stride_h = 64
    p.scale, p.dtype = 0.125, _lib.PCV_BF16
    for name, value in kw.items():
        setattr(p, name, value)
    return p


def _shard(m_total=4096, m_offset=1024, grad_q32=1 << 21):
    s = _lib.KeyShard()
    s.m_total, s.m_offset, s.grad_q32 = m_total, m_offset, grad_q32
    return s


@pytest.mark.parametrize("pkw, skw, msg", [
    ({}, {"m_offset": 1023}, b"even"),
    ({}, {"m_offset": 3584}, b"outside m_total"),
    ({}, {"m_offset": -2}, b"outside m_total"),
    ({}, {"grad_q32": 0}, b"grad_q32 is NULL"),
    ({}, {"grad_q32": (1 << 21) + 4}, b"16-byte aligned"),
    ({"dqk": 200}, {}, b"[8, 192]"),
    ({"dv": 256}, {}, b"[8, 192]"),
    ({"dropout_p": 1.0}, {}, b"dropout_p"),
    ({"causal": 1}, {"m_total": 1100, "m_offset": 0}, b"OK"),
    ({"causal": 1, "N": 2000}, {"m_total": 1100, "m_offset": 0}, b"m_total >= N"),
])
def test_bwd_shard_rejects_bad_arguments_before_any_cuda_call(pkw, skw, msg):
    lib = _lib.lib()
    p, s = _bwd_params(**pkw), _shard(**skw)
    rc = lib.pcv_attn_bwd_shard(ctypes.byref(p), ctypes.byref(s), None)
    if msg == b"OK":  # every argument passes: what fails on a CPU-only box is the device itself
        assert rc != 0 and b"shard" not in lib.pcv_last_error()
        return
    assert rc == 2 and msg in lib.pcv_last_error(), (rc, lib.pcv_last_error())
    assert lib.pcv_attn_bwd_shard_supported(ctypes.byref(p), ctypes.byref(s)) == 0
    assert msg in lib.pcv_last_error()


def test_bwd_shard_rejects_null_arguments():
    lib = _lib.lib()
    p, s = _bwd_params(), _shard()
    need = ctypes.c_size_t(0)
    assert lib.pcv_attn_bwd_shard(None, ctypes.byref(s), None) == 1 and b"NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_bwd_shard(ctypes.byref(p), None, None) == 1 and b"NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_bwd_shard_supported(None, ctypes.byref(s)) == 0
    assert lib.pcv_attn_bwd_shard_supported(ctypes.byref(p), None) == 0 and b"NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_bwd_shard_workspace_bytes(None, ctypes.byref(s), ctypes.byref(need)) == 1
    assert lib.pcv_attn_bwd_shard_workspace_bytes(ctypes.byref(p), None, ctypes.byref(need)) == 1
    assert lib.pcv_attn_bwd_shard_workspace_bytes(ctypes.byref(p), ctypes.byref(s), None) == 1


def test_bwd_shard_workspace_is_computed_without_a_device():
    """Up to head dim 128 the dQ kernel accumulates into the caller's grad_q32: the workspace is the statistics blocks
    alone (the unsharded backward adds its fp32 dQ accumulator).  Above 128 both hold the same dQ partials."""
    lib = _lib.lib()
    need, full = ctypes.c_size_t(0), ctypes.c_size_t(0)
    p, s = _bwd_params(), _shard()
    assert lib.pcv_attn_bwd_shard_workspace_bytes(ctypes.byref(p), ctypes.byref(s), ctypes.byref(need)) == 0
    assert lib.pcv_attn_bwd_workspace_bytes(ctypes.byref(p), ctypes.byref(full)) == 0
    stats = 768 * 2 * 4 * 4  # 768 B per (b, h, 64 queries), 200 queries padded to 256
    assert need.value == (stats + 255) // 256 * 256
    dq32 = 4 * 1 * 200 * 4 * 64
    assert full.value == need.value + (dq32 + 255) // 256 * 256
    p = _bwd_params(dqk=160, dv=160)
    assert lib.pcv_attn_bwd_shard_workspace_bytes(ctypes.byref(p), ctypes.byref(s), ctypes.byref(need)) == 0
    assert lib.pcv_attn_bwd_workspace_bytes(ctypes.byref(p), ctypes.byref(full)) == 0
    assert need.value == full.value > (stats + 255) // 256 * 256 + 2 * 4 * 200 * 4 * 160


def _fwd_params(**kw):
    """A partial-state forward over keys [1024, 2048) of 4096 (fake, never dereferenced pointers)."""
    p = _lib.AttnParams()
    p.q = p.k = p.v = 1 << 20
    p.B, p.H, p.N, p.M, p.dqk, p.dv = 2, 8, 256, 1024, 32, 160
    p.q_stride_b, p.q_stride_n, p.q_stride_h = 0, 256, 32
    p.k_stride_b, p.k_stride_m, p.k_stride_h = 1024 * 256, 256, 32
    p.v_stride_b, p.v_stride_m, p.v_stride_h = 1024 * 1280, 1280, 160
    p.scale, p.dtype, p.m_total, p.m_offset = 32 ** -0.5, _lib.PCV_BF16, 4096, 1024
    p.write_partial = 1
    p.part_o = p.part_m = p.part_l = 1 << 21
    for name, value in kw.items():
        setattr(p, name, value)
    return p


@pytest.mark.parametrize("kw, dropout_p, rc, msg", [
    ({"m_offset": 1023}, 0.1, 2, b"even"),
    ({}, 0.0, 2, b"dropout_p"),
    ({}, 1.0, 2, b"dropout_p"),
    ({}, -0.1, 2, b"dropout_p"),
    ({"m_offset": 3584}, 0.1, 1, b"outside m_total"),
    ({"write_partial": 0, "out": 1 << 22}, 0.1, 2, b"write_partial"),
    ({"impl": _lib.PCV_IMPL_TCGEN05_PAIR}, 0.1, 2, b"single-CTA"),
])
def test_fwd_shard_rejects_bad_arguments_before_any_cuda_call(kw, dropout_p, rc, msg):
    lib = _lib.lib()
    p = _fwd_params(**kw)
    got = lib.pcv_attn_fwd_partial_dropout_shard(ctypes.byref(p), ctypes.c_float(dropout_p), ctypes.c_uint64(1), None)
    assert got == rc and msg in lib.pcv_last_error(), (got, lib.pcv_last_error())
    assert lib.pcv_attn_fwd_partial_dropout_shard_supported(ctypes.byref(p), ctypes.c_float(dropout_p)) == 0
    assert msg in lib.pcv_last_error()


def test_fwd_shard_null_params_and_the_old_entry_point_still_refuses_shards():
    lib = _lib.lib()
    assert lib.pcv_attn_fwd_partial_dropout_shard(None, ctypes.c_float(0.1), ctypes.c_uint64(1), None) == 1
    assert b"NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_fwd_partial_dropout_shard_supported(None, ctypes.c_float(0.1)) == 0
    p = _fwd_params()
    assert lib.pcv_attn_fwd_partial_dropout(ctypes.byref(p), ctypes.c_float(0.1), ctypes.c_uint64(1), None) == 2
    assert b"sharding" in lib.pcv_last_error()


# ---- fp64 math of a key shard in the kernels' conventions ---------------------------------------------------------
def _scores_log2(q, k, H, scale, pad, causal, m_total, m_offset):
    """(B, H, N, M) log2-domain scores of the keys [m_offset, m_offset + M) with the kernels' fill -FLT_MAX."""
    B = k.shape[0]
    s = O.masked_scores(O.split_heads(q.double().expand(B, -1, -1), H) * scale, O.split_heads(k.double(), H), pad,
                        causal, m_total, m_offset)
    fill = s == -torch.finfo(s.dtype).max
    return (s * O.LOG2E).masked_fill(fill, -FLT_MAX)


def oracle_partial(q, k, v, H, scale, pad, causal, m_total, m_offset, out, dropout_p=0.0, seed=0):
    t = _scores_log2(q, k, H, scale, pad, causal, m_total, m_offset)
    m = t.amax(-1)
    p = torch.exp2(t - m[..., None])
    l = p.sum(-1)
    if dropout_p > 0.0:
        B, _, N, M = p.shape
        keep = torch.from_numpy(D.keep_mask(B, H, N, m_offset + M, dropout_p, seed)[..., m_offset:])
        p = p * keep * D.survivor_scale(dropout_p)
    out[0].copy_(p @ O.split_heads(v.double(), H))
    out[1].copy_(m)
    out[2].copy_(l)


def oracle_keep(B, H, N, j0, j1, p, seed, device):
    return torch.from_numpy(D.keep_mask(B, H, N, j1, p, seed)[..., j0:j1])


def shim_backward(q, k, v, out, grad_out, m, l, H, scale, pad, causal, m_total, m_offset, dropout_p, seed):
    return ops._backward_shim(q, k, v, out, grad_out, m.float(), l.float(), H, scale, pad, causal, dropout_p, seed,
                              m_total, m_offset)


def _oracle_kernels():
    from perceiver_io_b200.dist import ShardKernels

    def rescale_(po, pm, pl, new_m):
        w = torch.exp2(pm - new_m)
        po.mul_(w[..., None])
        pl.mul_(w)
        pm.copy_(new_m)

    return ShardKernels(partial=oracle_partial, rescale_=rescale_, finalize=lambda po, pl, dt: O.merge_heads(
        po / pl[..., None]).to(dt), partial_dropout=oracle_partial, backward=shim_backward)


def _eager(q, k, v, H, scale, pad, causal, dropout_p=0.0, seed=0):
    """The reference's eager formula (modules.py:146-164), nn.Dropout on the probabilities as attn * keep * rp."""
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    s = O.masked_scores(O.split_heads(q.expand(B, -1, -1), H) * scale, O.split_heads(k, H), pad, causal)
    a = s.softmax(-1)
    if dropout_p > 0.0:
        a = a * torch.from_numpy(D.keep_mask(B, H, N, M, dropout_p, seed)).to(a.dtype) * D.survivor_scale(dropout_p)
    return O.merge_heads(a @ O.split_heads(v, H))


def _problem(Bq, causal, seed=0, B=2, H=2, N=6, M=300, dqk=8, dv=12):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(Bq, N, H * dqk, generator=g, dtype=torch.float64) * 2
    k = torch.randn(B, M, H * dqk, generator=g, dtype=torch.float64)
    v = torch.randn(B, M, H * dv, generator=g, dtype=torch.float64)
    go = torch.randn(B, N, H * dv, generator=g, dtype=torch.float64)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, :256] = True   # the first shard is wholly padding for batch row 0
    pad[1, :] = True      # batch row 1 is padded everywhere: uniform attention over all keys
    return q, k, v, go, pad, dqk ** -0.5


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("dropout_p", [0.0, 0.1])
@pytest.mark.parametrize("Bq", [1, 2])
def test_shim_with_key_offset_matches_autograd(causal, dropout_p, Bq, monkeypatch):
    """Each shard's shim from the MERGED statistics: grad_k / grad_v are the shard's rows of the unsharded gradient, and
    the grad_q contributions sum to the unsharded grad_q."""
    monkeypatch.setattr(ops, "_dropout_keep", oracle_keep)
    monkeypatch.setattr(ops, "_compute_dtype", lambda dt: torch.float32)
    monkeypatch.setitem(ops.backward_config, "max_score_bytes", 4 * 2 * 2 * 6 * 128)   # 128-key chunks
    q, k, v, go, pad, scale = _problem(Bq, causal)
    H, M, seed = 2, k.shape[1], 0x5EED_0001
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
    o = _eager(qa, ka, va, H, scale, pad, causal, dropout_p, seed)
    gq, gk, gv = torch.autograd.grad(o, (qa, ka, va), go)
    t = _scores_log2(q, k, H, scale, pad, causal, M, 0)
    m = t.amax(-1)
    l = torch.exp2(t - m[..., None]).sum(-1)
    got_q = torch.zeros_like(gq)
    for b, e in ((0, 128), (128, 256), (256, 300)):
        sq, sk, sv = shim_backward(q.float(), k[:, b:e].float(), v[:, b:e].float(), o.detach().float(), go.float(),
                                   m, l, H, scale, pad[:, b:e], causal, M, b, dropout_p, seed)
        got_q += sq.double()
        for got, ref, name in ((sk, gk[:, b:e], "k"), (sv, gv[:, b:e], "v")):
            err = (got.double() - ref).abs().max().item()
            assert err <= 2e-5 * max(1.0, gv.abs().max().item(), gk.abs().max().item()), (name, b, err)
    assert got_q.shape == gq.shape
    assert (got_q - gq).abs().max().item() <= 2e-5 * max(1.0, gq.abs().max().item())


# ---- gloo ---------------------------------------------------------------------------------------------------------
def _init(rank, world, port):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ops._dropout_keep = oracle_keep
    ops._compute_dtype = lambda dt: torch.float32


def _rel(got, ref):
    return (got.double() - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _two_rank_worker(rank, world, port, queue):
    from perceiver_io_b200.dist import sharded_attention, shard_bounds

    _init(rank, world, port)
    try:
        errs = {}
        H = 2
        for name, Bq, causal, dropout_p in (("bq1", 1, False, 0.0), ("bqB_causal", 2, True, 0.0),
                                            ("dropout_causal", 1, True, 0.1), ("dropout_bqB", 2, False, 0.1)):
            q, k, v, go, pad, scale = _problem(Bq, causal)
            M = k.shape[1]
            b, e = shard_bounds(M, world, rank)
            seed = 0x1234_5678_9ABC if dropout_p else None
            qa = q.clone().requires_grad_()
            ks, vs = k[:, b:e].clone().requires_grad_(), v[:, b:e].clone().requires_grad_()
            out = sharded_attention(qa, ks, vs, H, scale, M, b, pad[:, b:e], causal, kernels=_oracle_kernels(),
                                    dropout_p=dropout_p, dropout_seed=seed)
            out.backward(go)
            qr, kr, vr = (t.clone().requires_grad_() for t in (q, k, v))
            ref = _eager(qr, kr, vr, H, scale, pad, causal, dropout_p, seed or 0)
            ref.backward(go)
            errs[name] = max(_rel(out.detach(), ref.detach()), _rel(qa.grad, qr.grad), _rel(ks.grad, kr.grad[:, b:e]),
                             _rel(vs.grad, vr.grad[:, b:e]))

        # dropout_seed=None: ranks seeded differently still drop with one mask (the seed is broadcast from rank 0)
        torch.manual_seed(1000 + rank)
        q, k, v, go, pad, scale = _problem(1, True)
        M = k.shape[1]
        b, e = shard_bounds(M, world, rank)
        seeds = []
        kern = _oracle_kernels()

        def recording_partial(*a):
            seeds.append(a[-1])
            oracle_partial(*a)

        kern.partial_dropout = recording_partial
        ks, vs = k[:, b:e].clone().requires_grad_(), v[:, b:e].clone().requires_grad_()
        qa = q.clone().requires_grad_()
        out = sharded_attention(qa, ks, vs, H, scale, M, b, pad[:, b:e], True, kernels=kern, dropout_p=0.1)
        out.backward(go)
        all_seeds = [None] * world
        dist.all_gather_object(all_seeds, seeds[0])
        qr, kr, vr = (t.clone().requires_grad_() for t in (q, k, v))
        ref = _eager(qr, kr, vr, H, scale, pad, True, 0.1, seeds[0])
        ref.backward(go)
        errs["broadcast_seed"] = max(_rel(out.detach(), ref.detach()), _rel(qa.grad, qr.grad),
                                     _rel(ks.grad, kr.grad[:, b:e]), _rel(vs.grad, vr.grad[:, b:e]))

        # without autograd: bit for bit the protocol as it ran before training support (partial, MAX all-reduce,
        # rescale, one packed SUM all-reduce, finalize)
        q, k, v, go, pad, scale = _problem(1, True)
        kern = _oracle_kernels()
        with torch.no_grad():
            got = sharded_attention(q, k[:, b:e], v[:, b:e], H, scale, M, b, pad[:, b:e], True, kernels=kern)
        B, N, dv = k.shape[0], q.shape[1], v.shape[2] // H
        rows = B * H * N
        flat = torch.empty(rows * dv + rows, dtype=torch.float32)
        po, pl = flat[: rows * dv].view(B, H, N, dv), flat[rows * dv:].view(B, H, N)
        pm = torch.empty(B, H, N)
        kern.partial(q, k[:, b:e], v[:, b:e], H, scale, pad[:, b:e], True, M, b, (po, pm, pl))
        m_glob = pm.clone()
        dist.all_reduce(m_glob, op=dist.ReduceOp.MAX)
        kern.rescale_(po, pm, pl, m_glob)
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
        before = kern.finalize(po, pl, q.dtype)
        queue.put((rank, errs, all_seeds, bool(torch.equal(got, before)), got.grad_fn is None))
    finally:
        dist.destroy_process_group()


def _run(target, world, timeout=240):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    queue = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, world, port, queue)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = [queue.get(timeout=timeout) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    for p in procs:
        assert p.exitcode == 0
    return results


def test_two_rank_gloo_training_gradients_equal_unsharded_autograd():
    results = _run(_two_rank_worker, 2)
    for rank, errs, seeds, bitwise, no_graph in results:
        for name, err in errs.items():
            assert err <= 2e-5, (rank, name, err)
        assert seeds[0] == seeds[1], seeds
        assert bitwise and no_graph, rank


def _grid_worker(rank, world, port, queue):
    """B=2 on 4 ranks: 2 batch groups x 2 key shards; each batch group's backward reduces dQ over its own sub-group."""
    from perceiver_io_b200.dist import grid_position, m_shard_group, plan_grid, shard_bounds, sharded_attention

    _init(rank, world, port)
    try:
        H = 2
        q, k, v, go, pad, scale = _problem(2, True)
        M = k.shape[1]
        bg, mg = plan_grid(2, world)
        gb, gm = grid_position(rank, bg, mg)
        group = m_shard_group(bg, mg)
        rows = slice(gb, gb + 1)
        b, e = shard_bounds(M, mg, gm)
        qa = q[rows].clone().requires_grad_()
        ks, vs = k[rows, b:e].clone().requires_grad_(), v[rows, b:e].clone().requires_grad_()
        out = sharded_attention(qa, ks, vs, H, scale, M, b, pad[rows, b:e], True, group=group,
                                kernels=_oracle_kernels(), dropout_p=0.1, dropout_seed=77)
        out.backward(go[rows])
        # a batch group is its own problem: the mask hashes the group's local batch index
        qr1, kr1, vr1 = (t[rows].clone().requires_grad_() for t in (q, k, v))
        ref1 = _eager(qr1, kr1, vr1, H, scale, pad[rows], True, 0.1, 77)
        ref1.backward(go[rows])
        err = max(_rel(qa.grad, qr1.grad), _rel(ks.grad, kr1.grad[:, b:e]), _rel(vs.grad, vr1.grad[:, b:e]))
        queue.put((rank, (bg, mg, gb, gm), err))
    finally:
        dist.destroy_process_group()


def test_four_rank_gloo_grid_training_gradients():
    results = _run(_grid_worker, 4)
    assert sorted(r[1] for r in results) == [(2, 2, 0, 0), (2, 2, 0, 1), (2, 2, 1, 0), (2, 2, 1, 1)]
    for rank, _, err in results:
        assert err <= 2e-5, (rank, err)


def _module_worker(rank, world, port, queue):
    """cross_attention_sharded in training mode (attention dropout on) + reduce_shard_grads: every CrossAttention
    parameter gets the gradient of the unsharded module step."""
    from perceiver_io_b200 import CrossAttention
    from perceiver_io_b200.dist import cross_attention_sharded, reduce_shard_grads, shard_bounds

    _init(rank, world, port)
    try:
        torch.manual_seed(0)
        H, D, C, N, M = 2, 16, 12, 6, 300
        mod = CrossAttention(num_heads=H, num_q_input_channels=D, num_kv_input_channels=C, dropout=0.1).double().train()
        ref_mod = copy.deepcopy(mod)
        g = torch.Generator().manual_seed(5)
        x_q = torch.randn(1, N, D, generator=g, dtype=torch.float64)
        x_kv = torch.randn(2, M, C, generator=g, dtype=torch.float64)
        go = torch.randn(2, N, D, generator=g, dtype=torch.float64)
        pad = torch.zeros(2, M, dtype=torch.bool)
        pad[1, 250:] = True
        b, e = shard_bounds(M, world, rank)
        seeds = []
        kern = _oracle_kernels()

        def recording_partial(*a):
            seeds.append(a[-1])
            oracle_partial(*a)

        kern.partial_dropout = recording_partial
        torch.manual_seed(rank)  # the ranks' own generators differ: the seed still comes from rank 0
        out = cross_attention_sharded(mod, x_q, x_kv[:, b:e], M, b, pad[:, b:e], kernels=kern).last_hidden_state
        out.backward(go)
        attn = mod.attention
        reduce_shard_grads(list(mod.kv_norm.parameters()) + list(attn.k_proj.parameters())
                           + list(attn.v_proj.parameters()))

        ra = ref_mod.attention
        q = ra.q_proj(ref_mod.q_norm(x_q))
        kv = ref_mod.kv_norm(x_kv)
        o = _eager(q, ra.k_proj(kv), ra.v_proj(kv), H, ra.dp_scale, pad, False, 0.1, seeds[0])
        ra.o_proj(o).backward(go)
        ref_grads = dict(ref_mod.named_parameters())
        errs = {n: _rel(p.grad, ref_grads[n].grad) for n, p in mod.named_parameters()}
        queue.put((rank, errs))
    finally:
        dist.destroy_process_group()


def test_reduce_shard_grads_gives_every_cross_attention_parameter_its_unsharded_gradient():
    results = _run(_module_worker, 2)
    for rank, errs in results:
        assert len(errs) == 12  # q_norm, kv_norm, q_proj, k_proj, v_proj, o_proj: weight and bias each
        for name, err in errs.items():
            assert err <= 2e-5, (rank, name, err)
