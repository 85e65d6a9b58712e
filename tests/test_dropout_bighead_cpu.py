"""CPU checks of attention dropout above head dim 128: the one-pass dropout forward's C entry points and the mask range
export (symbols, argument checks before any CUDA call), the kernel instantiations in the library, and the backward
shim with dropout against fp64 autograd of the reference's eager formula on the numpy oracle's mask."""
import ctypes
import re

import pytest
import torch

from oracle import dropout_oracle as D
from perceiver_io_b200 import _lib, ops

NEW_SYMBOLS = ("pcv_attn_dropout_mask_range", "pcv_attn_fwd_partial_dropout_supported", "pcv_attn_fwd_partial_dropout")


def test_new_symbols_are_exported():
    lib = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in _lib.EXPORTS and hasattr(lib, name), name


def _params(**kw):
    """Parameters that pass validate_attn (fake, never dereferenced pointers): a partial-state call over all keys."""
    p = _lib.AttnParams()
    p.q = p.k = p.v = 1 << 20
    p.B, p.H, p.N, p.M, p.dqk, p.dv = 2, 8, 256, 1024, 32, 160
    p.q_stride_b, p.q_stride_n, p.q_stride_h = 0, 256, 32
    p.k_stride_b, p.k_stride_m, p.k_stride_h = 1024 * 256, 256, 32
    p.v_stride_b, p.v_stride_m, p.v_stride_h = 1024 * 1280, 1280, 160
    p.scale, p.dtype, p.m_total = 32 ** -0.5, _lib.PCV_BF16, 1024
    p.write_partial = 1
    p.part_o = p.part_m = p.part_l = 1 << 21
    for name, value in kw.items():
        setattr(p, name, value)
    return p


@pytest.mark.parametrize("kw, dropout_p, rc, msg", [
    ({"write_partial": 0, "out": 1 << 22}, 0.1, 2, b"write_partial"),
    ({"m_total": 2048}, 0.1, 2, b"sharding"),
    ({"m_total": 2048, "m_offset": 1024}, 0.1, 2, b"sharding"),
    ({"impl": _lib.PCV_IMPL_TCGEN05_PAIR}, 0.1, 2, b"single-CTA"),
    ({"impl": _lib.PCV_IMPL_SIMT}, 0.1, 2, b"single-CTA"),
    ({}, 0.0, 2, b"dropout_p"),
    ({}, 1.0, 2, b"dropout_p"),
    ({"B": 0}, 0.1, 1, b"B=0"),
    ({"q": 0}, 0.1, 1, b"NULL"),
])
def test_partial_dropout_rejects_bad_arguments_before_any_cuda_call(kw, dropout_p, rc, msg):
    lib = _lib.lib()
    p = _params(**kw)
    got = lib.pcv_attn_fwd_partial_dropout(ctypes.byref(p), ctypes.c_float(dropout_p), ctypes.c_uint64(1), None)
    assert got == rc and msg in lib.pcv_last_error(), (got, lib.pcv_last_error())
    assert lib.pcv_attn_fwd_partial_dropout_supported(ctypes.byref(p), ctypes.c_float(dropout_p)) == 0
    assert msg in lib.pcv_last_error()


def test_partial_dropout_rejects_null_params():
    lib = _lib.lib()
    assert lib.pcv_attn_fwd_partial_dropout(None, ctypes.c_float(0.1), ctypes.c_uint64(1), None) == 1
    assert b"NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_fwd_partial_dropout_supported(None, ctypes.c_float(0.1)) == 0


@pytest.mark.parametrize("keep, B, H, N, k0, k1, p", [
    (None, 1, 1, 8, 0, 8, 0.1),
    (1 << 20, 0, 1, 8, 0, 8, 0.1),
    (1 << 20, 1, 1, 0, 0, 8, 0.1),
    (1 << 20, 1, 1, 8, -1, 8, 0.1),
    (1 << 20, 1, 1, 8, 8, 8, 0.1),
    (1 << 20, 1, 1, 8, 9, 8, 0.1),
    (1 << 20, 1, 1, 8, 0, 8, 1.0),
    (1 << 20, 1, 1, 8, 0, 8, -0.5),
])
def test_mask_range_rejects_bad_arguments_before_any_cuda_call(keep, B, H, N, k0, k1, p):
    lib = _lib.lib()
    rc = lib.pcv_attn_dropout_mask_range(keep, B, H, N, k0, k1, ctypes.c_float(p), ctypes.c_uint64(1), None)
    assert rc == 1 and b"dropout_mask" in lib.pcv_last_error()


def test_library_holds_exactly_the_32_dropout_forward_instantiations():
    """attn_fwd_drop_kernel<NQB, NVB, BF16>: NQB 1..8 x NVB 1..2 x bf16/fp16, no CTA-pair variant."""
    with open(_lib.LIB_PATH, "rb") as f:
        blob = f.read()
    found = re.findall(rb"20attn_fwd_drop_kernelILi(\d)ELi(\d)ELb([01])EEEv", blob)
    got = {(int(a), int(b), c == b"1") for a, b, c in found}
    assert got == {(nqb, nvb, bf) for nqb in range(1, 9) for nvb in (1, 2) for bf in (False, True)}


@pytest.mark.parametrize("p", [0.1, 0.25, 0.5, 0.9, 1e-4, 0.999])
def test_survivor_scale_is_the_kernels_rule(p):
    assert ops._dropout_scale(p) == D.survivor_scale(p)


def _eager_drop(q, k, v, H, scale, pad, causal, keep, rp):
    """The reference's eager formula (modules.py:146-164) with nn.Dropout on the probabilities as attn * keep * rp."""
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    qh = q.expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2) * scale
    kh = k.reshape(B, M, H, -1).transpose(1, 2)
    vh = v.reshape(B, M, H, -1).transpose(1, 2)
    s = qh @ kh.transpose(-1, -2)
    neg = -torch.finfo(s.dtype).max
    if pad is not None:
        s = s.masked_fill(pad[:, None, None, :], neg)
    if causal:
        s = s.masked_fill(torch.ones(N, M, dtype=torch.bool).triu(M - N + 1), neg)
    attn = s.softmax(-1) * keep.to(s.dtype) * rp
    return (attn @ vh).transpose(1, 2).reshape(B, N, -1)


class _Ctx:
    pass


@pytest.mark.parametrize("dropout_p", [0.1, 0.5])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("with_stats", [False, True])
def test_dropout_shim_matches_autograd_on_the_oracle_mask(dropout_p, causal, with_stats, monkeypatch):
    """Batch-1 q, a pad mask with one fully padded row, head dims above 128 and 3 key chunks."""
    B, N, M, H, dqk, dv = 2, 6, 300, 2, 136, 160
    seed = 0x123456789A
    g = torch.Generator().manual_seed(3)
    q = torch.randn(1, N, H * dqk, generator=g, dtype=torch.float64, requires_grad=True)
    k = torch.randn(B, M, H * dqk, generator=g, dtype=torch.float64, requires_grad=True)
    v = torch.randn(B, M, H * dv, generator=g, dtype=torch.float64, requires_grad=True)
    pad = torch.zeros(B, M, dtype=torch.bool)
    pad[0, 230:] = True
    pad[1, :] = True
    scale = dqk ** -0.5
    keep = torch.from_numpy(D.keep_mask(B, H, N, M, dropout_p, seed))
    o = _eager_drop(q, k, v, H, scale, pad, causal, keep, D.survivor_scale(dropout_p))
    go = torch.randn(o.shape, generator=g, dtype=torch.float64)
    gq, gk, gv = torch.autograd.grad(o, (q, k, v), go)

    chunks = []

    def oracle_keep(B_, H_, N_, j0, j1, p_, seed_, device):
        assert (B_, H_, N_, p_, seed_) == (B, H, N, dropout_p, seed)
        chunks.append((j0, j1))
        return keep[..., j0:j1]

    monkeypatch.setattr(ops, "_dropout_keep", oracle_keep)
    monkeypatch.setattr(ops, "_compute_dtype", lambda dt: torch.float32)
    monkeypatch.setitem(ops.backward_config, "max_score_bytes", 4 * B * H * N * 128)   # 128-key chunks
    pm = pl = None
    if with_stats:  # the dropout-free statistics the forward kernel saves (log2 domain)
        qh = q.detach().float().expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
        kh = k.detach().float().reshape(B, M, H, -1).transpose(1, 2)
        t = (qh @ kh.transpose(-1, -2)) * (scale * 1.4426950408889634)
        neg = -torch.finfo(torch.float32).max
        t = t.masked_fill(pad[:, None, None, :], neg)
        if causal:
            t = t.masked_fill(torch.ones(N, M, dtype=torch.bool).triu(M - N + 1), neg)
        pm = t.amax(-1)
        pl = torch.exp2(t - pm[..., None]).sum(-1)
    ctx = _Ctx()
    ctx.saved_tensors = (q.detach().float(), k.detach().float(), v.detach().float(), pad, o.detach().float(), pm, pl)
    ctx.meta = (H, scale, causal)
    ctx.dropout = (dropout_p, seed)
    r = ops._FusedAttention.backward(ctx, go.float())
    assert chunks[-3:] == [(0, 128), (128, 256), (256, 300)]
    for got, ref, name in zip(r[:3], (gq, gk, gv), "qkv"):
        assert got.shape == ref.shape
        err = (got.double() - ref).abs().max().item()
        assert err <= 2e-5 * ref.abs().max().item(), (name, err, ref.abs().max().item())
    assert all(x is None for x in r[3:])
