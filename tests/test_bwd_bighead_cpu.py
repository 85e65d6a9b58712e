"""CPU checks of the attention backward for head dims up to 192: the kernel instantiations in the library, the
argument checks of pcv_attn_bwd_supported (before any CUDA call), and the zero-padding of head dims that are not
multiples of 8 around the backward kernels, with an fp64 CPU stand-in for the kernels."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

from conftest import ROOT
from perceiver_io_b200 import _lib, ops


def _lib_blob():
    with open(_lib.LIB_PATH, "rb") as f:
        return f.read()


def test_library_holds_exactly_the_backward_instantiations_with_one_dq_template():
    """bwd_dkdv_kernel<NQB, NVB, BF16, OUT>: the single-pass kernels (OUT 0) for NQB, NVB <= 2; for the five box pairs
    with a third box, a dV pass (OUT 1) and a dK pass (OUT 2).  bwd_dq_kernel<NQB, NVB, BF16, KS>: 128-key stages at
    <= 2 boxes, 64-key stages for the five wide pairs; no other dQ or dQ-cast kernel."""
    blob = _lib_blob()
    small = {(q, v) for q in (1, 2) for v in (1, 2)}
    wide = {(q, v) for q in (1, 2, 3) for v in (1, 2, 3)} - small
    assert len(wide) == 5
    dkdv = {(int(a), int(b), c == b"1", int(o))
            for a, b, c, o in re.findall(rb"15bwd_dkdv_kernelILi(\d)ELi(\d)ELb([01])ELi(\d)EEEv", blob)}
    assert dkdv == ({(q, v, bf, 0) for q, v in small for bf in (False, True)}
                    | {(q, v, bf, o) for q, v in wide for bf in (False, True) for o in (1, 2)})
    dq = {(int(a), int(b), c == b"1", int(k))
          for a, b, c, k in re.findall(rb"13bwd_dq_kernelILi(\d)ELi(\d)ELb([01])ELi(\d+)EEEv", blob)}
    assert dq == ({(q, v, bf, 128) for q, v in small for bf in (False, True)}
                  | {(q, v, bf, 64) for q, v in wide for bf in (False, True)})
    assert b"bwd_dq64_kernel" not in blob and b"bwd_cast_dq_kernel" not in blob


# ptxas at the commit that folded the two dQ kernels into one (CUDA 12.9, the Makefile's flags): (stack, spill stores,
# spill loads) bytes of the kernels that spill; every other backward kernel is spill-free.  All use 168 registers
# (384-thread CTAs, one per SM).
BWD_SPILLS = {f"bwd_{k}<2, 2, {bf}, {x}>": v for bf in ("false", "true")
              for k, x, v in (("dkdv_kernel", 0, (40, 52, 56)), ("dq_kernel", 128, (24, 28, 52)))}


def test_backward_kernels_hold_their_registers_and_spills():
    log = os.path.join(ROOT, "build", "pcv_attn_bwd.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was not built in this tree")
    text = open(log).read()
    seen = set()
    for e in text.split("Compiling entry function")[1:]:
        mangled = e.split("'")[1]
        if not re.search(r"bwd_(dkdv|dq)_kernel", mangled):
            continue
        name = subprocess.run(["c++filt", mangled], capture_output=True, text=True).stdout
        name = re.sub(r"^void (pcv::\(anonymous namespace\)::)?", "", name.split("(CUtensorMap")[0].strip())
        seen.add(name)
        own = next(line for line in e.split("\n") if "spill" in line)   # the kernel's own line, not a callee's
        stack, stores, loads = map(int, re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill "
                                                   r"loads", own).groups())
        limit = BWD_SPILLS.get(name, (0, 0, 0))
        assert stack <= limit[0] and stores <= limit[1] and loads <= limit[2], (name, own)
        assert int(e.split("Used ")[1].split(" registers")[0]) == 168, (name, e[:300])
    assert len(seen) == 2 * (4 + 5 * 2) + 2 * 9, sorted(seen)   # dK/dV kernels, then the dQ kernels
    assert set(BWD_SPILLS) <= seen


def _bwd_params(dqk, dv, **kw):
    """pcv_attn_bwd_params with fake, never dereferenced, 16-byte aligned pointers and dense strides."""
    p = _lib.AttnBwdParams()
    B, H, N, M = 2, 8, 256, 1024
    p.q = p.k = p.v = p.out = p.grad_out = p.grad_q = p.grad_k = p.grad_v = 1 << 20
    p.stat_m = p.stat_l = 1 << 21
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.q_stride_b, p.q_stride_n, p.q_stride_h = 0, H * dqk, dqk
    p.k_stride_b, p.k_stride_m, p.k_stride_h = M * H * dqk, H * dqk, dqk
    p.v_stride_b, p.v_stride_m, p.v_stride_h = M * H * dv, H * dv, dv
    p.o_stride_b, p.o_stride_n, p.o_stride_h = N * H * dv, H * dv, dv
    p.go_stride_b, p.go_stride_n, p.go_stride_h = N * H * dv, H * dv, dv
    p.gq_stride_b, p.gq_stride_n, p.gq_stride_h = N * H * dqk, H * dqk, dqk
    p.gk_stride_b, p.gk_stride_m, p.gk_stride_h = M * H * dqk, H * dqk, dqk
    p.gv_stride_b, p.gv_stride_m, p.gv_stride_h = M * H * dv, H * dv, dv
    p.scale, p.dtype = dqk ** -0.5, _lib.PCV_BF16
    for name, value in kw.items():
        setattr(p, name, value)
    return p


def _reason(p):
    lib = _lib.lib()
    ok = lib.pcv_attn_bwd_supported(ctypes.byref(p))
    return ok, lib.pcv_last_error()


@pytest.mark.parametrize("dqk, dv", [(192, 192), (32, 160), (136, 136), (160, 32), (136, 192), (72, 184)])
def test_supported_reaches_the_device_check_for_head_dims_up_to_192(dqk, dv):
    """Without a GPU the only reason left is the device: the head-dim checks pass."""
    ok, why = _reason(_bwd_params(dqk, dv))
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the device check passes")
    assert ok == 0
    assert b"head dims" not in why and b"attn_bwd not applicable" in why, why


@pytest.mark.parametrize("dqk, dv, msg", [
    (200, 200, b"head dims must be in [8, 192]"),
    (264, 264, b"head dims must be in [8, 192]"),
    (32, 200, b"head dims must be in [8, 192]"),
    (196, 32, b"head dims must be multiples of 8"),
    (196, 196, b"head dims must be multiples of 8"),
])
def test_supported_rejects_head_dims_without_a_cuda_call(dqk, dv, msg):
    ok, why = _reason(_bwd_params(dqk, dv))
    assert ok == 0 and msg in why, why


def test_wide_workspace_holds_the_dq_partials():
    """Above 128 the workspace grows by one fp32 dQ partial per (batch contribution, split); it is computed without
    the device (the split of the wide dQ kernel does not depend on the SM count)."""
    lib = _lib.lib()
    sizes = {}
    for dqk, dv in ((128, 128), (136, 136)):
        need = ctypes.c_size_t(0)
        assert lib.pcv_attn_bwd_workspace_bytes(ctypes.byref(_bwd_params(dqk, dv)), ctypes.byref(need)) == 0
        sizes[dqk] = need.value
    one_dq = 4 * 1 * 256 * 8 * 136                  # batch-1 q: (1, N, H*dqk) fp32
    assert sizes[136] >= 2 * one_dq                 # B = 2 contributions, at least one split each
    assert sizes[136] > sizes[128]


# ---- padding of odd head dims around the kernels --------------------------------------------------------------
def _eager(q, k, v, H, scale, pad, causal):
    """The reference's eager formula (modules.py:146-164)."""
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
    return (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, N, -1)


def _stats(q, k, H, scale, pad, causal):
    """part_m / part_l of the forward kernel (log2 domain), fp64."""
    B, M, N = k.shape[0], k.shape[1], q.shape[1]
    qh = q.expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = k.reshape(B, M, H, -1).transpose(1, 2)
    t = (qh @ kh.transpose(-1, -2)) * (scale * 1.4426950408889634)
    neg = -torch.finfo(t.dtype).max
    if pad is not None:
        t = t.masked_fill(pad[:, None, None, :], neg)
    if causal:
        t = t.masked_fill(torch.ones(N, M, dtype=torch.bool).triu(M - N + 1), neg)
    m = t.amax(-1)
    return m, torch.exp2(t - m[..., None]).sum(-1)


@pytest.mark.parametrize("with_pad", [False, True])
@pytest.mark.parametrize("causal", [False, True])
def test_odd_head_dims_are_padded_around_the_backward_kernels(with_pad, causal, monkeypatch):
    """131 / 131 (the image classifier's encoder cross-attention), batch-1 q: the operands reach the kernels padded to
    136 per head with zeros, and the gradients that come back equal fp64 autograd of the unpadded eager formula."""
    B, N, M, H, d = 2, 5, 40, 2, 131
    g = torch.Generator().manual_seed(5)
    q = torch.randn(1, N, H * d, generator=g, dtype=torch.float64, requires_grad=True)
    k = torch.randn(B, M, H * d, generator=g, dtype=torch.float64, requires_grad=True)
    v = torch.randn(B, M, H * d, generator=g, dtype=torch.float64, requires_grad=True)
    pad = None
    if with_pad:
        pad = torch.zeros(B, M, dtype=torch.bool)
        pad[0, 29:] = True
        pad[1, 3:] = True
    scale = d ** -0.5
    o = _eager(q, k, v, H, scale, pad, causal)
    go = torch.randn(o.shape, generator=g, dtype=torch.float64)
    ref = torch.autograd.grad(o, (q, k, v), go)
    pm, pl = _stats(q.detach(), k.detach(), H, scale, pad, causal)

    def fp64_kernels(q_, k_, v_, out_, go_, pm_, pl_, H_, scale_, pad_, causal_, dropout_p, dropout_seed, shard, mode):
        for t in (q_, k_, v_, out_, go_):
            assert t.dim() == 3 and t.shape[2] == H * 136
            assert (t.unflatten(2, (H, 136))[..., d:] == 0).all()
        assert pm_ is pm and pl_ is pl and pad_ is pad and causal_ == causal and scale_ == scale
        assert shard is None and mode == "try"
        qq, kk, vv = (t.detach().clone().requires_grad_() for t in (q_, k_, v_))
        oo = _eager(qq, kk, vv, H, scale_, pad_, causal_)
        # the kernels take out and delta = rowsum(dO * O) from their operands: the padded out must be the forward's
        assert torch.allclose(oo.detach(), out_, rtol=0, atol=1e-12)
        return torch.autograd.grad(oo, (qq, kk, vv), go_)

    monkeypatch.setattr(ops, "_backward_kernels", fp64_kernels)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "_compute_dtype", lambda dt: dt)  # the fp64 stand-in takes the fp64 operands
    got = ops._backward(q.detach(), k.detach(), v.detach(), o.detach(), go, pm, pl, H, scale, pad, causal, 0.0, 0)
    for gr, r, name in zip(got, ref, "qkv"):
        assert gr.shape == r.shape, name
        err = (gr - r).abs().max().item()
        assert err <= 1e-12 * max(1.0, r.abs().max().item()), (name, err)


def test_backward_route_declines_what_the_kernels_do_not_cover(monkeypatch):
    monkeypatch.setattr(ops, "_backward_kernels", lambda *a: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    q = torch.zeros(1, 3, 8 * 2)
    k = v = torch.zeros(1, 4, 8 * 2)
    assert ops._backward(q, k, v, q, q, None, None, 2, 1.0, None, False, 0.0, 0) is None
