"""CPU-side checks of the LayerNorm -> Linear backward (pcv_ln_linear_bwd): symbols and struct layout, argument checks
before any CUDA call, the workspace formula (no device needed), and an fp64 restatement of exactly the decomposition
the kernels compute, against fp64 autograd of LayerNorm -> Linear."""
import ctypes
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT
from perceiver_io_b200 import _lib

HEADER = os.path.join(ROOT, "include", "pcv_attn.h")
NEW = ("pcv_ln_linear_bwd_supported", "pcv_ln_linear_bwd_workspace_bytes", "pcv_ln_linear_bwd")


def test_new_symbols_are_declared_and_exported():
    text = open(HEADER).read()
    lib = _lib.lib()
    for name in NEW:
        assert name in _lib.EXPORTS and name in text
        assert hasattr(lib, name)


def test_struct_layout_matches_header(tmp_path):
    cls = _lib.LnLinearBwdParams
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{HEADER}"', "int main(void){",
             'printf("size %zu\\n", sizeof(pcv_ln_linear_bwd_params));']
    lines += [f'printf("{f} %zu\\n", offsetof(pcv_ln_linear_bwd_params, {f}));' for f, _ in cls._fields_]
    lines.append("return 0;}")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-o", str(exe), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)]).decode().split("\n") if l)
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def _valid_params(rows=1000, C=1024, n_k=1024, n_v=1024):
    """Plausible (never dereferenced) 16-byte aligned addresses for every pointer."""
    p = _lib.LnLinearBwdParams()
    addr = iter(range(0x10000, 0x10000 + 0x1000 * 20, 0x1000))
    p.x, p.row_stats, p.w, p.gamma, p.beta = (next(addr) for _ in range(5))
    p.grad_k, p.grad_v = next(addr), next(addr)
    p.grad_x, p.grad_w, p.grad_b, p.grad_gamma, p.grad_beta = (next(addr) for _ in range(5))
    p.x_stride_row, p.gk_stride_row, p.gv_stride_row = C, n_k, n_v
    p.rows, p.C, p.n_k, p.n_v, p.dtype = rows, C, n_k, n_v, _lib.PCV_BF16
    p.workspace, p.workspace_bytes = next(addr), 1 << 40
    return p


@pytest.mark.parametrize("change, reason", [
    (dict(row_stats=None), b"row_stats"),
    (dict(C=12, x_stride_row=16), b"multiple of 8"),
    (dict(n_k=32, gk_stride_row=32), b"K width"),
    (dict(n_v=12, gv_stride_row=16), b"V width"),
    (dict(dtype=_lib.PCV_F32), b"dtype"),
    (dict(grad_k=None), b"grad_k"),
    (dict(grad_x=None, grad_w=None, grad_b=None, grad_gamma=None, grad_beta=None), b"no gradient"),
    (dict(x=0x10008), b"aligned"),
    (dict(x_stride_row=1020), b"strides"),
    (dict(rows=0), b"row count"),
])
def test_bad_arguments_are_rejected_before_any_cuda_call(change, reason):
    lib = _lib.lib()
    assert lib.pcv_ln_linear_bwd(None, None) == 1 and b"NULL" in lib.pcv_last_error()
    p = _valid_params()
    for k, v in change.items():
        setattr(p, k, v)
    assert lib.pcv_ln_linear_bwd(ctypes.byref(p), None) != 0
    assert b"ln_linear_bwd" in lib.pcv_last_error() and reason in lib.pcv_last_error(), lib.pcv_last_error()
    assert lib.pcv_ln_linear_bwd_supported(ctypes.byref(p)) == 0
    assert reason in lib.pcv_last_error()


def test_too_small_workspace_is_rejected_before_any_cuda_call():
    lib = _lib.lib()
    p = _valid_params()
    p.workspace_bytes = 256
    assert lib.pcv_ln_linear_bwd(ctypes.byref(p), None) == 4 and b"workspace" in lib.pcv_last_error()
    p.workspace_bytes = 1 << 40
    p.workspace = 0x10010  # 16- but not 256-byte aligned
    assert lib.pcv_ln_linear_bwd(ctypes.byref(p), None) == 4 and b"workspace" in lib.pcv_last_error()


def _up(b):
    return (b + 255) // 256 * 256


def workspace_formula(rows, C, n_k, n_v):
    """Row partials (128-channel tiles x rows float2), column partials (128-row blocks x C float2), dW split partials
    (splits x n x C f32) and db split partials (splits x n f32), each rounded up to 256 bytes.  The split count fills
    two CTAs per SM of a 132-SM H100 with the (128 x 128) output tiles, at most 32 and at most one per 64 rows."""
    n = n_k + n_v
    tiles = -(-C // 128) * -(-n // 128)
    kb_rows = -(-rows // 64)
    splits = max(1, min(264 // tiles, 32, kb_rows))
    return (_up(-(-C // 128) * rows * 8) + _up(-(-rows // 128) * C * 8) + _up(splits * n * C * 4) + _up(splits * n * 4))


@pytest.mark.parametrize("rows, C, n_k, n_v", [(1000, 1024, 1024, 1024), (4096, 768, 256, 1280), (300, 64, 64, 72),
                                              (513, 72, 128, 8), (2048, 512, 512, 0), (524288, 1024, 1024, 1024)])
def test_workspace_bytes_follow_the_formula_without_a_device(rows, C, n_k, n_v):
    lib = _lib.lib()
    p = _valid_params(rows, C, n_k, n_v)
    need = ctypes.c_size_t(0)
    assert lib.pcv_ln_linear_bwd_workspace_bytes(ctypes.byref(p), ctypes.byref(need)) == 0
    assert need.value == workspace_formula(rows, C, n_k, n_v)
    # the size depends on the problem alone: pointers, strides and dtype do not move it
    p.x, p.dtype, p.grad_x = 0x20000, _lib.PCV_F16, None
    again = ctypes.c_size_t(0)
    assert lib.pcv_ln_linear_bwd_workspace_bytes(ctypes.byref(p), ctypes.byref(again)) == 0
    assert again.value == need.value


# ----------------------------------------------------------------------------------------------------------------
# fp64 restatement of the kernels' decomposition
# ----------------------------------------------------------------------------------------------------------------
def decomposed_grads(x, gamma, beta, w, G, eps=1e-5, tile=128, splits=3):
    """What pcv_ln_linear_bwd computes, step by step, in fp64: dy = G W with per-(row, 128-column tile) partials of
    sum dx_hat and sum dx_hat * x_hat summed in tile order (two-phase dx); P^T = x_hat^T G as row-split partials plus
    the rank-1 beta term; db as row-split column sums of G; dgamma / dbeta as 128-row block partials."""
    R, C = x.shape
    mean = x.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(1, keepdim=True) + eps)
    xh = (x - mean) * rstd
    g = torch.ones(C, dtype=x.dtype) if gamma is None else gamma
    b = torch.zeros(C, dtype=x.dtype) if beta is None else beta
    dy = G @ w
    dxh = dy * g
    a = sum(dxh[:, c:c + tile].sum(1) for c in range(0, C, tile))
    bb = sum((dxh * xh)[:, c:c + tile].sum(1) for c in range(0, C, tile))
    dx = rstd * (dxh - (a[:, None] + xh * bb[:, None]) / C)
    bounds = [R * s // splits for s in range(splits + 1)]
    pt = sum(xh[r0:r1].T @ G[r0:r1] for r0, r1 in zip(bounds, bounds[1:]))           # (C, n)
    db = sum(G[r0:r1].sum(0) for r0, r1 in zip(bounds, bounds[1:]))
    dw = pt.T * g[None, :] + db[:, None] * b[None, :]
    dgamma = sum((dy * xh)[r:r + tile].sum(0) for r in range(0, R, tile))
    dbeta = sum(dy[r:r + tile].sum(0) for r in range(0, R, tile))
    return dx, dw, db, dgamma, dbeta


@pytest.mark.parametrize("affine, bias, n_k, n_v, C", [
    (True, True, 128, 72, 200),     # C tail (not a multiple of 64 or 128), V width not a multiple of 64
    (False, True, 64, 64, 96),      # LayerNorm without affine part
    (True, False, 64, 8, 136),      # Linear without bias
    (True, True, 192, 0, 264),      # K only
])
def test_decomposition_matches_fp64_autograd(affine, bias, n_k, n_v, C):
    torch.manual_seed(0)
    R, n = 300, n_k + n_v
    x = (torch.randn(R, C, dtype=torch.float64) * 1.3 + 20.0).requires_grad_()
    gamma = (torch.rand(C, dtype=torch.float64) + 0.5).requires_grad_() if affine else None
    beta = (torch.randn(C, dtype=torch.float64) * 30.0).requires_grad_() if affine else None
    w = (torch.randn(n, C, dtype=torch.float64) / C ** 0.5).requires_grad_()
    b = torch.randn(n, dtype=torch.float64).requires_grad_() if bias else None
    G = torch.randn(R, n, dtype=torch.float64)
    out = F.linear(F.layer_norm(x, (C,), gamma, beta, 1e-5), w, b)
    out.backward(G)
    dx, dw, db, dgamma, dbeta = decomposed_grads(x.detach(), None if gamma is None else gamma.detach(),
                                                 None if beta is None else beta.detach(), w.detach(), G)
    pairs = [("dx", dx, x.grad), ("dW", dw, w.grad)]
    if bias:
        pairs.append(("db", db, b.grad))
    if affine:
        pairs += [("dgamma", dgamma, gamma.grad), ("dbeta", dbeta, beta.grad)]
    for name, got, want in pairs:
        err = (got - want).abs().max().item() / want.abs().max().item()
        assert err <= 1e-12, f"{name}: relative error {err:.3e}"


def test_incoming_gradients_are_given_a_row_stride_the_kernels_take():
    """A gradient broadcast along the rows (row stride 0), a transposed one and an unaligned view are copied to
    (rows, n) rows with a row stride that covers the row; a usable slice is passed through as is."""
    from perceiver_io_b200 import ops

    n = 16
    bc = ops._gemm_rows(torch.ones(n, dtype=torch.bfloat16).expand(4, n), n)
    assert bc.stride() == (n, 1) and torch.equal(bc, torch.ones(4, n, dtype=torch.bfloat16))
    tr = torch.randn(n, 4).to(torch.bfloat16).t()
    assert ops._gemm_rows(tr, n).stride() == (n, 1)
    base = torch.randn(4, 3 * n).to(torch.bfloat16)
    view = base[:, n:2 * n]
    out = ops._gemm_rows(view, n)
    assert out.data_ptr() % 16 == 0 and out.stride(0) >= n and torch.equal(out, view)
