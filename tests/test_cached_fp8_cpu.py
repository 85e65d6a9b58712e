"""CPU checks of the tensor-core attention on an FP8 KV cache (pcv_attn_cached_fp8, the whole-cache instantiations of
attn_cached_kernel in csrc/pcv_attn_cached.cu): its entry points refuse what they do not cover before any CUDA call, the
workspace and the split plan are the restated ones of cached_fp8_variants.py, the variant matrix of the GPU tests reaches
every instantiation, the build of the kernel has no spills and no serialised wgmma, the host route picks the kernel by
query rows, and the CPU emulation of the kernel's arithmetic stays within half of the element-wise gate of
test_gpu_cached_fp8.py."""
import ctypes
import os
import re

import pytest
import torch

import cached_fp8_variants as CV
from conftest import ROOT
from perceiver_io_b200 import _lib, ops

F8 = torch.float8_e4m3fn


def _params(N=8, M=300, dqk=64, dv=64, impl=_lib.PCV_IMPL_AUTO, B=2, H=2):
    p = _lib.AttnParams()
    p.q, p.k, p.v, p.out = 1 << 20, 2 << 20, 3 << 20, 4 << 20  # never dereferenced: the checks run first
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.q_stride_b, p.q_stride_n, p.q_stride_h = N * H * dqk, H * dqk, dqk
    p.k_stride_b, p.k_stride_m, p.k_stride_h = M * H * dqk, H * dqk, dqk
    p.v_stride_b, p.v_stride_m, p.v_stride_h = M * H * dv, H * dv, dv
    p.o_stride_b, p.o_stride_n, p.o_stride_h = N * H * dv, H * dv, dv
    p.scale, p.dtype, p.m_total, p.impl = 0.125, _lib.PCV_BF16, M, impl
    f = _lib.DecodeFp8()
    f.k_descale, f.v_descale = 5 << 20, 6 << 20
    return p, f


def _refine(p, f, what):
    if what == "partial":
        p.write_partial = 1
        p.part_o = p.part_m = p.part_l = 8 << 20
    elif what == "shard":
        p.m_total, p.m_offset = p.M + 100, 100
    elif what == "k_stride":
        p.k_stride_m = p.H * p.dqk + 8
    elif what == "v_stride":
        p.v_stride_b = p.M * p.H * p.dv + 8
    elif what == "q_stride":
        p.q_stride_n = p.H * p.dqk + 4
    elif what == "q_align":
        p.q = (1 << 20) + 8
    elif what == "k_align":
        p.k = (2 << 20) + 4
    elif what == "k_descale":
        f.k_descale = None
    elif what == "v_descale":
        f.v_descale = None
    elif what == "q_dtype":
        p.dtype = _lib.PCV_E4M3
    return p, f


REFUSALS = [
    ({"N": 65}, None, b"more than 64 query rows"),
    ({"dqk": 40}, None, b"multiples of 16"),
    ({"dv": 24}, None, b"multiples of 16"),
    ({"dqk": 272}, None, b"head dim > 256"),
    ({"dv": 272}, None, b"head dim > 256"),
    ({"impl": _lib.PCV_IMPL_DECODE}, None, b"impl must be AUTO"),
    ({"impl": _lib.PCV_IMPL_TCGEN05}, None, b"impl must be AUTO"),
    ({}, "partial", b"no write_partial"),
    ({}, "shard", b"no key shard"),
    ({}, "k_stride", b"multiples of 16 elements"),
    ({}, "v_stride", b"multiples of 16 elements"),
    ({}, "q_stride", b"multiples of 8 elements"),
    ({}, "q_align", b"16-byte aligned"),
    ({}, "k_align", b"16-byte aligned"),
    ({}, "k_descale", b"NULL"),
    ({}, "v_descale", b"NULL"),
    ({}, "q_dtype", b"e4m3 operands"),
]


@pytest.mark.parametrize("kw,what,reason", REFUSALS)
def test_cached_fp8_refusals_without_gpu(kw, what, reason):
    lib = _lib.lib()
    p, f = _refine(*_params(**kw), what)
    assert lib.pcv_attn_cached_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert reason in lib.pcv_last_error()
    assert lib.pcv_attn_cached_fp8(ctypes.byref(p), ctypes.byref(f), None) != 0
    assert reason in lib.pcv_last_error()


def test_cached_fp8_null_arguments():
    lib = _lib.lib()
    p, f = _params()
    assert lib.pcv_attn_cached_fp8_supported(ctypes.byref(p), None) == 0
    assert b"fp8 params are NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_cached_fp8(ctypes.byref(p), None, None) != 0
    assert lib.pcv_attn_cached_fp8_supported(None, ctypes.byref(f)) == 0
    assert b"params is NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_cached_fp8_workspace_bytes(ctypes.byref(p), None) != 0
    assert b"bytes is NULL" in lib.pcv_last_error()


@pytest.mark.parametrize("N,M,dqk,dv,dtype", [(1, 1, 16, 16, _lib.PCV_BF16), (5, 300, 96, 96, _lib.PCV_F16),
                                              (64, 16384, 128, 128, _lib.PCV_BF16), (64, 7, 256, 256, _lib.PCV_F16),
                                              (33, 100, 256, 16, _lib.PCV_BF16)])
def test_cached_fp8_accepts_its_range(N, M, dqk, dv, dtype):
    lib = _lib.lib()
    p, f = _params(N=N, M=M, dqk=dqk, dv=dv)
    p.dtype = dtype
    assert lib.pcv_attn_cached_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 1, lib.pcv_last_error()


def test_decode_entries_keep_refusing_more_than_four_rows():
    lib = _lib.lib()
    p, f = _params(N=5)
    p.impl = _lib.PCV_IMPL_DECODE
    assert lib.pcv_attn_decode_fp8_supported(ctypes.byref(p), ctypes.byref(f)) == 0
    assert b"more than 4 query rows" in lib.pcv_last_error()


@pytest.mark.parametrize("B,H,N,M,dqk,dv", [(1, 1, 1, 1, 16, 16), (2, 2, 8, 300, 64, 64), (8, 8, 64, 16384, 128, 128),
                                            (3, 2, 63, 805, 96, 96), (16, 12, 16, 6144, 96, 96),
                                            (1, 1, 5, 65536, 256, 256), (4, 3, 17, 1000, 256, 48)])
def test_workspace_matches_the_restatement(B, H, N, M, dqk, dv):
    lib = _lib.lib()
    p, _ = _params(N=N, M=M, dqk=dqk, dv=dv, B=B, H=H)
    need = ctypes.c_size_t(0)
    assert lib.pcv_attn_cached_fp8_workspace_bytes(ctypes.byref(p), ctypes.byref(need)) == 0
    assert need.value == CV.workspace_bytes(B, H, N, M, dqk, dv, CV.device_sms())


@pytest.mark.parametrize("sms", [132, 114, 78])
@pytest.mark.parametrize("B,H,M", [(1, 1, 1), (1, 1, 63), (2, 2, 65), (3, 2, 805), (8, 8, 16384), (1, 1, 65536),
                                   (16, 12, 6144), (1, 1, 100000)])
@pytest.mark.parametrize("dqk,dv", [(16, 16), (96, 96), (128, 128), (256, 256), (192, 64)])
def test_split_plan_covers_every_key_once(sms, B, H, M, dqk, dv):
    pl = CV.plan(B, H, M, dqk, dv, sms)
    ranges = CV.split_ranges(M, pl)
    assert len(ranges) == pl["nsplit"] <= CV.MAX_SPLITS
    covered = []
    for kb, ke in ranges:
        assert kb % CV.KEYS == 0 and ke > kb, (kb, ke)   # whole tiles, no empty split
        covered += range(kb, ke)
    assert covered == list(range(M))
    tail = M - (pl["tiles"] - 1) * CV.KEYS
    assert 1 <= tail <= CV.KEYS
    if pl["nsplit"] > 1:
        assert pl["tiles_per_split"] >= CV.MIN_TILES
    assert 2 <= pl["stages"] <= CV.MAX_STAGES
    assert pl["smem"] <= (CV.PAIR_BUDGET if pl["per_sm"] == 2 else CV.SMEM_LIMIT)


def test_split_edge_shape_has_its_structure():
    """SPLIT_M at EDGE_B x EDGE_H: three splits of five tiles on any SM count, the last split three tiles and its last
    tile 37 keys."""
    for sms in (132, 114, 78, 66):
        for dqk, dv in {(d, v) for _, d, v in CV.VARIANT_CASES}:
            pl = CV.plan(CV.EDGE_B, CV.EDGE_H, CV.SPLIT_M, dqk, dv, sms)
            assert (pl["nsplit"], pl["tiles_per_split"]) == (3, 5), pl
            assert CV.split_ranges(CV.SPLIT_M, pl)[-1] == (640, 805)
            assert CV.SPLIT_M % CV.KEYS == 37


def test_variant_matrix_reaches_every_instantiation():
    reach = CV.reachable_variants()
    assert len(reach) == 8
    cover = {}
    for case in CV.VARIANT_CASES:
        cover.setdefault(CV.variant_of(case[0], case[2]), []).append(CV.case_id(case))
    assert set(cover) == reach, reach - set(cover)
    # GiantMIDI's head dims (96 / 96) and the benchmark's (128 / 128) are among the GPU cases
    assert {(96, 96), (128, 80)} <= {(d, v) for _, d, v in CV.VARIANT_CASES}


def cached_kernel_entries(win):
    """The ptxas log entries of attn_cached_kernel<BF16, FP8, WIN, NVB> with the given WIN, and the log's text; None
    when the library was not built in this tree."""
    log = os.path.join(ROOT, "build", "pcv_attn_cached.ptxas.log")
    if not os.path.exists(log):
        return None, None
    text = open(log).read()
    entries = text.split("Compiling entry function")[1:]
    args = [(re.search(r"attn_cached_kernelILb([01])ELb([01])ELb([01])ELi([1-4])E", e.split("\n")[0]), e)
            for e in entries]
    assert sum(m is not None for m, _ in args) == 24   # 8 whole-cache + 16 window instantiations, nothing else
    return [e for m, e in args if m is not None and m.group(3) == str(int(win))], text


def test_whole_cache_instantiations_have_no_spills_and_no_serialised_wgmma():
    kernels, text = cached_kernel_entries(win=False)
    if kernels is None:
        pytest.skip("the library was not built in this tree")
    assert len(kernels) == 8, len(kernels)
    for e in kernels:
        assert "ELb1ELb0ELi" in e.split("\n")[0]   # e4m3 rows only
        assert "0 bytes spill stores, 0 bytes spill loads" in e, e[:300]
    assert "C7515" not in text and "C7512" not in text


def test_route_picks_the_kernel_by_query_rows():
    from perceiver_io_b200 import modules

    assert ops.DECODE_MAX_ROWS == 4 and modules.KV8_MAX_ROWS == 64
    f = _lib.DecodeFp8()
    for N, entry in ((1, "pcv_attn_decode_fp8"), (4, "pcv_attn_decode_fp8"), (5, "pcv_attn_cached_fp8"),
                     (64, "pcv_attn_cached_fp8"), (65, "pcv_attn_cached_fp8")):
        p, _ = _params(N=N, impl=_lib.PCV_IMPL_DECODE)
        assert ops._fp8_entry(p, f, None) == entry
        assert p.impl == (_lib.PCV_IMPL_AUTO if N > 4 else _lib.PCV_IMPL_DECODE)
    p, _ = _params(N=8, impl=_lib.PCV_IMPL_DECODE)
    assert ops._fp8_entry(p, f, object()) == "pcv_attn_decode_window_fp8"   # windows keep the decode entry
    assert ops._fp8_entry(p, None, None) == "pcv_attn_decode"


EMU_CASES = [(case, N, M, causal) for case in CV.VARIANT_CASES for N, M, causal in
             ((5, 65, True), (64, 130, False), (8, CV.SPLIT_M, True))]


@pytest.mark.parametrize("case,N,M,causal", EMU_CASES,
                         ids=[f"{CV.case_id(c)}-n{N}-m{M}-{'causal' if cz else 'full'}" for c, N, M, cz in EMU_CASES])
def test_emulation_stays_within_half_the_gate(case, N, M, causal):
    """The kernel's arithmetic (cached_fp8_variants.emulate) against fp64 attention on the dequantised codes: at most
    half of the element-wise gate of the GPU tests, with left padding and a wholly padded batch row."""
    dt, dqk, dv = case
    B, H = 3, 2
    q, k8, v8, kd, vd = CV.random_operands(B, B, N, M, H, dqk, dv, dt, seed=N + M + dqk)
    pad = CV.left_pad(B, M)
    got = CV.emulate(q, k8, v8, kd, vd, H, 0.3, pad, causal, dt)
    kq, vq = ops.fp8_dequantize(k8, kd, H, torch.float64), ops.fp8_dequantize(v8, vd, H, torch.float64)
    depth = CV.serial_depth(CV.plan(B, H, M, dqk, dv))
    bound, ref = CV.element_bound(q, kq, vq, H, 0.3, pad, causal, CV.DTYPE[dt], depth)
    ratio = ((got.double() - ref).abs() / bound).max().item()
    print(f"[emulation] {CV.case_id(case)} N={N} M={M} causal={causal}: worst err / gate {ratio:.3f}")
    assert ratio <= 0.5, ratio
