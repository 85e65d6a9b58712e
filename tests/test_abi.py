"""CPU-side checks of the drop-in boundary: libpcv_attn.so loads without a GPU, exports every symbol
include/pcv_attn.h declares, and the ctypes mirrors in perceiver_io_b200/_lib.py have the exact C layout."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

from conftest import ROOT
from perceiver_io_b200 import _lib

HEADER = os.path.join(ROOT, "include", "pcv_attn.h")


def _declared_functions():
    text = open(HEADER).read()
    return sorted(set(re.findall(r"PCV_API\s+[\w\s\*]+?\b(pcv_\w+)\s*\(", text)))


def test_library_is_built_in_tree():
    assert os.path.exists(_lib.LIB_PATH), "run __graft_entry__.build() first"


def test_every_declared_symbol_is_exported():
    lib = _lib.lib()
    declared = _declared_functions()
    assert len(declared) >= 10
    assert sorted(_lib.EXPORTS) == declared
    for name in declared:
        assert hasattr(lib, name), name


def test_abi_version_2_and_error_string_without_gpu():
    lib = _lib.lib()
    assert lib.pcv_abi_version() == 2
    # no second-pass dropout forward: pcv_attn_fwd_partial_dropout + pcv_attn_combine are the dropout forward
    for name in ("pcv_attn_fwd_dropout", "pcv_attn_fwd_dropout_supported", "pcv_attn_fwd_dropout_workspace_bytes"):
        assert not hasattr(lib, name), name
    # argument validation happens before any CUDA call, so it is testable on a CPU-only box
    rc = lib.pcv_attn_fwd(None, None)
    assert rc == 1
    assert b"NULL" in lib.pcv_last_error()
    p = _lib.AttnParams()
    rc = lib.pcv_attn_fwd(ctypes.byref(p), None)
    assert rc == 1 and b"pointer" in lib.pcv_last_error()


def test_ctypes_layout_matches_header(tmp_path):
    structs = {
        "pcv_attn_params": _lib.AttnParams,
        "pcv_combine_params": _lib.CombineParams,
        "pcv_rotary_params": _lib.RotaryParams,
        "pcv_rescale_params": _lib.RescaleParams,
        "pcv_peer_combine_params": _lib.PeerCombineParams,
        "pcv_kv_append_params": _lib.KvAppendParams,
        "pcv_device_info": _lib.DeviceInfo,
        "pcv_kvproj_params": _lib.KvProjParams,
        "pcv_ln_stats_params": _lib.LnStatsParams,
        "pcv_merge_params": _lib.MergeParams,
        "pcv_shard_fuse": _lib.ShardFuse,
        "pcv_attn_bwd_params": _lib.AttnBwdParams,
    }
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(void){"]
    for cname, cls in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines.append("return 0;}")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-o", str(exe), str(src)])
    out = subprocess.check_output([str(exe)]).decode().split("\n")
    got = dict(l.split() for l in out if l)
    for cname, cls in structs.items():
        assert int(got[cname]) == ctypes.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, f"{cname}.{fname}"


def test_kv_project_validates_before_any_cuda_call():
    lib = _lib.lib()
    assert lib.pcv_kv_project(None, None) == 1 and b"NULL" in lib.pcv_last_error()
    assert lib.pcv_ln_stats(None, None) == 1 and b"NULL" in lib.pcv_last_error()
    p = _lib.KvProjParams()
    assert lib.pcv_kv_project(ctypes.byref(p), None) == 1 and b"NULL" in lib.pcv_last_error()


def test_ops_refuse_cpu_tensors():
    import torch
    from perceiver_io_b200 import ops

    q = torch.zeros(1, 4, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.attention(q, q, q, num_heads=1, scale=1.0)


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "perceiver_io_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), f


def test_backward_and_mask_entry_points_validate_before_any_cuda_call():
    """pcv_attn_bwd / pcv_attn_dropout_mask reject bad arguments on a CPU-only box (no launch)."""
    lib = _lib.lib()
    assert lib.pcv_attn_bwd(None, None) == 1 and b"NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_bwd_supported(None) == 0
    need = ctypes.c_size_t(0)
    assert lib.pcv_attn_bwd_workspace_bytes(None, ctypes.byref(need)) == 1
    p = _lib.AttnBwdParams()
    p.B, p.H, p.N, p.M, p.dqk, p.dv, p.dtype = 2, 4, 200, 1000, 64, 64, _lib.AttnParams().dtype
    p.q_stride_b = 1  # non-zero: one latent array per batch row
    assert lib.pcv_attn_bwd_workspace_bytes(ctypes.byref(p), ctypes.byref(need)) == 0
    # statistics blocks (768 B per 64 queries) + fp32 dQ accumulator, each rounded up to 256 bytes
    stats = 768 * 2 * 4 * 4
    dq32 = 4 * 2 * 200 * 4 * 64
    assert need.value == (stats + 255) // 256 * 256 + (dq32 + 255) // 256 * 256
    assert lib.pcv_attn_dropout_mask(None, 1, 1, 8, 8, ctypes.c_float(0.1), ctypes.c_uint64(1), None) == 1
    assert b"dropout_mask" in lib.pcv_last_error()
