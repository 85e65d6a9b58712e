"""CPU checks of the device-row entry points of the decode step (pcv_attn_decode_window (_fp8), pcv_kv_append_at (_fp8),
pcv_rotary_apply_at (_fp8)): for each input they do not cover, the status and the reason they give before any CUDA
call, and that the window decode sizes its workspace like the other decode entry points."""
import ctypes

import pytest

from perceiver_io_b200 import _lib

DEC, DEC8 = "pcv_attn_decode_window", "pcv_attn_decode_window_fp8"
APP, APP8 = "pcv_kv_append_at", "pcv_kv_append_at_fp8"
ROT, ROT8 = "pcv_rotary_apply_at", "pcv_rotary_apply_at_fp8"
OP = {DEC: "decode", DEC8: "decode", APP: "append", APP8: "append", ROT: "rotary", ROT8: "rotary"}
ACCEPT = "accept"  # the checks pass: a launch would run, so only a *_supported query is made


def _decode(N=1, dqk=64, dv=64):
    H, B, M = 2, 2, 300
    p = _lib.AttnParams()
    p.q, p.k, p.v, p.out = 1 << 20, 2 << 20, 3 << 20, 4 << 20  # never dereferenced: the checks run first
    p.B, p.H, p.N, p.M, p.dqk, p.dv = B, H, N, M, dqk, dv
    p.q_stride_b, p.q_stride_n, p.q_stride_h = N * H * dqk, H * dqk, dqk
    p.k_stride_b, p.k_stride_m, p.k_stride_h = M * H * dqk, H * dqk, dqk
    p.v_stride_b, p.v_stride_m, p.v_stride_h = M * H * dv, H * dv, dv
    p.o_stride_b, p.o_stride_n, p.o_stride_h = N * H * dv, H * dv, dv
    p.scale, p.dtype, p.m_total, p.impl = 0.125, _lib.PCV_BF16, M, _lib.PCV_IMPL_AUTO
    f = _lib.DecodeFp8()
    f.k_descale, f.v_descale = 5 << 20, 6 << 20
    return p, f


def _append(C=64):
    B, n, cap = 2, 1, 64
    p = _lib.KvAppendParams()
    p.k_new, p.v_new, p.k_dst, p.v_dst = (i << 20 for i in range(3, 7))
    p.kn_stride_b, p.kn_stride_l, p.vn_stride_b, p.vn_stride_l = n * C, C, n * C, C
    p.kd_stride_b, p.kd_stride_l, p.vd_stride_b, p.vd_stride_l = cap * C, C, cap * C, C
    p.B, p.L_old, p.n, p.Ck, p.Cv, p.dtype = B, 0, n, C, C, _lib.PCV_BF16
    f = _lib.KvFp8Scales()
    f.k_inv_scale, f.v_inv_scale = 7 << 20, 8 << 20
    return p, f


def _rotary(d=32):
    p = _lib.RotaryParams()
    p.x, p.y, p.angles = 1 << 20, 2 << 20, 3 << 20
    p.x_stride_b, p.x_stride_n, p.x_stride_h = 4 * 2 * d, 2 * d, d
    p.y_stride_b, p.y_stride_n, p.y_stride_h = 4 * 2 * d, 2 * d, d
    p.a_stride_n = d
    p.B, p.n, p.H, p.d, p.rotate_dim, p.dtype = 1, 4, 2, d, d, _lib.PCV_BF16
    f = _lib.RotaryFp8()
    f.y_inv_scale = 4 << 20
    return p, f


# case -> {entry point: (status of the launch entry point, reason substring) or ACCEPT}; the *_supported queries of the
# window decode return 0 with the same reason.  Entry points a case does not apply to are left out.
CASES = {
    "rows_null": {DEC: (1, b"rows is NULL"), DEC8: (1, b"rows"), APP: (1, b"kv_append_at: params or rows are NULL"),
                  APP8: (1, b"kv_append_at_fp8: params are NULL"), ROT: (1, b"rotary_at: params or rows are NULL"),
                  ROT8: (1, b"rotary_at_fp8: params are NULL")},
    "bounds_null": {DEC: (2, b"rows->bounds is NULL"), DEC8: (2, b"rows->bounds is NULL"),
                    APP: (1, b"kv_append_at: rows->bounds NULL"), APP8: (1, b"kv_append_at_fp8: rows->bounds NULL"),
                    ROT: (1, b"rotary_at: rows->bounds NULL"), ROT8: (1, b"rotary_at_fp8: rows->bounds NULL")},
    "capacity": {DEC: (2, b"M must equal rows->capacity"), DEC8: (2, b"M must equal rows->capacity"),
                 APP: (1, b"kv_append_at: rows->bounds NULL or capacity < 1"),
                 APP8: (1, b"kv_append_at_fp8: rows->bounds NULL or capacity < 1"),
                 ROT: (1, b"rotary_at: rows->bounds NULL or capacity < 1"),
                 ROT8: (1, b"rotary_at_fp8: rows->bounds NULL or capacity < 1")},
    "cache": {APP: (1, b"kv_append_at: an append at device rows takes no cache"),
              APP8: (1, b"kv_append_at_fp8: an append at device rows takes no cache")},
    "partial": {DEC: (2, b"window decode writes the normalised output only (no write_partial)"),
                DEC8: (2, b"window decode writes the normalised output only (no write_partial)")},
    "shard": {DEC: (2, b"window decode takes no key shard"), DEC8: (2, b"window decode takes no key shard")},
    "tcgen05": {DEC: (2, b"impl must be AUTO or DECODE"), DEC8: (2, b"impl must be AUTO or DECODE")},
    "n5": {DEC: (2, b"more than 4 query rows"), DEC8: (2, b"more than 4 query rows")},
    "bf16_head_dim_12": {DEC: (2, b"head dims must be multiples of 8"), DEC8: (2, b"head dims must be multiples of 16"),
                         APP: ACCEPT, APP8: (1, b"kv_append_fp8: Ck and Cv must be multiples of 16"), ROT: ACCEPT,
                         ROT8: ACCEPT},
    "e4m3_head_dim_40": {DEC: ACCEPT, DEC8: (2, b"head dims must be multiples of 16"), APP: ACCEPT,
                         APP8: (1, b"kv_append_fp8: Ck and Cv must be multiples of 16"), ROT: ACCEPT, ROT8: ACCEPT},
    "e4m3_k_stride": {DEC: ACCEPT, DEC8: (2, b"e4m3 k/v strides must be multiples of 16 elements"), APP: ACCEPT,
                      APP8: (1, b"kv_append_fp8: e4m3 strides must be multiples of 16 bytes")},
    "descale_null": {DEC8: (2, b"k_descale / v_descale are NULL"), APP8: (1, b"k_inv_scale / v_inv_scale are NULL"),
                     ROT8: (1, b"rotary_fp8: y_inv_scale is NULL")},
}


def _inputs(case, entry):
    """(params, fp8 params, rows or None) of `case` for `entry`."""
    op = OP[entry]
    hd = {"bf16_head_dim_12": 12, "e4m3_head_dim_40": 40}.get(case)
    if op == "decode":
        p, f = _decode(N=5 if case == "n5" else 1, **({"dqk": hd, "dv": hd} if hd else {}))
        cap = p.M
    elif op == "append":
        p, f = _append(**({"C": hd} if hd else {}))
        cap = 64
    else:
        p, f = _rotary(**({"d": hd} if hd else {}))
        cap = 64
    rows = _lib.DevRows()
    rows.bounds, rows.capacity = 9 << 20, cap
    if case == "rows_null":
        rows = None
    elif case == "bounds_null":
        rows.bounds = None
    elif case == "capacity":
        rows.capacity = p.M + 1 if op == "decode" else 0
    elif case == "cache":
        p.L_old, p.k_cache, p.v_cache = 10, 1 << 20, 2 << 20
        p.kc_stride_b, p.kc_stride_l, p.vc_stride_b, p.vc_stride_l = 64 * p.Ck, p.Ck, 64 * p.Cv, p.Cv
    elif case == "partial":
        p.write_partial = 1
        p.part_o = p.part_m = p.part_l = 8 << 20
    elif case == "shard":
        p.m_total, p.m_offset = p.M + 100, 100
    elif case == "tcgen05":
        p.impl = _lib.PCV_IMPL_TCGEN05
    elif case == "e4m3_k_stride":
        if op == "decode":
            p.k_stride_m = p.H * p.dqk + 8
        else:
            p.kd_stride_l = p.Ck + 8
    elif case == "descale_null":
        if op == "decode":
            f.v_descale = None
        elif op == "append":
            f.k_inv_scale = None
        else:
            f.y_inv_scale = None
    return p, f, rows


def _ref(x):
    return None if x is None else ctypes.byref(x)


def _supported(entry, p, f, rows):
    lib = _lib.lib()
    if entry == DEC:
        return lib.pcv_attn_decode_window_supported(_ref(p), _ref(rows))
    return lib.pcv_attn_decode_window_fp8_supported(_ref(p), _ref(f), _ref(rows))


def _launch(entry, p, f, rows):
    fn = getattr(_lib.lib(), entry)
    if entry in (DEC, APP, ROT):
        return fn(_ref(p), _ref(rows), None)
    return fn(_ref(p), _ref(f), _ref(rows), None)


TABLE = [(case, entry, want) for case, row in CASES.items() for entry, want in row.items()]


@pytest.mark.parametrize("case,entry,want", TABLE, ids=[f"{c}-{e}" for c, e, _ in TABLE])
def test_device_row_entry_points_refuse_before_any_cuda_call(case, entry, want):
    lib = _lib.lib()
    p, f, rows = _inputs(case, entry)
    if want == ACCEPT:
        if entry in (DEC, DEC8):
            assert _supported(entry, p, f, rows) == 1, lib.pcv_last_error()
        return
    status, reason = want
    if entry in (DEC, DEC8):
        assert _supported(entry, p, f, rows) == 0
        assert reason in lib.pcv_last_error()
    assert _launch(entry, p, f, rows) == status, lib.pcv_last_error()
    assert reason in lib.pcv_last_error()


@pytest.mark.parametrize("entry", [DEC, DEC8])
def test_window_decode_covers_the_base_params(entry):
    assert _supported(entry, *_inputs(None, entry)) == 1, _lib.lib().pcv_last_error()


def test_window_decode_fp8_refuses_null_fp8_params():
    lib = _lib.lib()
    p, _, rows = _inputs(None, DEC8)
    assert lib.pcv_attn_decode_window_fp8_supported(ctypes.byref(p), None, ctypes.byref(rows)) == 0
    assert b"attn_decode_window_fp8: fp8 params are NULL" in lib.pcv_last_error()
    assert lib.pcv_attn_decode_window_fp8(ctypes.byref(p), None, ctypes.byref(rows), None) == 1
    assert b"attn_decode_window_fp8: fp8 params or rows are NULL" in lib.pcv_last_error()


@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("M", [1024, 6144])
def test_decode_workspace_queries_agree(N, M):
    lib = _lib.lib()
    p, _ = _decode(N=N)
    p.M = p.m_total = M
    p.k_stride_b, p.v_stride_b = M * p.H * p.dqk, M * p.H * p.dv
    sizes = []
    for query in ("pcv_attn_decode_window_workspace_bytes", "pcv_attn_decode_fp8_workspace_bytes",
                  "pcv_attn_workspace_bytes"):
        need = ctypes.c_size_t(0)
        assert getattr(lib, query)(ctypes.byref(p), ctypes.byref(need)) == 0, lib.pcv_last_error()
        sizes.append(need.value)
    assert sizes[0] > 0 and sizes.count(sizes[0]) == 3, sizes
