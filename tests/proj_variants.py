"""Variant matrix, launch rules and exact probes of the LayerNorm-folded projection kernels (perceiver_io_b200/csrc/
pcv_kvproj.cu: the producer forward and the row statistics; pcv_lnlin_bwd.cu: the LayerNorm -> Linear backward), shared
by their GPU tests (test_gpu_proj_variants.py) and the CPU companion (test_proj_variants_cpu.py).  Nothing here needs a
GPU.  Each rule cites the line of the .cu file it restates.

The 42 instantiations:
  - kvproj_kernel<BF16, FUSE, CG>         8  (pcv_kvproj.cu:240-244, dispatched :527-535)
  - kvproj_fp8_kernel<BF16, FUSE>         4  (:247-252, dispatched :489-491)
  - ln_stats_reg_kernel<T, NCH = 1..8>   16  (:262-264, dispatched :364-374)
  - ln_stats_kernel<T>                    2  (:311-313, dispatched :375-377)
  - lnlin_{dx, dx_fixup, dw, db, dw_finish, colsum}_kernel x 2 dtypes  12  (pcv_lnlin_bwd.cu:115-494, launched :521-619)
"""
import itertools

import torch

BF16, FP16 = "bf16", "fp16"
DTYPES = (BF16, FP16)
TORCH_DTYPE = {BF16: torch.bfloat16, FP16: torch.float16}

# ---- pcv_kvproj.cu ----
BM, BN, BK = 128, 128, 64   # rows / output columns per CTA, channels per stage (:31-33)
STAGES = 6                  # the TMA ring (:35)
STATS_CAP = 132 * 8         # both statistics kernels: at most 132 * 8 blocks of 8 warps (:365, :376)
REG_ROWS_PER_SWEEP = STATS_CAP * 8 * 2   # register kernel: two rows per warp iteration (:269) -> 16 896
GEN_ROWS_PER_SWEEP = STATS_CAP * 8       # generic kernel: one row per warp (:316) -> 8 448
REG_MAX_C = 2048            # reg_ok (:362-363)

# ---- pcv_lnlin_bwd.cu ----
WORKERS, MAX_SPLITS = 132, 32   # kWorkers, kMaxSplits (:42-43)
FIXUP_ROWS_PER_SWEEP = WORKERS * 8 * 8   # lnlin_dx_fixup_kernel: min(ceil(rows / 8), 132 * 8) blocks of 8 warps (:561)
FINISH_CAP = WORKERS * 16       # lnlin_dw_finish_kernel blocks (:610)
COLSUM_RANGES = 8               # lnlin_colsum_kernel: threadIdx.y ranges of row blocks (:474)


def cdiv(a, b):
    return -(-a // b)


# ---- producer rules ----
def fuse_selected(has_stats, ln_eps):
    """launch_kv_project / _fp8 (:480, :515): the in-kernel statistics run when row_stats == nullptr && ln_eps > 0."""
    return (not has_stats) and ln_eps > 0.0


def producer_grid(rows, n_total, cg):
    """launch_gemm (:387): m_blocks rounded up to whole pairs for CG = 2 (a pair's spare block is all padding), tiles_n =
    ceil(n_total / 128) (:471, :512); kvproj_body (:83-87): the column tile is the fastest grid index, cluster rank r
    of a CG = 2 pair takes row block 2 (cid / tiles_n) + r, and loads the 64-column half r of the weight box for both
    CTAs (:110-111).  Returns (m_blocks, tiles_n, [(blockIdx, m_blk, n_blk, rank)])."""
    m_blocks = cdiv(rows, BM * cg) * cg
    tiles_n = cdiv(n_total, BN)
    blocks = []
    for bid in range(m_blocks * tiles_n):
        cid, rank = bid // cg, bid % cg
        blocks.append((bid, (cid // tiles_n) * cg + rank, cid % tiles_n, rank))
    return m_blocks, tiles_n, blocks


def num_kb(C):
    """num_kb = ceil(C / 64) (:470, :511): the last stage's channels past C come from the TMA zero fill."""
    return cdiv(C, BK)


# ---- row statistics rules ----
def stats_route(C, stride, base_aligned=True):
    """launch_ln_stats_t (:362-377): ("reg", NCH) when reg_ok = C % 256 == 0, C <= 2048, stride % 8 == 0 and x 16-byte
    aligned; else ("generic", path) where ln_stats_kernel takes its vector path for a row that is 16-byte aligned with
    C % 8 == 0 (:318), the scalar path otherwise ("mixed" when rows differ)."""
    if C % 256 == 0 and C <= REG_MAX_C and stride % 8 == 0 and base_aligned:
        return ("reg", C // 256)
    if C % 8:
        return ("generic", "scalar")
    if not base_aligned:
        return ("generic", "scalar" if stride % 8 == 0 else "mixed")
    return ("generic", "vector" if stride % 8 == 0 else "mixed")


def stats_blocks(rows, route):
    """Grid of the statistics kernel (:365, :376) and the rows one sweep of its grid-stride loop covers."""
    if route[0] == "reg":
        return min(cdiv(rows, 16), STATS_CAP), REG_ROWS_PER_SWEEP
    return min(cdiv(rows, 8), STATS_CAP), GEN_ROWS_PER_SWEEP


# ---- backward rules ----
def make_plan(rows, C, n_k, n_v):
    """make_plan (pcv_lnlin_bwd.cu:54-76): m_blocks = ceil(rows / 128), kb_rows = ceil(rows / 64), tiles_c / tiles_n =
    ceil(C / 128) / ceil(n / 128), splits = max(1, min(264 / tiles, 32, kb_rows)); workspace bytes as the library's."""
    n = n_k + n_v
    m_blocks, kb_rows = cdiv(rows, 128), cdiv(rows, 64)
    tiles_c, tiles_n = cdiv(C, 128), cdiv(n, 128)
    splits = max(1, min(2 * WORKERS // (tiles_c * tiles_n), MAX_SPLITS, kb_rows))
    up = lambda b: cdiv(b, 256) * 256
    nbytes = up(tiles_c * rows * 8) + up(m_blocks * C * 8) + up(splits * n * C * 4) + up(splits * n * 4)
    return dict(m_blocks=m_blocks, kb_rows=kb_rows, tiles_c=tiles_c, tiles_n=tiles_n, splits=splits, bytes=nbytes)


def split_rows(rows, kb_rows, splits):
    """[r0, r1) of every dW / db split (:308, :434): 64-row blocks kb_rows * s / splits .. kb_rows * (s + 1) / splits."""
    return [(kb_rows * s // splits * 64, min(kb_rows * (s + 1) // splits * 64, rows)) for s in range(splits)]


def colsum_ranges(m_blocks):
    """lnlin_colsum_kernel (:474): thread row y sums row blocks m_blocks * y / 8 .. m_blocks * (y + 1) / 8."""
    return [(m_blocks * y // COLSUM_RANGES, m_blocks * (y + 1) // COLSUM_RANGES) for y in range(COLSUM_RANGES)]


NEED_NAMES = ("x", "w", "b", "gamma", "beta")


def bwd_kernels(needs):
    """Kernels launch_t runs for needs = (grad_x, grad_w, grad_b, grad_gamma, grad_beta) (:534-617): dx when grad_x or
    a column sum is wanted (col_part = nullptr without dgamma / dbeta, :548; no grad_x store without grad_x, :172), the
    fixup with grad_x, colsum with dgamma or dbeta, db without grad_w but with grad_b, dw with grad_w, finish with
    grad_w or grad_b."""
    gx, gw, gb, gg, gbe = needs
    col = gg or gbe
    out = set()
    if gx or col:
        out.add("dx")
    if gx:
        out.add("dx_fixup")
    if col:
        out.add("colsum")
    if gb and not gw:
        out.add("db")
    if gw:
        out.add("dw")
    if gw or gb:
        out.add("dw_finish")
    return out


# ---- the instantiations ----
def all_instantiations():
    s = set()
    for dt, fuse, cg in itertools.product(DTYPES, (False, True), (1, 2)):
        s.add(("kvproj", dt, fuse, cg))
    for dt, fuse in itertools.product(DTYPES, (False, True)):
        s.add(("kvproj_fp8", dt, fuse))
    for dt, nch in itertools.product(DTYPES, range(1, 9)):
        s.add(("ln_stats_reg", dt, nch))
    for dt in DTYPES:
        s.add(("ln_stats", dt))
    for dt, k in itertools.product(DTYPES, ("dx", "dx_fixup", "dw", "db", "dw_finish", "colsum")):
        s.add(("lnlin_" + k, dt))
    return s


# ---- the case matrix ----
# producer shapes: name -> (rows, C, n_k, n_v, x_stride)
PRODUCER_SHAPES = {
    "rows1": (1, 256, 128, 64, 256),
    "rows127_c200": (127, 200, 64, 72, 200),      # C = 200: the last stage holds 8 channels, 56 zero-filled
    "rows128_c64": (128, 64, 64, 8, 64),
    "rows129_c72": (129, 72, 128, 8, 72),
    "pair_spare": (300, 128, 128, 128, 128),      # CG = 2: blocks 2 and 3 pair up, block 3 (rows 384..511) is padding
    "n_first_half": (256, 128, 128, 40, 128),     # n_total = 168 ends inside the first 64-column half of tile 1
    "c8": (200, 8, 64, 8, 8),
    "c448_ring": (300, 448, 64, 64, 448),         # 7 k-blocks: the 6-stage ring wraps
    "c1024_ring": (260, 1024, 128, 256, 1024),
    "nk0": (200, 256, 0, 136, 256),
    "nv0": (200, 256, 192, 0, 256),
    "kv_split64": (150, 128, 64, 128, 128),       # the K/V split inside column tile 0
    "kv_split192": (150, 128, 192, 128, 128),     # ... inside column tile 1
    "x_stride": (190, 136, 64, 64, 200),          # x row stride 200 > C = 136
}


def check_producer_shape(name, cg=2):
    """Assert the structure a producer shape is named for."""
    rows, C, n_k, n_v, xs = PRODUCER_SHAPES[name]
    n = n_k + n_v
    m_blocks, tiles_n, blocks = producer_grid(rows, n, cg)
    if name.startswith("rows"):
        assert rows in (1, 127, 128, 129)
    if name == "pair_spare":
        spare = [b for b in blocks if b[1] * BM >= rows]
        assert cg == 2 and spare and all(b[3] == 1 for b in spare), "the spare block must be rank 1 of a pair"
    if name == "n_first_half":
        assert 0 < n % BN <= 64
    if name in ("rows127_c200", "rows129_c72", "c8"):
        assert C % BK != 0
    if name.endswith("_ring"):
        assert num_kb(C) > STAGES
    if name == "nk0":
        assert n_k == 0
    if name == "nv0":
        assert n_v == 0
    if name.startswith("kv_split"):
        assert n_k % BN != 0 and n > n_k
    if name == "x_stride":
        assert xs > C
    if name in ("c8", "rows128_c64", "rows129_c72", "rows127_c200"):
        assert C in (8, 64, 72, 200)
    return m_blocks, tiles_n


# statistics shapes: name -> (rows, C, stride, offset elements)
STATS_SHAPES = {f"nch{k}": (257 + 2 * k, 256 * k, 256 * k, 0) for k in range(1, 9)}   # odd rows: the 2-row tail
STATS_SHAPES.update({
    "gen_vector": (333, 200, 200, 0),
    "gen_scalar_odd_c": (99, 131, 131, 0),
    "gen_scalar_unaligned": (101, 256, 264, 4),    # base 8 bytes off 16-byte alignment: generic, scalar path
    "gen_over_cap": (65, 2304, 2304, 0),
    "reg_two_sweeps": (17001, 256, 256, 0),
    "gen_two_sweeps": (17001, 264, 264, 0),
})


def check_stats_shape(name):
    rows, C, stride, off = STATS_SHAPES[name]
    route = stats_route(C, stride, off % 8 == 0)
    blocks, per_sweep = stats_blocks(rows, route)
    if name.startswith("nch"):
        assert route == ("reg", int(name[3:])) and rows % 2 == 1
    if name == "gen_vector":
        assert route == ("generic", "vector")
    if name.startswith("gen_scalar"):
        assert route == ("generic", "scalar")
    if name == "gen_over_cap":
        assert C > REG_MAX_C and route == ("generic", "vector")
    if name.endswith("two_sweeps"):
        assert blocks == STATS_CAP and rows > per_sweep
    return route


# backward shapes: name -> (rows, C, n_k, n_v)
BWD_SHAPES = {
    "splits1": (512, 1024, 1024, 2048),
    "splits32": (4000, 128, 64, 64),
    "splits_kb_rows": (300, 64, 64, 0),
    "rows1": (1, 64, 64, 8),
    "fixup_sweep": (9000, 256, 64, 8),
    "mblocks5": (637, 200, 128, 72),
    "mblocks11": (1300, 264, 64, 136),
    "nk0": (700, 256, 0, 136),
    "nv0": (700, 256, 192, 0),
}


def check_bwd_shape(name):
    rows, C, n_k, n_v = BWD_SHAPES[name]
    pl = make_plan(rows, C, n_k, n_v)
    if name == "splits1":
        assert pl["splits"] == 1 and pl["kb_rows"] > 1
    if name == "splits32":
        assert pl["splits"] == MAX_SPLITS
    if name in ("splits_kb_rows", "rows1"):
        assert pl["splits"] == pl["kb_rows"] and rows < 64 * pl["splits"]
    if name == "rows1":
        assert rows == 1
    if name == "fixup_sweep":
        assert rows > FIXUP_ROWS_PER_SWEEP
    if name.startswith("mblocks"):
        assert pl["m_blocks"] < 8 or pl["m_blocks"] % 8 != 0
        assert any(b0 == b1 for b0, b1 in colsum_ranges(pl["m_blocks"])) == (pl["m_blocks"] < 8)
    if name == "nk0":
        assert n_k == 0
    if name == "nv0":
        assert n_v == 0
    return pl


ALL_NEEDS = (True, True, True, True, True)
# every subset that changes which kernels launch, or what the dx kernel stores (want_x, want_col)
NEEDS_SUBSETS = {
    "all": ALL_NEEDS,
    "x": (True, False, False, False, False),
    "gamma": (False, False, False, True, False),
    "beta": (False, False, False, False, True),
    "x_gamma": (True, False, False, True, False),
    "w": (False, True, False, False, False),
    "b": (False, False, True, False, False),
    "w_b": (False, True, True, False, False),
    "x_b": (True, False, True, False, False),
    "x_w": (True, True, False, False, False),
    "b_beta": (False, False, True, False, True),
    "w_beta": (False, True, False, False, True),
    "x_b_beta": (True, False, True, False, True),
}


def case_instantiations(kind, dt, **kw):
    """The instantiations one case launches."""
    if kind == "proj":
        fuse = fuse_selected(kw["has_stats"], kw["ln_eps"])
        if kw.get("fp8"):
            return {("kvproj_fp8", dt, fuse)}
        return {("kvproj", dt, fuse, kw["cg"])}
    if kind == "stats":
        r = stats_route(kw["C"], kw["stride"], kw.get("aligned", True))
        return {("ln_stats_reg", dt, r[1])} if r[0] == "reg" else {("ln_stats", dt)}
    return {("lnlin_" + k, dt) for k in bwd_kernels(kw["needs"])}


def matrix_instantiations():
    """The instantiations the GPU module's matrix reaches: producer shapes x {none, separate, fused} x CG 1 / 2, the
    e4m3 producer x {none, separate, fused}, every statistics shape, every backward shape and needs subset, both dtypes
    each."""
    s = set()
    for dt in DTYPES:
        for mode, cg in itertools.product(("none", "separate", "fused"), (1, 2)):
            s |= case_instantiations("proj", dt, has_stats=mode == "separate", ln_eps=0.0 if mode == "none" else 1e-5,
                                     cg=cg)
            s |= case_instantiations("proj", dt, has_stats=mode == "separate", ln_eps=0.0 if mode == "none" else 1e-5,
                                     fp8=True)
        for rows, C, stride, off in STATS_SHAPES.values():
            s |= case_instantiations("stats", dt, C=C, stride=stride, aligned=off % 8 == 0)
        for needs in NEEDS_SUBSETS.values():
            s |= case_instantiations("bwd", dt, needs=needs)
    return s


# ---- exact probes ----
def producer_probe(rows, C, n, seed, ln, dtype=torch.bfloat16):
    """Operands on which every fp32 intermediate of the producer is exact (CPU tensors):
      - no LayerNorm: x in -3..3, W in -2..2, bias in -4..4 (|x.w| <= 6 C < 2^24);
      - LayerNorm (ln=True): row r is mu_r +- 2^k_r (half the channels each way, mu in -8..8, k in 0..2), so with
        eps = 0 the statistics are (mu, 2^-k) exactly and x_hat = +-1; gamma in {1/2, 1, 2}, W in -2..2 (gamma W
        exact), beta in -2..2 and bias in -4..4 (t exact).  C must be a power of two for the register kernel's
        mean = sum * (1 / C) to be exact.
    Returns (x, gamma, beta, w, bias, mu, k) (gamma / beta / mu / k None without LayerNorm)."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, generator=g).double()
    w = ri(-2, 2, n, C)
    bias = ri(-4, 4, n)
    if not ln:
        return ri(-3, 3, rows, C).to(dtype), None, None, w.to(dtype), bias.to(dtype), None, None
    mu = ri(-8, 8, rows)
    k = ri(0, 2, rows)
    sign = torch.ones(rows, C, dtype=torch.float64)
    for r in range(rows):
        sign[r, torch.randperm(C, generator=g)[: C // 2]] = -1.0
    x = mu[:, None] + sign * (2.0 ** k)[:, None]
    gamma = 2.0 ** ri(-1, 1, C)
    beta = ri(-2, 2, C)
    return x.to(dtype), gamma.to(dtype), beta.to(dtype), w.to(dtype), bias.to(dtype), mu, k


def bwd_probe(rows, C, n, seed, dtype=torch.bfloat16):
    """Backward operands on which dy, dx_hat, a, b, P, db, dgamma and dbeta are exact in fp32 and dx_hat is exact in 16
    bits: x rows mu +- 2^k (x_hat = +-1 with eps = 0), G and W in {-1, 0, 1} (|dy| <= n <= 256), gamma in {1/2, 1}, beta
    in {-1, -1/2, 0, 1/2, 1}.  C a power of two (the fixup's 1 / C is exact)."""
    assert n <= 256 and C & (C - 1) == 0
    x, _, _, _, _, mu, k = producer_probe(rows, C, 8, seed, True, dtype)
    g = torch.Generator().manual_seed(seed + 1)
    ri = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, generator=g).double()
    G = ri(-1, 1, rows, n)
    W = ri(-1, 1, n, C)
    gamma = 2.0 ** ri(-1, 0, C)
    beta = ri(-2, 2, C) / 2
    return x, gamma.to(dtype), beta.to(dtype), W.to(dtype), G.to(dtype), mu, k


def vt_coords(rows, keys_per_batch, n_k, n_v, dv):
    """Where kvproj_body writes V column n of row r in V^T (:220-225): (b, h, c, m) = (r / M, c' / dv, c' % dv, r % M) with
    c' = n - n_k.  Returns a (rows, n_v, 4) int64 tensor."""
    r = torch.arange(rows)[:, None].expand(rows, n_v)
    c = torch.arange(n_v)[None, :].expand(rows, n_v)
    b, m = r // keys_per_batch, r % keys_per_batch
    return torch.stack([b, c // dv, c % dv, m], -1)


def vt_digit_probe(coord, digit, rows, C, n_k, n_v, keys_per_batch, dv, dtype=torch.bfloat16):
    """(x, w) of the no-LayerNorm e4m3 probe pass that writes base-16 digit `digit` of coordinate `coord` (0 b, 1 h,
    2 c, 3 m) into every V^T element: the value is a small integer, exact in e4m3.  Row coordinates (b, m) come from
    x[:, 0] against w[:, 0] = 1; column coordinates (h, c) from x[:, 0] = 1 against w[:, 0]."""
    n = n_k + n_v
    x = torch.zeros(rows, C, dtype=torch.float64)
    w = torch.zeros(n, C, dtype=torch.float64)
    r = torch.arange(rows)
    cv = torch.arange(n_v)
    val_row = {0: r // keys_per_batch, 3: r % keys_per_batch}
    val_col = {1: cv // dv, 2: cv % dv}
    if coord in val_row:
        x[:, 0] = ((val_row[coord] >> (4 * digit)) & 15).double()
        w[:, 0] = 1.0
    else:
        x[:, 0] = 1.0
        w[n_k:, 0] = ((val_col[coord] >> (4 * digit)) & 15).double()
    return x.to(dtype), w.to(dtype)
