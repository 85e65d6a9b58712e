"""Variant matrix and schedule shapes of the tensor-core attention backward (perceiver_io_b200/csrc/pcv_attn_bwd.cu),
shared by its GPU tests (test_gpu_bwd_variants.py) and their CPU companion (test_bwd_variants_cpu.py).  Nothing here
needs a GPU.

launch_attn_bwd instantiates (launch_shape), with NQB = pad64(dqk) / 64 and NVB = pad64(dv) / 64 boxes of 64
channels, bf16 or fp16:
  - head dims up to 128: bwd_dkdv_kernel<NQB, NVB, BF16, kOutBoth> and bwd_dq_kernel<NQB, NVB, BF16, 128>;
  - a head dim above 128 (NQB or NVB = 3): bwd_dkdv_kernel<.., kOutDV> (the dV pass), bwd_dkdv_kernel<.., kOutDK>
    (the dK pass) and bwd_dq_kernel<NQB, NVB, BF16, 64>.
Every kernel below keeps a TMA ring of NS stages whose phase runs on across the persistent kernels' tiles / work items;
the schedule shapes make that carry-over, the ring's wrap and the dQ split edges actually happen."""
import itertools

BF16, FP16 = "bf16", "fp16"
DTYPES = (BF16, FP16)
TILE = 128                  # kT: keys per dK/dV tile, queries per dQ tile
SMEM_LIMIT = 227 * 1024     # kSmemLimit
BOX = TILE * 128            # kBoxBytes: 128 rows x 64 16-bit channels
BOX64 = 64 * 128            # kBox64: a 64-row box
BARRIERS = 2048             # the bytes each Cfg keeps for its barriers
KWIDE_SPLIT_SMS = 132       # kWideSplitSms: the wide dQ split is planned for 132 SMs whatever the device


def boxes(d):
    return (d + 63) // 64


def is_wide(dqk, dv):
    """wide_bwd: a head dim above 128 takes the wide kernels."""
    return dqk > 128 or dv > 128


# ---- the instantiations one call reaches ----
def variants_of(dqk, dv, dt):
    """Kernel symbols (name, NQB, NVB, dtype, flag) a backward with these head dims launches.  flag: OUT of
    bwd_dkdv_kernel (0 both, 1 dV, 2 dK), KS (the keys per ring stage) of bwd_dq_kernel."""
    nq, nv = boxes(dqk), boxes(dv)
    if is_wide(dqk, dv):
        return {("dkdv", nq, nv, dt, 1), ("dkdv", nq, nv, dt, 2), ("dq", nq, nv, dt, 64)}
    return {("dkdv", nq, nv, dt, 0), ("dq", nq, nv, dt, 128)}


def reachable_variants():
    """Every instantiation launch_attn_bwd can reach: head dims 8..192 in multiples of 8 (attn_bwd_supported)."""
    out = set()
    for dqk, dv in itertools.product(range(8, 193, 8), repeat=2):
        for dt in DTYPES:
            out |= variants_of(dqk, dv, dt)
    return out


# ---- ring slot counts (NS) ----
def cfg1_slots(nqb, nvb):
    """Cfg1<NQB, NVB>::kSlots (dK/dV kernel): K and V resident, (NQB + NVB) 64-row Q / dO boxes per stage, at most 8."""
    return min(8, (SMEM_LIMIT - (nqb + nvb) * BOX - BARRIERS) // ((nqb + nvb) * BOX64))


def dq_slots(nqb, nvb, ks):
    """Cfg2<NQB, NVB, KS>::kSlots (bwd_dq_kernel): Q and dO resident, (NQB + NVB) KS-row K / V boxes per stage, at
    most 4."""
    return min(4, (SMEM_LIMIT - (nqb + nvb) * BOX - BARRIERS) // ((nqb + nvb) * ks * 128))


# ---- the plan ----
def dq_split(units, nk, sms):
    """dq_split: (tiles_per_split, splits) of the dQ kernel's key tiles.  Aim at ~64 key tiles per CTA, but at least
    ~4 CTAs per SM in all, and keep more than 4 tiles per split."""
    s = max(1, (nk + 63) // 64)
    while units * s < 4 * sms and s < nk and (nk + s - 1) // s > 4:
        s += 1
    tps = (nk + s - 1) // s
    return tps, (nk + tps - 1) // tps


def plan(B, H, N, M, dqk, dv, sms):
    """The launch geometry launch_attn_bwd derives (bwd_layout, bwd_setup, launch_shape)."""
    nq, nk = (N + TILE - 1) // TILE, (M + TILE - 1) // TILE              # bwd_layout
    nqb, nvb = boxes(dqk), boxes(dv)
    wide = is_wide(dqk, dv)
    # bwd_layout (wide: kWideSplitSms) / bwd_setup (the device's SM count)
    tps, splits = dq_split(B * H * nq, nk, KWIDE_SPLIT_SMS if wide else sms)
    tiles = B * H * nk  # p.total_tiles; the dK/dV grid is min(total_tiles, sms) in both launchers
    # the first key of the last dQ split (tiles of 128 keys; the wide kernel's stages are 64 keys, two per tile)
    p = dict(nq=nq, nk=nk, nq64=(N + 63) // 64, wide=wide, tiles=tiles, dkdv_grid=min(tiles, sms),
             last_split_key0=(splits - 1) * tps * TILE,
             dkdv_ns=cfg1_slots(nqb, nvb), tps=tps, splits=splits)
    # bwd_dq_kernel: work items (b, h, query tile, split); 64-key stages walked persistently by at most one CTA per SM
    # (wide), else 128-key stages on one CTA per item.  A split is tps tiles of 128 keys: tps * 128 / KS stages.
    ks = 64 if wide else TILE
    items, nks, per_split = B * H * nq * splits, (M + ks - 1) // ks, tps * (TILE // ks)
    p.update(dq_ks=ks, dq_ns=dq_slots(nqb, nvb, ks), dq_items=items, dq_grid=min(items, sms) if wide else items,
             dq_stages=[min(nks, s * per_split + per_split) - s * per_split for s in range(splits)])
    return p


# ---- the matrix: every instantiation, from head dims that are not multiples of 64 (zero-filled box tails) ----
SMALL_PAIRS = [(dqk, dv) for dqk in (40, 120) for dv in (56, 120)]             # (NQB, NVB) in {1, 2}^2
WIDE_PAIRS = [(184, 56), (184, 120), (184, 184), (40, 184), (120, 184)]      # the five pairs with a third box
VARIANT_CASES = [(dqk, dv, dt) for dt in DTYPES for dqk, dv in SMALL_PAIRS + WIDE_PAIRS]


def case_id(case):
    dqk, dv, dt = case
    return f"{dt}-qk{dqk}-v{dv}"


# ---- schedule shapes: name -> (B, H, N, M) and the structure check_bwd_schedule asserts ----
SCHEDULE_SHAPES = {
    "dkdv_carry": (2, 2, 130, 12700),  # (a) 400 key tiles: >= 3 per CTA; nq64 = 3, so a ring pass starts mid-tile
    "dkdv_wrap": (1, 1, 700, 300),     # (b) nq64 = 11 > NS: the ring wraps inside a tile (11 % NS != 0 as well)
    "dq_split": (3, 8, 64, 11300),     # (c) + (d): 18 splits of 5 tiles (> NS), the last one of 4
    "wide_dq_items": (3, 8, 64, 2700),  # (c) + (d) + (e): 144 wide dQ items, 6 splits of 8 stages (> NS), the last of 3
}
SCHEDULE_CASES = {
    "dkdv_carry": [(dqk, dv, dt) for dt in DTYPES for dqk, dv in SMALL_PAIRS + [(184, 184), (40, 184)]],
    "dkdv_wrap": [(dqk, dv, dt) for dt in DTYPES for dqk, dv in SMALL_PAIRS + [(184, 184), (40, 184)]],
    "dq_split": [(dqk, dv, dt) for dt in DTYPES for dqk, dv in SMALL_PAIRS],
    "wide_dq_items": [(dqk, dv, dt) for dt in DTYPES for dqk, dv in [(184, 184), (40, 184)]],
}


def check_bwd_schedule(shape, case, sms):
    """Assert that SCHEDULE_SHAPES[shape] has, for the variant `case` on `sms` SMs, the structure it is named for.
    Returns a one-line description of the plan."""
    B, H, N, M = SCHEDULE_SHAPES[shape]
    dqk, dv, _dt = case
    p = plan(B, H, N, M, dqk, dv, sms)
    ns, stages = p["dq_ns"], p["dq_stages"]
    if shape == "dkdv_carry":      # (a)
        per_cta = p["tiles"] // p["dkdv_grid"]
        nq64, ns1 = p["nq64"], p["dkdv_ns"]
        assert per_cta >= 2, f"{p['tiles']} tiles on {p['dkdv_grid']} CTAs"
        assert nq64 % ns1 != 0, f"nq64 {nq64} is a multiple of NS {ns1}"
        # `it` runs on across tiles: some pass over the ring (a phase flip) starts inside a later tile of every CTA
        flips = range(ns1, per_cta * nq64, ns1)
        assert any(f >= nq64 and f % nq64 for f in flips), f"no ring pass starts inside a later tile: {list(flips)}"
    elif shape == "dkdv_wrap":     # (b)
        assert p["nq64"] > p["dkdv_ns"], f"nq64 {p['nq64']} <= NS {p['dkdv_ns']}"
    elif shape in ("dq_split", "wide_dq_items"):
        assert p["splits"] >= 2 and stages[-1] < stages[0], f"splits {stages}"          # (c)
        assert min(stages[:-1]) > ns, f"splits of {stages} stages through {ns} slots"    # (d)
        if shape == "wide_dq_items":                                                    # (e)
            assert p["wide"] and p["dq_items"] > sms, f"{p['dq_items']} work items on {sms} CTAs"
    else:
        raise KeyError(shape)
    return (f"{shape} {case_id(case)} at {sms} SMs: dK/dV {p['tiles']} tiles on {p['dkdv_grid']} CTAs, nq64 "
            f"{p['nq64']}, NS {p['dkdv_ns']}; dQ {p['dq_items']} items on {p['dq_grid']} CTAs, stages per split "
            f"{stages[0]}..{stages[-1]} x {p['splits']}, NS {ns}")


# ---- tile-edge sweep: every (N, M) pair meets one small and one wide variant, taken in turn from these ----
EDGE_N = (1, 63, 64, 65, 127, 128, 129)
EDGE_M = (1, 2, 63, 64, 65, 127, 128, 129, 257)
EDGE_SMALL = [(40, 56, BF16), (120, 120, FP16)]
EDGE_WIDE = [(184, 120, FP16), (40, 184, BF16)]


def edge_variants(i):
    """The small and the wide variant of the i-th (N, M) pair."""
    return EDGE_SMALL[i % 2], EDGE_WIDE[(i // 2) % 2]
