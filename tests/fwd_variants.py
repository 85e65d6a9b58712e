"""Variant matrix and schedule shapes of the tensor-core forward kernel (perceiver_io_b200/csrc/pcv_attn_tc.cu), shared
by its GPU tests (test_gpu_fwd_variants.py) and their CPU companion (test_fwd_variants_cpu.py).  Nothing here needs a GPU.

launch_attn_tc instantiates attn_fwd_kernel<NQB, NVB, BF16, PAIR>:
  - NQB = pad64(dqk) / 64 Q/K boxes (1..8);
  - V runs in passes of at most 128 channels, each pass with NVB = ceil(dv_pass / 64) V boxes (1..2);
  - bf16 or fp16 operands;
  - PAIR: the 2-CTA cluster kernel (impl "tcgen05_pair"), which takes dqk and dv <= 128 only.
NQB <= 2 runs the pipelined schedule (ping-pong, peeled prologue / epilogue), larger NQB the serial one."""
import collections
import itertools

BF16, FP16 = "bf16", "fp16"
DTYPES = (BF16, FP16)
TILE = 128          # keys per key tile = query rows per CTA tile
MAX_DV_PASS = 128   # V channels per launch


def pad64(d):
    return (d + 63) // 64 * 64


def nqb_of(dqk):
    return pad64(dqk) // 64


def nvb_passes(dv):
    """NVB of each V pass of a call with v head dim dv."""
    return [(min(MAX_DV_PASS, dv - off) + 63) // 64 for off in range(0, dv, MAX_DV_PASS)]


def pair_supported(dqk, dv):
    return pad64(dqk) <= 128 and pad64(dv) <= 128


def variants_of(dqk, dv, dtype, pair):
    """The (NQB, NVB, dtype, pair) instantiations one call launches."""
    return {(nqb_of(dqk), nvb, dtype, pair) for nvb in nvb_passes(dv)}


def reachable_variants():
    """Every instantiation the dispatch can reach: head dims up to 512 in multiples of 8 (the TMA stride rule)."""
    out = set()
    for dqk, dv in itertools.product(range(8, 513, 8), repeat=2):
        for dt in DTYPES:
            out |= variants_of(dqk, dv, dt, False)
            if pair_supported(dqk, dv):
                out |= variants_of(dqk, dv, dt, True)
    return out


def ring_slots(nqb):
    """FwdCfg<NQB, NVB>::kSlots: 16 KB K/V ring slots left in 227 KB of shared memory next to Q and the barriers."""
    return min(16, (227 * 1024 - nqb * 16384 - 2048) // 16384)


def case_id(case):
    dqk, dv, dt, pair = case
    return f"{dt}-qk{dqk}-v{dv}" + ("-pair" if pair else "")


# ---- section 1: every instantiation, each from head dims that are not multiples of 64 (zero-filled box tails) ----
# (dqk, dv, dtype, pair).  qk 40 .. 456 give NQB 1 .. 8; v 56 / 120 give NVB 1 / 2; v 184 runs an NVB 2 pass and an
# NVB 1 pass in one call.
_QK = (40, 72, 136, 200, 264, 328, 392, 456)
VARIANT_CASES = (
    [(dqk, dv, dt, False) for dt in DTYPES for dqk in _QK for dv in (56, 120)]
    + [(128, 184, dt, False) for dt in DTYPES]
    + [(512, 56, dt, False) for dt in DTYPES]
    + [(dqk, dv, dt, True) for dt in DTYPES for dqk in (40, 72) for dv in (56, 120)]
    + [(128, 120, dt, True) for dt in DTYPES]
)

# ---- section 2: schedule shapes, per pipelined variant and NQB 3 / 7 of the serial schedule ----
SCHEDULE_VARIANTS = (
    [(dqk, dv, dt, pair) for dt in DTYPES for pair in (False, True) for dqk in (40, 120) for dv in (56, 120)]
    + [(dqk, dv, dt, False) for dt in DTYPES for dqk, dv in ((136, 120), (392, 56))]
)
# name -> (B, H, N, M)
SCHEDULE_SHAPES = {
    "one_tile": (2, 2, 256, 512),         # every CTA: one segment of one key tile (prologue + epilogue only)
    "ring": (2, 4, 120, 40000),           # ~19 (pair: ~38) tiles per CTA: the ring wraps; segments cross (b, h)
    "whole": (1, 2, 8600, 300),           # N > 66 * 128: whole-unit plan, some CTAs run two full segments
    "whole_causal": (1, 2, 8600, 8700),   # the same plan, causal
}


def workers_for(num_sms, pair):
    return num_sms // 2 if pair else num_sms


def plan_segments(B, H, N, M, workers, pair):
    """(counts, {cta: [(b, h, q0, t0, t1, slot), ...]}) of the kernel's work plan for one call."""
    from perceiver_io_b200 import _lib

    counts, segs = _lib.debug_plan(B, H, N, M, workers=workers, rows_per_unit=2 * TILE if pair else TILE)
    per_cta = collections.defaultdict(list)
    for cta, b, h, q0, _ntile, t0, t1, slot in segs:
        per_cta[cta].append((b, h, q0, t0, t1, slot))
    return counts, per_cta


def check_schedule(shape_name, case, workers, boxes_per_tile=None, slots=None):
    """Assert that the plan of SCHEDULE_SHAPES[shape_name] has the structure the shape is meant to exercise for the
    variant `case`, with `workers` CTAs (CTA pairs for the pair kernel).  `boxes_per_tile` / `slots` override the
    16-bit kernel's ring boxes per key tile and ring slots (the FP8 kernel's differ).  Returns a one-line description."""
    B, H, N, M = SCHEDULE_SHAPES[shape_name]
    dqk, dv, _dt, pair = case
    counts, per_cta = plan_segments(B, H, N, M, workers, pair)
    T = (M + TILE - 1) // TILE
    segs = [s for v in per_cta.values() for s in v]
    lengths = [t1 - t0 for _b, _h, _q0, t0, t1, _s in segs]
    per_cta_n = [len(v) for v in per_cta.values()]
    if shape_name == "one_tile":
        assert counts["slots"] > 0, "expected the split plan"
        assert max(per_cta_n) == 1 and set(lengths) == {1}, (per_cta_n, lengths)
    elif shape_name == "ring":
        assert counts["slots"] > 0 and counts["units"] > 0, "expected the split plan"
        nq = nqb_of(dqk)
        per_tile = nq + min(nvb_passes(dv)) if boxes_per_tile is None else boxes_per_tile
        ns = ring_slots(nq) if slots is None else slots
        boxes = max(lengths) * per_tile
        assert boxes >= 2 * ns, f"longest segment streams {boxes} boxes through {ns} slots"
        mixed = [v for v in per_cta.values() if len({(b, h) for b, h, *_ in v}) > 1]
        assert mixed, "no CTA runs segments of two (b, h)"
        assert any(t0 > 0 and slot >= 0 for v in mixed for _b, _h, _q0, t0, _t1, slot in v), "no split segment with t0 > 0"
    elif shape_name in ("whole", "whole_causal"):
        assert counts["slots"] == 0 and counts["units"] == 0, "expected the whole-unit plan"
        assert all((t0, t1) == (0, T) for _b, _h, _q0, t0, t1, _s in segs)
        assert max(per_cta_n) >= 2, "no CTA runs two full segments"
    else:
        raise KeyError(shape_name)
    return (f"{shape_name}: {counts['ctas']} CTAs, segments/CTA {min(per_cta_n)}..{max(per_cta_n)}, "
            f"tiles/segment {min(lengths)}..{max(lengths)}, {counts['slots']} split slots")


# ---- section 3: causal diagonal sweep ----
# M = N + shift.  Key tile [j0, j0 + 128) is mask-free for a warpgroup whose first row is n_wg iff j0 + 127 <= n_wg +
# shift.  With n_wg and j0 multiples of 64, shift = 63 (mod 64) makes a tile end exactly on a first row's diagonal,
# shift = 62 (mod 64) exactly one key past it; the others put the diagonal inside a tile.
DIAG_N = 416
DIAG_SHIFTS = (0, 1, 62, 63, 64, 65, 126, 127, 128, 129)
DIAG_SHARD_CUTS = (64, 259)   # interior shard offsets: one keeps shift (mod 64), one does not
DIAG_VARIANTS = [(dqk, dv, dt, pair) for dt in DTYPES for pair in (False, True) for dqk, dv in ((56, 120), (120, 56))]


def diag_poison_keys(M, shift):
    """Keys just past the causal diagonal of every row that starts a 64-row warpgroup: a leak at the mask-free-tile
    boundary lets exactly these in."""
    return [j for j in range(M) if (j - shift - 1) % 64 < 8]
