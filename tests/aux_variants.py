"""The rotary, KV-append and pad-packing kernels (csrc/pcv_aux.cu:187-431): their launch rules restated with the lines
they restate, the case matrix that reaches every instantiation and path, fp64 / exact oracles, and mutants of the rules.
Shared by test_aux_variants_cpu.py (the rules against the library's ptxas log and the oracles against the mutants, on
the CPU) and test_gpu_aux_variants.py (the kernels against the oracles).

Instantiations (17): rotary_kernel<T, AT> (T bf16 / fp16: 4), rotary_fp8_kernel<T, AT> (T bf16 / fp16 / e4m3: 6),
kv_append_kernel<AT> (2), kv_append_fp8_kernel<T, AT> (T bf16 / fp16: 4) and pack_pad_kernel (1).  AT: the rows are read
from device memory when the kernel runs (the *_at entry points).  kv_append_kernel picks a 16-byte or a 2-byte path per
segment (`vec`, :276-277)."""
import re
from typing import NamedTuple, Optional, Tuple

import torch

BF16, FP16, FP32, E4M3 = "bf16", "fp16", "fp32", "e4m3"
TORCH_DTYPE = {BF16: torch.bfloat16, FP16: torch.float16, FP32: torch.float32, E4M3: torch.float8_e4m3fn}
ELEM_BYTES = {BF16: 2, FP16: 2, FP32: 4, E4M3: 1}
E4M3_MAX = 448.0

THREADS = 256                 # every launch in pcv_aux.cu uses 256-thread blocks
ROTARY_MAX_BLOCKS = 132 * 16  # launch_rotary (pcv_aux.cu:561-562)
APPEND_MAX_BLOCKS = 132 * 8   # launch_kv_append (:632-634), the fp8 append included
PACK_MAX_BLOCKS = 1024        # launch_pack_pad (:426)


def cdiv(a, b):
    return -(-a // b)


# ---- the 17 instantiations ----
def all_instantiations():
    s = {("rotary", t, at) for t in (BF16, FP16) for at in (False, True)}
    s |= {("rotary_fp8", t, at) for t in (BF16, FP16, E4M3) for at in (False, True)}
    s |= {("kv_append", at) for at in (False, True)}
    s |= {("kv_append_fp8", t, at) for t in (BF16, FP16) for at in (False, True)}
    return s | {("pack_pad",)}


_TYPE_OF = {"__nv_bfloat16": BF16, "__half": FP16, "unsigned char": E4M3}


def instantiation_of(demangled: str):
    """The instantiation a demangled kernel name stands for, e.g. 'rotary_fp8_kernel<unsigned char, true>' ->
    ('rotary_fp8', 'e4m3', True); None for any other kernel of the file."""
    m = re.match(r"(rotary_kernel|rotary_fp8_kernel|kv_append_fp8_kernel|kv_append_kernel|pack_pad_kernel)(<(.*)>)?$",
                 demangled)
    if m is None:
        return None
    kind = m.group(1)[:-len("_kernel")]
    args = [a.strip() for a in m.group(3).split(",")] if m.group(3) else []
    at = args[-1] == "true" if args else None
    if kind == "pack_pad":
        return ("pack_pad",)
    if kind == "kv_append":
        return (kind, at)
    return (kind, _TYPE_OF[args[0]], at)


# ---- the grids (one thread per unit of work, grid-stride loops) ----
def rotary_work(B, n, H, d):
    """Channel pairs, one thread each: (d + 1) / 2 per head row (:561), the half pair of an odd d included."""
    return B * n * H * ((d + 1) // 2)


def rotary_blocks(B, n, H, d):
    return min(cdiv(rotary_work(B, n, H, d), THREADS), ROTARY_MAX_BLOCKS)


def pad_words_per_row(M):
    """pcv_common.cuh: whole 128-key tiles, 4 words each; the bits past M are zero."""
    return 4 * cdiv(M, 128)


def pack_blocks(B, M):
    return min(cdiv(B * pad_words_per_row(M), THREADS), PACK_MAX_BLOCKS)


def sweeps(work, blocks):
    """How many times the grid-stride loop of a grid of `blocks` 256-thread blocks passes over `work` items."""
    return cdiv(work, blocks * THREADS)


class Seg(NamedTuple):
    """A CopySeg (:246-253) in bytes: src / dst are byte offsets from 16-byte aligned allocations."""
    src: int
    dst: int
    s_sb: int
    s_sl: int
    d_sb: int
    d_sl: int
    rows: int
    row_bytes: int
    dst_row0: int


def vec_path(s: Seg) -> bool:
    """kv_append_kernel's predicate (:276-277): both pointers, the four byte strides and row_bytes multiples of 16."""
    return ((s.src | s.dst | s.s_sb | s.s_sl | s.d_sb | s.d_sl | s.row_bytes) & 15) == 0


def segment_work(s: Seg, fp8: bool) -> int:
    """Work items of a segment: 16-byte vectors (vec path, and every fp8 segment: :327) or 2-byte elements (:293)."""
    if s.rows == 0:
        return 0
    return s.rows * (s.row_bytes >> 4 if fp8 or vec_path(s) else s.row_bytes >> 1)


def append_blocks(B, segs):
    """launch_kv_append (:632-634): maxwork counts 16-byte vectors whatever the path, so a row of fewer than 16 bytes
    counts 0 and its grid is one block per segment."""
    maxwork = max([1] + [B * s.rows * (s.row_bytes >> 4) for s in segs])
    return min(cdiv(maxwork, THREADS), APPEND_MAX_BLOCKS)


# ---- the rows of the AT instantiations ----
def at_rows(bounds_b: Tuple[int, int], i: int, capacity: int):
    """at_rows<true> (:192-200): (angle row, output row, written) of input row i of a batch row with bounds (w0, w1).  A
    row is skipped when its angle row is negative or at or past capacity, whichever output row it would go to."""
    arow = bounds_b[0] + i
    return arow, (arow if bounds_b[1] else i), 0 <= arow < capacity


def dst_row(bound_b: int, row: int, capacity: int):
    """dst_row<true> (:261-266): (destination row, written); rows before 0 or at or past capacity are skipped."""
    r = bound_b + row
    return r, 0 <= r < capacity


def angle_row0(n_angles, n, right_align):
    """ops._rotary_params (ops.py:786): the last n angle rows when right_align, else the first n."""
    return n_angles - n if right_align else 0


def a_stride_b(Ba, B, stride0):
    """ops._rotary_params (ops.py:782): a batch-1 angle tensor is broadcast (stride 0) over B > 1 rows."""
    return 0 if (Ba == 1 and B > 1) else stride0


# ---- the case matrix ----
class RotaryCase(NamedTuple):
    name: str
    dt: str             # input: bf16 / fp16, or e4m3 codes (fp8 output only)
    fp8: bool           # e4m3 output (rotary_fp8_kernel)
    at: bool
    B: int
    n: int
    H: int
    d: int
    rd: int             # rotate_dim
    Ba: int = 1         # angle batch (B: per-batch angles)
    extra_angles: int = 0
    right_align: bool = False
    x_pad: int = 0      # extra elements per x row: x is a column slice of a wider tensor
    y_pad: int = 0
    bounds: Optional[tuple] = None   # AT: per batch row (row0, out-row flag); one entry: shared (bounds_stride_b 0)
    capacity: int = 0

    @property
    def instantiation(self):
        return ("rotary_fp8" if self.fp8 else "rotary", self.dt, self.at)

    @property
    def n_angles(self):
        return self.capacity if self.at else self.n + self.extra_angles

    @property
    def work(self):
        return rotary_work(self.B, self.n, self.H, self.d)

    @property
    def sweeps(self):
        return sweeps(self.work, rotary_blocks(self.B, self.n, self.H, self.d))

    def rows(self):
        """(arow (B, n), yrow (B, n), written (B, n)) as python lists."""
        if not self.at:
            r0 = angle_row0(self.n_angles, self.n, self.right_align)
            return ([[r0 + i for i in range(self.n)]] * self.B, [list(range(self.n))] * self.B,
                    [[True] * self.n] * self.B)
        out = ([], [], [])
        for b in range(self.B):
            bb = self.bounds[b % len(self.bounds)]
            rs = [at_rows(bb, i, self.capacity) for i in range(self.n)]
            for k in range(3):
                out[k].append([r[k] for r in rs])
        return out

    @property
    def out_rows(self):
        """Rows of the output tensor: the arena's capacity when some row goes to its table row, else n."""
        return self.capacity if self.at and any(f for _, f in self.bounds) else self.n


# AT bounds: a negative first row (the first rows skipped), a row ending exactly at capacity - 1, rows running past
# capacity, and a row in the middle; with and without the output-row flag
AT_BOUNDS = ((-3, 1), (34, 1), (38, 0), (5, 0))
AT_CAPACITY = 40


def _rotary_cases():
    c = []
    for dt in (BF16, FP16):
        c += [
            RotaryCase(f"{dt}-big", dt, False, False, 2, 4100, 8, 66, 66),
            RotaryCase(f"{dt}-odd-d-perbatch-ralign", dt, False, False, 3, 37, 3, 67 if dt == BF16 else 33,
                       64 if dt == BF16 else 32, Ba=3, extra_angles=13, right_align=True),
            RotaryCase(f"{dt}-rd0", dt, False, False, 2, 9, 2, 8 if dt == BF16 else 9, 0),
            RotaryCase(f"{dt}-rd2-strided", dt, False, False, 2, 11, 3, 10, 2, x_pad=5, y_pad=3),
            RotaryCase(f"{dt}-full-strided-bcast", dt, False, False, 3, 21, 2, 64, 64, extra_angles=4, right_align=True,
                       x_pad=7),
            RotaryCase(f"{dt}-at", dt, False, True, 4, 6, 3, 67 if dt == BF16 else 64, 64 if dt == BF16 else 32,
                       bounds=AT_BOUNDS, capacity=AT_CAPACITY, y_pad=1),
            RotaryCase(f"{dt}-at-rd0", dt, False, True, 4, 6, 2, 9, 0, bounds=AT_BOUNDS, capacity=AT_CAPACITY),
        ]
    c.append(RotaryCase("bf16-at-big", BF16, False, True, 2, 2100, 8, 66, 66, bounds=((3, 1),), capacity=4200))
    for dt in (BF16, FP16, E4M3):
        c += [
            RotaryCase(f"{dt}-fp8-perbatch-ralign", dt, True, False, 3, 37, 3, 66, 32, Ba=3, extra_angles=9,
                       right_align=True),
            RotaryCase(f"{dt}-fp8-rd0", dt, True, False, 2, 13, 2, 16, 0),
            RotaryCase(f"{dt}-fp8-full-strided", dt, True, False, 2, 19, 2, 64, 64, x_pad=6, y_pad=2),
            RotaryCase(f"{dt}-fp8-at", dt, True, True, 4, 6, 3, 64, 64, bounds=AT_BOUNDS, capacity=AT_CAPACITY),
            RotaryCase(f"{dt}-fp8-at-rd0", dt, True, True, 4, 6, 2, 16, 0, bounds=AT_BOUNDS, capacity=AT_CAPACITY),
        ]
    c.append(RotaryCase("bf16-fp8-big", BF16, True, False, 2, 4100, 8, 66, 66))
    return c


ROTARY_CASES = _rotary_cases()


class AppendCase(NamedTuple):
    name: str
    dt: str             # new rows: bf16 / fp16 / fp32
    fp8: bool           # e4m3 arena (kv_append_fp8_kernel)
    at: bool
    B: int
    L_old: int
    n: int
    Ck: int
    Cv: int
    pad: int = 0        # extra elements per row of every tensor (strided rows)
    shift: int = 0      # first element of every view inside its padded row (0 <= shift <= pad)
    alias_k: bool = False   # the K cache pointer equals the K destination's (an in-place half: skipped)
    bounds: Optional[tuple] = None   # AT: first arena row of every batch row; one entry: shared
    capacity: int = 0

    @property
    def instantiation(self):
        return ("kv_append_fp8", self.dt, self.at) if self.fp8 else ("kv_append", self.at)

    @property
    def dst_rows(self):
        return self.capacity if self.at else self.L_old + self.n

    def segments(self):
        """The four CopySegs launch_kv_append builds (:616-631), in bytes, with the in-place skip (:624)."""
        es = ELEM_BYTES[self.dt]
        ds = 1 if self.fp8 else es
        segs = []
        for y, (C, cache) in enumerate(((self.Ck, True), (self.Ck, False), (self.Cv, True), (self.Cv, False))):
            row = C + self.pad
            rows = self.L_old if cache else self.n
            src_es = ds if cache else es
            src_off, dst_off = self.shift * src_es, self.shift * ds
            s_sb, s_sl = rows * row * src_es, row * src_es
            d_sb, d_sl = self.dst_rows * row * ds, row * ds
            if y == 0 and self.alias_k:
                # the K cache is a view at k_dst's pointer with the batch stride of a dense cache: copied, batch row 1
                # would read rows of batch row 0; the launch skips it because the pointers are equal
                src_off, s_sb, s_sl, rows = dst_off, self.L_old * row * ds, d_sl, 0
            segs.append(Seg(src_off, dst_off, s_sb, s_sl, d_sb, d_sl, rows, C * ds, 0 if cache else self.L_old))
        return segs

    @property
    def paths(self):
        """The paths the launch takes: 'vec' / 'scalar' of every segment with rows (fp8: 'vec' throughout)."""
        return {("vec" if self.fp8 or vec_path(s) else "scalar") for s in self.segments() if s.rows}

    @property
    def blocks(self):
        return append_blocks(self.B, self.segments())

    @property
    def sweeps(self):
        return max(sweeps(self.B * segment_work(s, self.fp8), self.blocks) for s in self.segments())


APPEND_AT_BOUNDS = (-2, 7, 36, 0)   # a negative first row, rows past capacity, the middle, row 0
APPEND_CAPACITY = 40


def _append_cases():
    c = []
    for dt in (BF16, FP32):
        es = ELEM_BYTES[dt]
        odd = 60 if dt == BF16 else 61    # rows of 120 / 244 bytes: the scalar path
        c += [
            AppendCase(f"{dt}-vec", dt, False, False, 3, 17, 5, 64, 32),
            AppendCase(f"{dt}-scalar", dt, False, False, 3, 17, 5, odd, 8 if dt == BF16 else 4),
            AppendCase(f"{dt}-strided-vec", dt, False, False, 2, 9, 4, 64, 64, pad=16 // es, shift=8 // es * 2),
            AppendCase(f"{dt}-strided-scalar", dt, False, False, 2, 9, 4, 64, 64, pad=3, shift=1),
            AppendCase(f"{dt}-inplace-k", dt, False, False, 2, 12, 3, 64, 40, alias_k=True),
            AppendCase(f"{dt}-tiny-rows", dt, False, False, 3, 5, 4, 6 // es + 1, 2),   # C * es < 16: one block
            AppendCase(f"{dt}-no-cache", dt, False, False, 2, 0, 7, 64, 24),
            AppendCase(f"{dt}-at-vec", dt, False, True, 4, 0, 6, 64, 32, bounds=APPEND_AT_BOUNDS,
                       capacity=APPEND_CAPACITY),
            AppendCase(f"{dt}-at-scalar", dt, False, True, 4, 0, 6, odd, 5, bounds=APPEND_AT_BOUNDS,
                       capacity=APPEND_CAPACITY),
        ]
    c += [
        AppendCase("fp16-vec", FP16, False, False, 2, 3, 2, 8, 16),
        AppendCase("fp16-at-scalar-strided", FP16, False, True, 2, 0, 5, 24, 8, pad=1, shift=1, bounds=(3,),
                   capacity=APPEND_CAPACITY),
        AppendCase("bf16-big-vec", BF16, False, False, 4, 0, 2100, 1024, 1024),
        AppendCase("bf16-big-scalar", BF16, False, False, 4, 0, 2100, 1020, 1020),
        AppendCase("fp32-at-big-vec", FP32, False, True, 2, 0, 2100, 512, 512, bounds=(5,), capacity=2200),
    ]
    for dt in (BF16, FP16):
        c += [
            AppendCase(f"{dt}-fp8", dt, True, False, 3, 17, 5, 64, 32),
            AppendCase(f"{dt}-fp8-strided", dt, True, False, 2, 9, 4, 32, 48, pad=16, shift=16),
            AppendCase(f"{dt}-fp8-inplace-k", dt, True, False, 2, 12, 3, 64, 16, alias_k=True),
            AppendCase(f"{dt}-fp8-at", dt, True, True, 4, 0, 6, 64, 32, bounds=APPEND_AT_BOUNDS,
                       capacity=APPEND_CAPACITY),
        ]
    c.append(AppendCase("bf16-fp8-big", BF16, True, False, 4, 0, 2100, 1024, 1024))
    return c


APPEND_CASES = _append_cases()


class PackCase(NamedTuple):
    name: str
    B: int
    M: int
    stride_pad: int = 0   # extra mask bytes per batch row: a column slice, stride_b = M + stride_pad
    dv: int = 16

    @property
    def words(self):
        return self.B * pad_words_per_row(self.M)

    @property
    def sweeps(self):
        return sweeps(self.words, pack_blocks(self.B, self.M))


PACK_CASES = [PackCase(f"M{M}", 3, M) for M in (1, 31, 32, 33, 127, 128, 129, 4097)] + [
    PackCase("M129-sliced", 3, 129, stride_pad=37),
    PackCase("M8193-B1024", 1024, 8193),      # 266,240 words: past one sweep of 1024 blocks
]
PACK_BWD_MS = (31, 32, 33, 127, 128, 129)


def matrix_instantiations():
    out = {c.instantiation for c in ROTARY_CASES} | {c.instantiation for c in APPEND_CASES}
    return out | ({("pack_pad",)} if PACK_CASES else set())


# ---- inputs ----
def angle_table(Ba, rows, rd, seed, device="cpu"):
    """(Ba, rows, rd) fp32 angles with a[2p] != a[2p+1]: uniform in [-8, 8) per channel, every 7th row (from row 3) all
    zero, and rows 5 and 6 mod 7 above 1e5 and 1e8, where sincosf takes its large-argument reduction."""
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(Ba, rows, rd, generator=g, dtype=torch.float64) * 16 - 8
    r = torch.arange(rows)
    a[:, r % 7 == 3] = 0
    a[:, r % 7 == 5] = 1e5 + torch.rand(Ba, int((r % 7 == 5).sum()), rd, generator=g, dtype=torch.float64) * 1e3
    a[:, r % 7 == 6] = 1e8 + torch.rand(Ba, int((r % 7 == 6).sum()), rd, generator=g, dtype=torch.float64) * 1e6
    return a.float().to(device)


def zero_angle_rows(angles):
    """(Ba, rows) bool: rows whose angles are all zero."""
    return (angles == 0).all(-1)


# ---- oracles ----
def rotate64(x, a, rd, mut=None):
    """The header's rotation (pcv_attn.h:143-145) in fp64: x (B, n, H, d) with per-row angles a (B, n, >= rd); channels
    [0, rd) rotated pairwise, the rest pass through.  -> (y, mag), mag = |x[2p]| + |x[2p+1]| on rotated channels, 0
    elsewhere.  Mutants: one angle per pair (a[2p] for both channels), swapped rotation sign, the pass-through boundary
    one pair early or one pair late (the extra pair rotated by the first pair's angles)."""
    x, a = x.double(), a.double()[:, :, None, :]
    d = x.shape[-1]
    np_ = rd // 2
    if mut == "pass_boundary_minus_pair":
        np_ = max(0, np_ - 1)
    y, mag = x.clone(), torch.zeros_like(x)
    e, o = x[..., 0:2 * np_:2], x[..., 1:2 * np_:2]
    ae, ao = a[..., 0:2 * np_:2], a[..., 1:2 * np_:2]
    if mut == "one_angle_per_pair":
        ao = ae
    if mut == "swapped_sign":
        y[..., 0:2 * np_:2] = e * torch.cos(ae) + o * torch.sin(ae)
        y[..., 1:2 * np_:2] = o * torch.cos(ao) - e * torch.sin(ao)
    else:
        y[..., 0:2 * np_:2] = e * torch.cos(ae) - o * torch.sin(ae)
        y[..., 1:2 * np_:2] = o * torch.cos(ao) + e * torch.sin(ao)
    m = (e.abs() + o.abs())
    mag[..., 0:2 * np_:2], mag[..., 1:2 * np_:2] = m, m
    if mut == "pass_boundary_plus_pair" and 2 * np_ + 2 <= d:
        c = 2 * np_
        e1, o1 = x[..., c], x[..., c + 1]
        y[..., c] = e1 * torch.cos(a[..., 0]) - o1 * torch.sin(a[..., 0])
        y[..., c + 1] = o1 * torch.cos(a[..., 1]) + e1 * torch.sin(a[..., 1])
    return y, mag


ROTARY_MUTANTS = ("one_angle_per_pair", "swapped_sign", "pass_boundary_minus_pair", "pass_boundary_plus_pair",
                  "angle_row_plus_1", "broadcast_batch_ignored")


def select_angles(case: RotaryCase, angles, mut=None):
    """The angle row of every input row, gathered: angles (Ba, n_angles, rd) -> (B, n, rd) fp64, with the rows of
    RotaryCase.rows and the a_stride_b rule.  Mutants: every angle row one later (clamped to the table); the batch
    stride ignored (batch row 0's angles everywhere)."""
    arow, _, ok = case.rows()
    arow = torch.tensor(arow, dtype=torch.long)
    if mut == "angle_row_plus_1":
        arow = arow + 1
    arow = arow.clamp(0, angles.shape[1] - 1)
    ab = torch.arange(case.B)[:, None].expand(-1, case.n)
    if a_stride_b(angles.shape[0], case.B, 1) == 0 or mut == "broadcast_batch_ignored":
        ab = torch.zeros_like(ab)
    return angles.double().cpu()[ab, arow].to(angles.device)


def half_ulp(x, dt):
    """Half the spacing of `dt` at |x| (fp64), subnormals included."""
    emin, mbits = {BF16: (-126, 7), FP16: (-14, 10), E4M3: (-6, 3)}[dt]
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** emin)))
    return 0.5 * torch.exp2(e - mbits)


FP32_SLACK = 2.0 ** -20   # sincosf (2 ulp), the fp32 products and the sum: test_gpu_fp8_kv_cache.py:146-148


def rotary_excess(got, ref, mag, dt, scale=1.0):
    """(|got - ref| - half an ulp of `dt` - the fp32 slack), fp64, <= 0 everywhere when the kernel is right.  `scale`:
    the e4m3 output's y_inv_scale (broadcast), applied to ref and mag."""
    ref, mag = ref * scale, mag * scale
    slack = FP32_SLACK * (mag + ref.abs())
    return (got.double() - ref).abs() - half_ulp(ref.abs() + slack, dt) - slack


def e4m3_codes(x32, inv):
    """The header's expression (pcv_attn.h:537, ops.kv_append_fp8): clamp(x.float() * inv, +-448).to(e4m3) -- one fp32
    product, round to nearest even, saturating."""
    return (x32.float() * inv.float()).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def requant_rd0(codes, descale, inv):
    """rotary_fp8_kernel at rotate_dim = 0 on e4m3 input (:382-401): (code * descale) * inv, two fp32 products (no add,
    so nothing to contract), then RNE to e4m3 with satfinite.  codes (..., H, d), descale / inv (H,)."""
    x = codes.float() * descale.float()[:, None]
    return e4m3_codes(x, inv[:, None].expand_as(x))


APPEND_MUTANTS = ("dst_row_plus_1", "segment_dropped", "in_place_not_skipped")


def append_oracle(case: AppendCase, dst, k_cache, v_cache, k_new, v_new, k_inv=None, v_inv=None, mut=None):
    """dst (k_dst, v_dst) after the launch, bit for bit: the old rows (unless the half is in place), then the new rows
    at dst_row (AT) or L_old + row, quantised to e4m3 codes for an fp8 arena.  Every tensor a (B, rows, C) view; dst
    tensors are cloned.  Mutants: every new row one row later (dropped at the end of the tensor); the fresh V segment
    (blockIdx.y 3, :274-275) dropped; the in-place half (:624) copied from its (differently strided) cache view."""
    out = []
    for half, (dst_t, cache, new, inv) in enumerate(((dst[0], k_cache, k_new, k_inv), (dst[1], v_cache, v_new, v_inv))):
        t = dst_t.clone()
        skip = half == 0 and case.alias_k and mut != "in_place_not_skipped"
        if case.L_old and not skip:
            t[:, :case.L_old] = cache
        if not (half == 1 and mut == "segment_dropped"):
            vals = e4m3_codes(new, inv) if case.fp8 else new
            rows, ok = append_rows(case)
            rows = rows + (mut == "dst_row_plus_1")
            ok = ok & (rows >= 0) & (rows < t.shape[1])
            bi = torch.arange(case.B)[:, None].expand_as(rows)
            dev = t.device
            t[bi[ok].to(dev), rows[ok].to(dev)] = vals[ok.to(dev)]
        out.append(t)
    return out


def append_rows(case: AppendCase):
    """(destination row (B, n), written (B, n)) of every new row: dst_row<AT> or L_old + row."""
    r = torch.arange(case.n)[None, :].expand(case.B, -1)
    if not case.at:
        return case.L_old + r, torch.ones(case.B, case.n, dtype=torch.bool)
    b0 = torch.tensor([case.bounds[b % len(case.bounds)] for b in range(case.B)])[:, None]
    rows = b0 + r
    return rows, (rows >= 0) & (rows < case.capacity)


PACK_MUTANTS = ("word_shifted_one_bit",)


def pack_words(pad, mut=None):
    """pack_pad_kernel (:406-419) on a (B, M) bool mask: (B, wpr) int64 words, bit i of word w = pad[b, 32 w + i] for
    32 w + i < M, 0 past M.  Mutant: every word shifted up one bit."""
    B, M = pad.shape
    wpr = pad_words_per_row(M)
    bits = torch.zeros(B, 32 * wpr, dtype=torch.int64, device=pad.device)
    bits[:, :M] = pad.long()
    w = (bits.reshape(B, wpr, 32) << torch.arange(32, device=pad.device)).sum(-1)
    if mut == "word_shifted_one_bit":
        w = (w << 1) & 0xFFFFFFFF
    return w


def unpack_words(words, M):
    B, wpr = words.shape
    bits = (words[..., None] >> torch.arange(32, device=words.device)) & 1
    return bits.reshape(B, 32 * wpr)[:, :M].bool()


def count_expect(pad, dv):
    """The count probe of the tensor-core forward (q = 0, v_j = e_(j mod dv)): every live score is 0, so a batch row
    with a live key has m = 0, l = its unpadded key count and o[c] = its unpadded keys j = c (mod dv); a fully padded
    row takes the finite fill (gpu_util.assert_partial_state): m = -FLT_MAX, l = M, o[c] = every key j = c (mod dv).
    -> (o (B, dv), m (B,), l (B,)) fp64."""
    B, M = pad.shape
    j = torch.arange(M, device=pad.device)
    onehot = torch.nn.functional.one_hot(j % dv, dv).double()
    live = (~pad).double()
    dead = ~(live.sum(-1) > 0)
    w = torch.where(dead[:, None], torch.ones_like(live), live)
    m = torch.where(dead, torch.full((B,), -torch.finfo(torch.float32).max, dtype=torch.float64, device=pad.device),
                    torch.zeros(B, dtype=torch.float64, device=pad.device))
    return w @ onehot, m, w.sum(-1)


def probe_mask(B, M, seed, device="cpu", stride_pad=0):
    """(B, M) bool view of a (B, M + stride_pad) mask: batch row 0 padded at every word edge (keys 0, 31, 32, 63, 64,
    127, 128 and M - 1) and at random keys, row 1 fully padded, row 2 unpadded, further rows random."""
    g = torch.Generator().manual_seed(seed)
    full = torch.rand(B, M + stride_pad, generator=g) < 0.4
    for j in (0, 31, 32, 63, 64, 127, 128, M - 1):
        if j < M:
            full[0, j] = True
    if B > 1:
        full[1, :M] = True
    if B > 2:
        full[2, :M] = False
    if M > 2 and B > 0:
        full[0, 1] = False      # row 0 keeps a live key
    return full.to(device)[:, :M]


# ---- the rotary backward shim (ops._Rotary.backward) ----
def rotary_backward_mutant(gy, angles, H, right_align, mut):
    """ops._Rotary.backward (ops.py:842-856) with its angle roles swapped ('swapped_pair_angles': ae <-> ao) or one
    angle per pair ('one_angle_per_pair'); gy (B, n, H*d)."""
    B, n, Cx = gy.shape
    d, f = Cx // H, angles.shape[-1]
    a = angles[:, angles.shape[1] - n:] if right_align else angles[:, :n]
    a = a[:, :, None, :].double()
    g = gy.double().reshape(B, n, H, d)
    ge, go = g[..., :f][..., 0::2], g[..., :f][..., 1::2]
    ae, ao = a[..., 0::2], a[..., 1::2]
    if mut == "swapped_pair_angles":
        ae, ao = ao, ae
    elif mut == "one_angle_per_pair":
        ao = ae
    dxe = ge * torch.cos(ae) + go * torch.sin(ao)
    dxo = go * torch.cos(ao) - ge * torch.sin(ae)
    return torch.cat([torch.stack([dxe, dxo], dim=-1).flatten(-2), g[..., f:]], dim=-1).reshape(B, n, Cx)


def rotary_autograd64(x, angles, H, right_align):
    """fp64 autograd reference of ops.rotary: x (B, n, H*d) -> y, with the reference's row selection."""
    B, n, Cx = x.shape
    a = angles.double()
    a = a[:, a.shape[1] - n:] if right_align else a[:, :n]
    y, _ = rotate64(x.reshape(B, n, H, Cx // H), a.expand(B, -1, -1), a.shape[-1])
    return y.reshape(B, n, Cx)
