"""The M-sharded forward's fused merge (peer_tail_kernel<BF16>, csrc/pcv_attn_tc.cu:171-269): its rules restated, the
flag protocol that lets G ranks run one after another on one GPU, the variant matrix, a restatement of the merge in
source order, and the gates the GPU test applies.  Shared by test_tail_variants_cpu.py (the rules, the matrix and the
gates against mutants, on the CPU) and test_gpu_tail_variants.py (the kernel on one GPU).

pcv_attn_fwd_sharded (csrc/pcv_api.cu) launches the attention kernel of rank r's key shard into part[r] (plus
tc_combine_kernel when the plan splits the keys) and then the tail: publish, wait for every rank's state, merge the
rows rank r owns from all G states, store them into every rank's output, a grid-wide arrival, a second flag exchange.
One GPU stands in for G ranks when every flag word rank r's tail waits on is written before its launch
(preset_flags) and the ranks are launched one after another: no wait can then block.  Launching two simulated ranks
at once is never safe: each tail needs its whole grid co-resident and would spin on the other."""
from typing import NamedTuple

import numpy as np
import torch

import merge_variants as MV

BF16, FP16 = MV.BF16, MV.FP16
DTYPES = MV.DTYPES
TORCH_DTYPE = MV.TORCH_DTYPE
MAX_PEERS = MV.MAX_PEERS    # PCV_MAX_PEERS (include/pcv_attn.h)
TAIL_THREADS = 256          # kTailThreads (pcv_attn_tc.cu:115); the grid is one CTA per SM (:1434-1440)
TAIL_WARPS = TAIL_THREADS // 32
CHANNEL_STEP = 128          # c = 4 * lane; c < dv; c += 128 (:206)
FLAG_WORDS = 64             # dist.PeerMerger's flag block (dist.py:178); the header asks for >= 32 words
ARRIVE_WORD = 18            # tail_grid_arrive_wait(lf + 18, epoch * grid, 42) (:176, :258)
STAMP_WORDS = tuple(range(24, 30))   # PCV_TAIL_STAMP(0..5) of CTA 0 (:181-184)
H100_SMS = 132              # the grid on an H100 SXM; the GPU test takes the device's own count
MAX_DV_PASS = 128           # one attention launch per 128 V channels (launch_attn_tc, pcv_attn_tc.cu:1418)
WAIT_SITES = (41, 42, 43)   # tail_wait_ge sites: complete flags, grid arrival, pushed flags (:195, :258, :263)


def cdiv(a, b):
    return -(-a // b)


# ---- the rules ----
def rank_rows(R, G, r):
    """Rank r's rows [R*r/G, R*(r+1)/G) of the flattened (b, h, n) space: launch_attn_tc (pcv_attn_tc.cu:1408-1409),
    the same rule as dist.PeerMerger's slices (merge_variants.peer_rows, dist.py:186-187)."""
    return MV.peer_rows(R, G, r)


def rows_per_iter(G):
    """RB = PCV_MAX_PEERS / G rows per warp iteration (:202)."""
    return MAX_PEERS // G


def warp_blocks(R, G, r):
    """nblk = ceil((row_end - row_begin) / RB) warp iterations of rank r (:203)."""
    lo, hi = rank_rows(R, G, r)
    return cdiv(hi - lo, rows_per_iter(G))


def source(j, G):
    """Source j of a warp iteration is row r0 + j / G of rank j % G (:211) -> (rr, g)."""
    return j // G, j % G


def source_live(j, G, r0, row_end):
    """A source is loaded iff rr < RB && r0 + rr < row_end (:213); a dead one holds m = -inf, l = 0, x = 0."""
    rr, _ = source(j, G)
    return rr < rows_per_iter(G) and r0 + rr < row_end


def dead_sources(G):
    """Sources that no row of a full iteration uses: j >= RB * G."""
    return [j for j in range(MAX_PEERS) if source(j, G)[0] >= rows_per_iter(G)]


def warp_loop_wraps(R, G, sms):
    """Some rank's warp loop runs a second round: nblk > grid * 8 warps (:204)."""
    return any(warp_blocks(R, G, r) > sms * TAIL_WARPS for r in range(G))


def channel_iters(dv):
    """The channel loop: lane l handles 4 channels at c = 4 l, 4 l + 128, ... below dv (:206).  -> list of the lanes
    active in each iteration."""
    return [[lane for lane in range(32) if 4 * lane + it * CHANNEL_STEP < dv] for it in range(cdiv(dv, CHANNEL_STEP))]


def complete_words(G):
    """lf[0, G): "rank g's partial state is complete", written by rank g, waited on by thread g (:191-195)."""
    return list(range(G))


def pushed_words(G):
    """lf[G, 2G): "rank g has pushed all its rows", written by rank g, waited on by thread g of CTA 0 (:260-264)."""
    return list(range(G, 2 * G))


def written_words(r, G):
    """(block, word) pairs rank r's tail writes: flags[g][r] and flags[g][G + r] for every g (:193, :262), its own
    arrival counter and its phase stamps."""
    out = {(g, r) for g in range(G)} | {(g, G + r) for g in range(G)}
    return out | {(r, ARRIVE_WORD)} | {(r, w) for w in STAMP_WORDS}


def preset_flags(flags, r, G, e):
    """Write the words of rank r's flag block that the OTHER ranks would have written by epoch e: lf[g] and lf[G + g]
    for every g != r.  `flags` is (G, FLAG_WORDS), rank g's block in row g (host or device)."""
    others = [g for g in range(G) if g != r]
    if others:
        flags[r, others] = e
        flags[r, [G + g for g in others]] = e


def wait_set_satisfied(flags, r, G, e, grid):
    """Every wait of rank r's tail at epoch e completes if launched now, alone: lf[0, G) and lf[G, 2G) >= e except
    rank r's own words (it writes them before it waits on them), and the arrival counter lf[18] == (e - 1) * grid, so
    that the grid's own arrivals take it to the target e * grid.  `flags` is a host copy, (G, FLAG_WORDS)."""
    lf = [int(x) for x in flags[r]]
    others = [g for g in range(G) if g != r]
    return (all(lf[g] >= e for g in others) and all(lf[G + g] >= e for g in others)
            and lf[ARRIVE_WORD] == (e - 1) * grid)


# ---- the variant matrix ----
class TailCase(NamedTuple):
    dt: str
    G: int
    B: int
    H: int
    N: int
    Ms: int         # keys per shard: m_total = G * Ms in G equal shards (dist.py takes the fused path only then)
    dqk: int
    dv: int
    mask: str       # "none", "pad" or "causal"
    o_pad: int      # elements after each output row of H * dv (o_stride_n = H * dv + o_pad)

    @property
    def R(self):
        return self.B * self.H * self.N

    @property
    def m_total(self):
        return self.G * self.Ms

    @property
    def shards(self):
        return [(g * self.Ms, (g + 1) * self.Ms) for g in range(self.G)]

    @property
    def W(self):
        return self.H * self.dv + self.o_pad

    @property
    def strides(self):
        return (self.N * self.W, self.W, self.dv)


TAIL_CASES = (
    # R = 9600: the warp loop wraps past 132 * 8 warps at G = 1 (RB = 8) and at G = 8 (RB = 1)
    TailCase(BF16, 1, 2, 8, 600, 256, 64, 64, "pad", 0),
    TailCase(FP16, 8, 2, 8, 600, 128, 64, 128, "causal", 0),
    # R < G: ranks that own no rows still publish, arrive and exit
    TailCase(BF16, 5, 1, 1, 3, 64, 32, 8, "causal", 8),
    TailCase(FP16, 6, 1, 1, 4, 24, 32, 200, "causal", 0),
    TailCase(FP16, 7, 1, 2, 3, 48, 64, 64, "none", 8),
    TailCase(BF16, 8, 1, 1, 5, 16, 16, 200, "none", 8),
    # the split plan: tc_combine_kernel writes each rank's state before the tail
    TailCase(FP16, 2, 3, 1, 129, 2048, 64, 64, "pad", 0),
    TailCase(BF16, 3, 1, 2, 200, 1536, 128, 200, "causal", 8),
    # every other (dtype, G), R not divisible by G, ragged last iterations, dv 8 / 64 / 128 / 200, both layouts
    TailCase(FP16, 1, 1, 3, 41, 96, 40, 200, "causal", 8),
    TailCase(BF16, 2, 2, 3, 37, 160, 72, 200, "pad", 8),
    TailCase(BF16, 3, 2, 1, 50, 64, 8, 8, "pad", 0),
    TailCase(FP16, 3, 1, 2, 7, 32, 32, 64, "causal", 8),
    TailCase(BF16, 4, 2, 2, 101, 32, 64, 128, "causal", 0),
    TailCase(FP16, 4, 2, 1, 3, 16, 16, 8, "pad", 8),
    TailCase(FP16, 5, 2, 2, 33, 48, 48, 64, "pad", 0),
    TailCase(BF16, 6, 2, 1, 19, 40, 24, 128, "pad", 8),
    TailCase(BF16, 7, 2, 2, 10, 24, 16, 64, "pad", 0),
    TailCase(FP16, 8, 2, 1, 30, 16, 24, 8, "pad", 8),
)


def case_id(c: TailCase) -> str:
    return (f"{c.dt}-G{c.G}-B{c.B}H{c.H}N{c.N}-Ms{c.Ms}-dqk{c.dqk}-dv{c.dv}-{c.mask}"
            + (f"-opad{c.o_pad}" if c.o_pad else ""))


def pad_mask(c: TailCase, seed=0):
    """(B, m_total) bool, True = padding, or None.  Batch row 1 is padded in every shard (every rank's row maximum is
    the finite fill: uniform rows); batch row 0 is padded over the whole last shard (one rank's maximum is the fill,
    the others' are live); about 20 % of the remaining keys are padded at random."""
    if c.mask != "pad":
        return None
    g = torch.Generator().manual_seed(seed)
    pad = torch.rand(c.B, c.m_total, generator=g) < 0.2
    pad[1] = True
    if c.G > 1:
        a, b = c.shards[-1]
        pad[0, a:b] = True
    return pad


def future_shards(c: TailCase, n=0):
    """Shards wholly in the future of query row n under the right-aligned causal mask (key j is masked for row n iff
    j > n + m_total - N): their partial state of that row is m = -inf, l = 0, so the merge weights them 0."""
    shift = c.m_total - c.N
    return [g for g, (a, _) in enumerate(c.shards) if a > n + shift]


# ---- the merge in source order, on the CPU ----
TAIL_MUTANTS = ("slice_off_by_one", "dead_guard_dropped", "rb_plus_one", "unweighted_l")


class AddressError(IndexError):
    """A load outside rank g's part buffer: on the device, a read past the allocation."""


def part_flat(po, pm, pl):
    """Rank g's part buffer as the tail addresses it (launch_attn_tc, pcv_attn_tc.cu:1400-1403): f32
    [ numerator (R, dv) | row max (R) | denominator (R) ] in one allocation."""
    return np.concatenate([po.reshape(-1), pm.reshape(-1), pl.reshape(-1)]).astype(np.float32)


def _fmaf(a, b, c):
    """fmaf on float32 operands: the exact product (48 bits) plus c in float64, rounded once more to float32; a double
    rounding that agrees with fmaf wherever the float64 sum is exact, as it is on the dyadic states."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def tail_emulate(parts, G, rank, R, dv, outs, dtype, mut=None):
    """Rank `rank`'s tail merge (pcv_attn_tc.cu:202-255) over `parts` (G flat f32 buffers, part_flat), in its order:
    per warp iteration the loads of the 8 sources, then per row the max, the weighted sums in source (= rank) order
    and the product with 1 / l, rounded to `dtype` and stored into every outs[g] ((R, dv) float32 tensors standing
    for the 16-bit rows).  Loads are bounds-checked (AddressError).  exp2 of the dyadic states is exact, as the
    device's exp2f is on integers (test_gpu_merge_variants.py::test_exp2f_of_integers_is_exact).
    Mutants: row_begin one row early; the dead-source guard dropped (every source loaded); RB = 8 / G + 1; l summed
    without the weights."""
    size = R * dv + 2 * R
    RB = rows_per_iter(G) + (1 if mut == "rb_plus_one" else 0)
    lo, hi = rank_rows(R, G, rank)
    if mut == "slice_off_by_one" and rank > 0:
        lo -= 1
    nblk = cdiv(hi - lo, RB)
    cs = np.arange(0, dv, 4)                                            # every lane's channel starts, all iterations
    cols = (cs[:, None] + np.arange(4)[None, :]).reshape(-1)

    def load(g, idx):
        if np.any(idx < 0) or np.any(idx >= size):
            raise AddressError(f"rank {rank}: load of rank {g}'s part at element {int(np.max(idx))} of {size}")
        return parts[g][idx]

    for blk in range(nblk):
        r0 = lo + blk * RB
        mg = np.full(MAX_PEERS, -np.inf, dtype=np.float32)
        lg = np.zeros(MAX_PEERS, dtype=np.float32)
        x = np.zeros((MAX_PEERS, cols.size), dtype=np.float32)
        for j in range(MAX_PEERS):
            rr, g = source(j, G)
            r = r0 + rr
            live = rr < RB and r < hi
            if mut == "dead_guard_dropped":
                live = g < G
            if live:
                mg[j] = load(g, np.array([R * dv + r]))[0]
                lg[j] = load(g, np.array([R * dv + R + r]))[0]
                x[j] = load(g, r * dv + cols)
        for rr in range(RB):
            r = r0 + rr
            if r >= hi:
                break
            js = [j for j in range(MAX_PEERS) if j // G == rr]
            m = np.float32(-np.inf)
            for j in js:
                m = np.maximum(m, mg[j])
            l = np.zeros(1, dtype=np.float32)
            acc = np.zeros(cols.size, dtype=np.float32)
            for j in js:
                w = np.float32(0.0) if mg[j] == -np.inf else np.float32(np.exp2(np.float64(mg[j]) - np.float64(m)))
                w1 = np.array([w], dtype=np.float32)
                l = _fmaf(np.array([lg[j]]), np.ones(1, np.float32) if mut == "unweighted_l" else w1, l)
                acc = _fmaf(x[j], np.full(cols.size, w, dtype=np.float32), acc)
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = np.float32(1.0) / l[0]
                val = (acc * inv).astype(np.float32)
            row = torch.from_numpy(val).to(dtype).float()
            for g in range(G):
                outs[g][r, cols] = row


# ---- the gates (the GPU test applies the same ones to the kernel's output, in (b, h, n) row order) ----
def _bits(t):
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t.view(torch.int32)


def gate_one_rank(outs, lo, hi, want, what=""):
    """After one rank's launch alone: rows [lo, hi) of every outs[g] equal `want` bit for bit, every other row is
    still NaN.  outs / want: (R, dv) in the output dtype."""
    for g, o in enumerate(outs):
        inside = torch.zeros(o.shape[0], dtype=torch.bool, device=o.device)
        inside[lo:hi] = True
        assert o[~inside].isnan().all(), f"{what}: out[{g}] has rows outside [{lo}, {hi}) written"
        assert torch.equal(_bits(o[inside]), _bits(want[inside].to(o.device))), \
            f"{what}: out[{g}] rows [{lo}, {hi}) differ from the merge"


def gate_complete(outs, want=None, what=""):
    """After every rank's launch: no NaN in any row, every outs[g] the same bits, equal to `want` when given."""
    for g, o in enumerate(outs):
        assert not o.isnan().any(), f"{what}: out[{g}] has {int(o.isnan().sum())} NaN elements (rows never written)"
        assert torch.equal(_bits(o), _bits(outs[0])), f"{what}: out[{g}] differs from out[0]"
    if want is not None:
        assert torch.equal(_bits(outs[0]), _bits(want.to(outs[0].device))), f"{what}: the merge differs from the reference"


def reference_rows(po, pm, pl, dtype):
    """RN16 of the fp64 merge (merge_variants.merge_reference) of (G, R, dv) states -> (R, dv) in dtype."""
    acc, _, l = MV.merge_reference(po, pm, pl)
    return (acc / l[..., None]).to(dtype)


def emulate_all(po, pm, pl, dtype, mut=None, order=None):
    """Every rank's tail on the CPU, rank G-1 first: -> (outs after rank G-1 alone, outs after all ranks)."""
    G, R, dv = po.shape
    parts = [part_flat(po[g].numpy(), pm[g].numpy(), pl[g].numpy()) for g in range(G)]
    outs = [torch.full((R, dv), float("nan")) for _ in range(G)]
    order = [G - 1] + list(range(G - 1)) if order is None else order
    first = None
    for i, r in enumerate(order):
        tail_emulate(parts, G, r, R, dv, outs, dtype, mut)
        if i == 0:
            first = [o.to(dtype) for o in outs]
    return first, [o.to(dtype) for o in outs]
