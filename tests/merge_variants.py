"""The CUDA-core attention kernel (csrc/pcv_attn_simt.cu) and the partial-state merge kernels (csrc/pcv_aux.cu:16-183):
their rules restated, the variant matrix that reaches every instantiation, and exact probes.  Shared by
test_merge_variants_cpu.py (the rules against the library and against mutants, on the CPU) and
test_gpu_merge_variants.py (the kernels against the probes and fp64).

Instantiations: attn_simt_kernel<T, DVW> (T in bf16 / fp16, DVW in 1, 2, 4, 8), combine_kernel<T>, combine_peers_kernel<T>
and rescale_kernel: 13.  A SIMT call runs in one of four modes: `direct` (one split writes the output), `split_combine`
(splits into the workspace, combine_kernel normalises), `single_partial` (one split writes the caller's partial state)
and `split_partial` (splits merged by combine_kernel into the partial state, the merge_partials path)."""
import itertools
from typing import NamedTuple, Optional

import torch

import decode_variants as DV

BF16, FP16 = "bf16", "fp16"
DTYPES = (BF16, FP16)
TORCH_DTYPE = {BF16: torch.bfloat16, FP16: torch.float16}
FLT_MAX = torch.finfo(torch.float32).max
LOG2E = 1.4426950408889634

ROWS_PER_CTA = 32          # kRowsPerCta (pcv_attn_simt.cu:20): 8 warps x 4 rows
KEYS_PER_TILE = 32         # kKeysPerTile (:21)
WANT_CTAS = 132 * 4        # make_plan: ~2 waves at 2 CTAs/SM (:192), not the device's SM count
SPLIT_KEYS = 256           # make_plan: at most ceil(M / 256) splits (:194)
SMEM_DEFAULT = 48 * 1024   # launch_t raises the dynamic shared-memory attribute above 48 KB (:210)
SMEM_MAX = 200 * 1024      # launch_attn_simt refuses larger tiles (:257)
DVWS = (1, 2, 4, 8)
MODES = ("direct", "split_combine", "single_partial", "split_partial")
MAX_PEERS = 8              # PCV_MAX_PEERS (include/pcv_attn.h)
PEERS_FAST_MAX_DV = 128    # combine_peers fast path: one float4 per lane (pcv_aux.cu:90-95)
# The exact probes weight their parts by exp2f of integers no smaller than this: exp2f is exact on the normal range
# (test_gpu_merge_variants.py::test_exp2f_of_integers_is_exact), not at every subnormal result.
MIN_PROBE_EXP = -126


def cdiv(a, b):
    return -(-a // b)


# ---- the SIMT plan (pcv_attn_simt.cu:189-205, 235-243, 150, 215-223) ----
class Plan(NamedTuple):
    nsplit: int
    kps: int          # keys per split, a multiple of 32
    smem: int         # dynamic shared memory bytes


def simt_plan(B, H, N, M, dqk, dv) -> Plan:
    ctas = cdiv(N, ROWS_PER_CTA) * B * H
    nsplit = max(1, min(cdiv(WANT_CTAS, ctas), cdiv(M, SPLIT_KEYS)))
    kps = cdiv(cdiv(M, nsplit), KEYS_PER_TILE) * KEYS_PER_TILE
    nsplit = cdiv(M, kps)
    dq2, dv2 = cdiv(dqk, 2), cdiv(dv, 2)
    qs = dq2 | 1
    return Plan(nsplit, kps, 4 * ((ROWS_PER_CTA + KEYS_PER_TILE) * qs + KEYS_PER_TILE * dv2))


def dvw_of(dv) -> Optional[int]:
    """launch_dv: the smallest DVW with 32 * DVW >= ceil(dv / 2) channel pairs; None above dv = 512."""
    w = cdiv(cdiv(dv, 2), 32)
    return next((d for d in DVWS if w <= d), None)


def mode_of(nsplit, partial) -> str:
    if nsplit == 1:
        return "single_partial" if partial else "direct"
    return "split_partial" if partial else "split_combine"


def split_ranges(M, plan: Plan):
    return [(s * plan.kps, min(M, (s + 1) * plan.kps)) for s in range(plan.nsplit)]


def workspace_bytes(B, H, N, M, dqk, dv) -> int:
    """attn_simt_workspace_bytes (:247-252): nsplit fp32 (o, m, l) states of every row when the plan splits."""
    nsplit = simt_plan(B, H, N, M, dqk, dv).nsplit
    return 4 * nsplit * B * H * N * (dv + 2) if nsplit > 1 else 0


def serial_depth(plan: Plan) -> int:
    """The longest chain of fp32 roundings a probability passes through (gpu_util.decode_element_bound's `depth`): the
    key-serial fma chain of o over a split, one rescale per tile, the 5-level warp_sum tree, the split merge, the final
    product with 1 / l."""
    return plan.kps + cdiv(plan.kps, KEYS_PER_TILE) + 5 + plan.nsplit + 2


# ---- the merge rules ----
def merge_weights(pm, m=None):
    """combine_kernel (pcv_aux.cu:29-35) / combine_peers (:110-117) / rescale (:166): w_g = 0 for m_g = -inf, else
    exp2(m_g - m) with m the row max (or rescale's new_m).  The finite fill m_g = -FLT_MAX has weight exp2(-FLT_MAX - m)
    = 0 against a live part and exp2(0) = 1 when every part is filled.  pm (G, rows) -> (w (G, rows), m (rows))."""
    if m is None:
        m = pm.amax(0)
    w = torch.where(pm == float("-inf"), torch.zeros_like(pm), torch.exp2(pm - m))
    return w, m


def peers_fast_path(dv, strides, part_ptrs, out_ptrs, aligned=True) -> bool:
    """launch_combine_peers' fast-path predicate (pcv_aux.cu peers_fast_path, stated in include/pcv_attn.h beside
    pcv_peer_combine_params): 16-byte loads of part_o rows, 8-byte stores of output rows.  aligned=False is the rule
    before the pointer terms were added (dv % 4 == 0 and dv <= 128 only)."""
    ok = dv % 4 == 0 and dv <= PEERS_FAST_MAX_DV
    if not aligned:
        return ok
    return (ok and all(s % 4 == 0 for s in strides) and all(p % 16 == 0 for p in part_ptrs)
            and all(p % 8 == 0 for p in out_ptrs))


def rescale_vector(dv, part_o_ptr, aligned=True) -> bool:
    """launch_rescale's float4 predicate; aligned=False is the rule before the pointer term (dv % 4 == 0 only)."""
    return dv % 4 == 0 and (not aligned or part_o_ptr % 16 == 0)


def peer_rows(rows, G, rank):
    """dist.PeerMerger's row slice of `rank` (dist.py:186-187)."""
    return rows * rank // G, rows * (rank + 1) // G


# ---- the variant matrix ----
class SimtCase(NamedTuple):
    dt: str
    B: int
    Bq: int
    H: int
    N: int
    M: int
    dqk: int
    dv: int
    causal: bool
    pad: bool
    partial: bool
    m_total: int       # == M unless the call is a key shard
    m_offset: int
    strided: bool      # q / k / v rows are slices of wider rows (row strides not multiples of 8)

    @property
    def plan(self) -> Plan:
        return simt_plan(self.B, self.H, self.N, self.M, self.dqk, self.dv)

    @property
    def variant(self):
        return (self.dt, dvw_of(self.dv), mode_of(self.plan.nsplit, self.partial))


DV_BY_DVW = {1: (1, 3, 64), 2: (65, 128), 4: (129, 256), 8: (257, 512)}
DQKS = (1, 37, 512, 513, 1024)
NS = (1, 31, 32, 33)
SHORT_MS = (1, 31, 32, 33, 255)
SPLIT_MS = (257, 511, 513, 767, 769)


def _matrix():
    cases, i = [], 0
    for dt in DTYPES:
        for dvw, dvs in DV_BY_DVW.items():
            for dv in dvs:
                for mode in MODES:
                    split = mode.startswith("split")
                    partial = mode.endswith("partial")
                    dqk, N = DQKS[i % len(DQKS)], NS[(i // 2) % len(NS)]
                    M = (SPLIT_MS if split else SHORT_MS)[i % 5]
                    Bq = 1 if i % 3 == 0 else 2
                    causal = M >= N and i % 2 == 1
                    m_total, m_offset = M, 0
                    if partial and i % 4 == 3:   # a key shard of a longer row, causal where it may be
                        m_offset = 7 + i % 11
                        m_total = M + m_offset + (i % 3) * 5
                        causal = m_total >= N
                    cases.append(SimtCase(dt, 2, Bq, 2, N, M, dqk, dv, causal, i % 5 != 2, partial, m_total, m_offset,
                                          i % 4 == 1))
                    i += 1
    return cases


SIMT_CASES = _matrix()


def case_id(c: SimtCase) -> str:
    s = f"{c.dt}-dqk{c.dqk}-dv{c.dv}-N{c.N}-M{c.M}" + ("-c" if c.causal else "") + ("-p" if c.pad else "")
    s += "-part" if c.partial else ""
    s += f"-sh{c.m_offset}of{c.m_total}" if c.m_total != c.M else ""
    return s + ("-bq1" if c.Bq == 1 else "") + ("-str" if c.strided else "")


def all_instantiations():
    return ({("attn_simt", dt, dvw) for dt in DTYPES for dvw in DVWS} | {("combine", dt) for dt in DTYPES}
            | {("combine_peers", dt) for dt in DTYPES} | {("rescale",)})


def case_instantiations(c: SimtCase):
    out = {("attn_simt", c.dt, dvw_of(c.dv))}
    if c.plan.nsplit > 1:
        out.add(("combine", c.dt))
    return out


# ---- probes of the SIMT kernel ----
def pad_mask(c: SimtCase, device="cpu"):
    """Batch row 1 fully padded (rows without a live key); batch row 0 padded on its second key and its last three."""
    if not c.pad:
        return None
    pad = torch.zeros(c.B, c.M, dtype=torch.bool, device=device)
    pad[1:] = True
    pad[0, 1:2] = True
    pad[0, max(0, c.M - 3):] = True
    return pad


def sets_of(c: SimtCase, device="cpu"):
    """(in_range, live) (B, N, M) of decode_variants.key_sets for the case's shard."""
    pad = pad_mask(c, device)
    return DV.key_sets(c.B, c.N, c.M, pad, c.causal, m_total=c.m_total, m_offset=c.m_offset, device=device)


def edge_marks(c: SimtCase, limit=60):
    """Keys under test of the count probe: the first and last key of every split, the first and last key of every
    32-key tile of the first and the last split (the ragged tile included), and the causal diagonal of the first and
    the last query row with the key after it.  Capped at `limit`, so that S stays below 64 codes (decode_variants)."""
    rs = split_ranges(c.M, c.plan)
    marks = {kb for kb, _ in rs} | {ke - 1 for _, ke in rs}
    for kb, ke in {rs[0], rs[-1]}:
        tiles = list(range(kb, ke, KEYS_PER_TILE))
        for j0 in tiles[:3] + tiles[-2:]:
            marks |= {j0, min(j0 + KEYS_PER_TILE, ke) - 1}
    if c.causal:
        shift = c.m_total - c.N - c.m_offset
        for n in (0, c.N - 1):
            marks |= {n + shift, n + shift + 1}
    marks = sorted(m for m in marks if 0 <= m < c.M)
    assert len(marks) <= limit, len(marks)
    return marks


def count_operands(c: SimtCase, seed=0, device="cpu"):
    """decode_variants.count_operands at the case's marks: q = 0, every live score is exactly 0."""
    pad = pad_mask(c, device)
    return DV.count_operands(c.B, c.Bq, c.N, c.M, c.H, c.dqk, c.dv, edge_marks(c),
                             torch.zeros(c.B, c.M, dtype=torch.bool, device=device) if pad is None else pad,
                             False, TORCH_DTYPE[c.dt], seed, device)


def simt_count_expect(v, H, in_range, live, dtype):
    """The count probe's output bit for bit: RN16(S * RN32(1 / L)).  The SIMT kernel and combine_kernel multiply by the
    fp32 reciprocal of l (pcv_attn_simt.cu:156, pcv_aux.cu:40), so the quotient of decode_variants.count_expect is not
    theirs; S and L are integers below 2^24."""
    S, L, _ = DV.count_state(v, H, in_range, live)
    assert S.abs().max().item() < 2 ** 24
    q = S.float() * (1.0 / L.float())[..., None]
    B, _, N, dv = q.shape
    return q.to(dtype).transpose(1, 2).reshape(B, N, H * dv)


def count_partial_expect(v, H, in_range, live):
    """The count probe's partial state bit for bit: o = S, l = L, m = 0 for live rows and -FLT_MAX for the others."""
    S, L, any_live = DV.count_state(v, H, in_range, live)
    m = torch.where(any_live, torch.zeros_like(L), torch.full_like(L, -FLT_MAX))
    return S.float(), m.float(), L.float()


NEEDLE_SCALE = DV.NEEDLE_SCALE


def needle_score(scale=NEEDLE_SCALE):
    """The needle's score as the kernel forms it: t = s * RN32(scale * log2e), s = 16 * 16 (pcv_attn_simt.cu:68, 115)."""
    sl = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    return (torch.tensor(256.0, dtype=torch.float32) * sl).item()


def needle_candidates(c: SimtCase):
    """Keys a needle is put on: the edge marks (split and tile edges, the diagonals) and the first and last padded key."""
    cand = set(edge_marks(c))
    pad = pad_mask(c)
    if pad is not None:
        idx = pad[0].nonzero()
        if idx.numel():
            cand |= {int(idx[0]), int(idx[-1])}
    return sorted(cand)


def needle_set(c: SimtCase, r):
    """(B, H, N) needles of round r (decode_variants.needles).  With dqk < N query rows share their needle channel
    (decode_variants.needle_channels), so they share one needle too."""
    nd = DV.needles(c.B, c.H, c.N, [needle_candidates(c)] * c.B, r)
    return nd[:, :, :1].expand(-1, -1, c.N).clone() if c.dqk < c.N else nd


def needle_rounds(c: SimtCase, cap=3):
    return min(cap, DV.needle_rounds([needle_candidates(c)] * c.B, c.H, c.N))


def needle_operands(c: SimtCase, needle, seed=0, device="cpu"):
    return DV.needle_operands(c.B, c.Bq, c.N, c.M, c.H, c.dqk, c.dv, needle, False, TORCH_DTYPE[c.dt], seed, device)


def needle_found(c: SimtCase, live, needle):
    B, H, N = needle.shape
    bi, ni = torch.arange(B)[:, None, None], torch.arange(N)[None, None, :]
    return live.cpu()[bi, ni, needle]                                          # (B, H, N)


def simt_needle_expect(c: SimtCase, v, in_range, live, needle):
    """Found: l = 1 (every other weight is exp2(-184.7) = 0 in fp32) and the row is RN16(v[needle]).  Not found: the
    count probe's row over the live keys (all of them score 0)."""
    B, M, H = c.B, c.M, c.H
    vh = v.double().reshape(B, M, H, -1)
    bi, hi = torch.arange(B)[:, None, None], torch.arange(H)[None, :, None]
    hit = vh[bi, needle, hi].float().to(TORCH_DTYPE[c.dt]).transpose(1, 2)      # (B, N, H, dv)
    base = simt_count_expect(v, H, in_range, live, TORCH_DTYPE[c.dt]).reshape(B, c.N, H, -1)
    return torch.where(needle_found(c, live, needle).transpose(1, 2)[..., None], hit, base).reshape(B, c.N, -1)


# ---- the SIMT kernel restated in torch fp32 (exact on the probes), with mutants ----
SIMT_MUTANTS = ("ke_plus_1", "ke_minus_1", "causal_shift_plus_1", "causal_shift_minus_1", "m_offset_ignored",
                "pad_out_of_range")


def simt_emulate(c: SimtCase, q, k, v, scale, mut=None):
    """The kernel's algorithm per split (pcv_attn_simt.cu:80-148), merged by merge_state and normalised as the kernel
    does.  Split order and key order do not matter on the probes: every partial sum is exact.  -> the output (B, N,
    H*dv) in the case's dtype, or the partial state (o, m, l) when c.partial."""
    B, M, H, N, dv = c.B, c.M, c.H, c.N, c.dv
    f32 = torch.float32
    qh = q.float().expand(B, -1, -1).reshape(B, N, H, -1).transpose(1, 2)
    kh = k.float().reshape(B, M, H, -1).transpose(1, 2)
    vh = v.float().reshape(B, M, H, -1).transpose(1, 2)
    sl = torch.tensor(scale, dtype=f32) * torch.tensor(LOG2E, dtype=f32)
    t_all = (qh @ kh.transpose(-1, -2)) * sl                                   # (B, H, N, M)
    pad = pad_mask(c)
    shift = c.m_total - N + {"causal_shift_plus_1": 1, "causal_shift_minus_1": -1}.get(mut, 0)
    jg = torch.arange(M) + (0 if mut == "m_offset_ignored" else c.m_offset)
    masked = torch.zeros(B, 1, N, M, dtype=torch.bool)
    if pad is not None:
        masked = masked | pad[:, None, None, :]
    if c.causal:
        masked = masked | (jg[None, :] > torch.arange(N)[:, None] + shift)[None, None]
    t_all = torch.where(masked, torch.full_like(t_all, -FLT_MAX), t_all)
    states = []
    for kb, ke in split_ranges(M, c.plan):
        ke = min(M, ke + 1) if mut == "ke_plus_1" else (ke - 1 if mut == "ke_minus_1" and ke - 1 > kb else ke)
        t, vv = t_all[..., kb:ke], vh[:, :, kb:ke]
        if mut == "pad_out_of_range":   # the ragged tile's lanes past ke filled as masked keys, V loaded as 0
            extra = cdiv(ke - kb, KEYS_PER_TILE) * KEYS_PER_TILE - (ke - kb)
            t = torch.cat([t, torch.full(t.shape[:-1] + (extra,), -FLT_MAX)], -1)
            vv = torch.cat([vv, torch.zeros(B, H, extra, dv)], 2)
        m = t.amax(-1)
        p = torch.exp2(t - m[..., None])
        states.append((p @ vv, m, p.sum(-1)))
    po, pm, pl = (torch.stack([s[i] for s in states]) for i in range(3))
    o, m, l = merge_state(po, pm, pl)
    if c.partial:
        return o, m, l
    out = (o * (1.0 / l)[..., None]).to(TORCH_DTYPE[c.dt])
    return out.transpose(1, 2).reshape(B, N, -1)


MERGE_MUTANTS = ("inf_weight_one", "ffill_weight_zero", "ffill_weight_zero_vs_live")


def merge_state(po, pm, pl, mut=None):
    """combine_kernel's merge in torch fp32, parts in order (pcv_aux.cu:29-47): (G, ..., dv) / (G, ...) -> (acc, m, l),
    un-normalised.  Mutants: a -inf part weighted 1; the finite fill weighted 0 (everywhere, or only against a live
    part)."""
    w, m = merge_weights(pm)
    if mut == "inf_weight_one":
        w = torch.where(pm == float("-inf"), torch.ones_like(w), w)
    elif mut == "ffill_weight_zero":
        w = torch.where(pm == -FLT_MAX, torch.zeros_like(w), w)
    elif mut == "ffill_weight_zero_vs_live":
        w = torch.where((pm == -FLT_MAX) & (m > -FLT_MAX), torch.zeros_like(w), w)
    acc = torch.zeros_like(po[0])
    l = torch.zeros_like(pl[0])
    for g in range(po.shape[0]):
        l = l + pl[g] * w[g]
        acc = acc + po[g] * w[g][..., None]
    return acc, m, l


def combine_emulate(po, pm, pl, dtype, mut=None):
    acc, _, l = merge_state(po, pm, pl, mut)
    return (acc * (1.0 / l)[..., None]).to(dtype)


# ---- dyadic partial states ----
ROW_KINDS = ("live", "dead", "dead_live", "dead_inf", "live_inf", "dead_live_inf")


def dyadic_states(G, rows, dv, seed, kinds=ROW_KINDS, base_range=40, span=12):
    """(po (G, rows, dv), pm (G, rows), pl (G, rows)) fp32 whose merge is exact in fp32: live parts have integer m =
    base - d (d in [0, span], one part at d = 0), l in 1..15 and o in -15..15; filled parts m = -FLT_MAX, an integer key
    count l and o a sum of integer V rows; -inf parts (padding slots, empty shards) m = -inf, l = 0, o = 0.  Row r is
    of kind kinds[r % len(kinds)] (with G = 1 the mixed kinds fall back to their first part).  The merged l is a power
    of two: the largest contributing part takes up the difference, so 1 / l is exact and the 16-bit output is the
    exact quotient rounded once."""
    g = torch.Generator().manual_seed(seed)
    po = torch.zeros(G, rows, dv, dtype=torch.float64)
    pm = torch.zeros(G, rows, dtype=torch.float64)
    pl = torch.zeros(G, rows, dtype=torch.float64)
    ri = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, generator=g).double()   # noqa: E731
    for r in range(rows):
        kind = kinds[r % len(kinds)]
        roles = {"live": ["L"], "dead": ["D"], "dead_live": ["D", "L"], "dead_inf": ["D", "I"], "live_inf": ["L", "I"],
                 "dead_live_inf": ["D", "L", "I"]}[kind]
        role = [roles[(gg + r) % len(roles)] for gg in range(G)]
        if "L" in roles and "L" not in role:
            role[0] = "L"
        if "D" in roles and "L" not in roles and "D" not in role:
            role[0] = "D"
        base = int(ri(-base_range, base_range))
        for gg, rl in enumerate(role):
            if rl == "L":
                pm[gg, r], pl[gg, r], po[gg, r] = base - int(ri(0, span)), ri(1, 15), ri(-15, 15, dv)
            elif rl == "D":
                pm[gg, r], pl[gg, r], po[gg, r] = -FLT_MAX, ri(1, 40), ri(-60, 60, dv)
            else:
                pm[gg, r], pl[gg, r] = float("-inf"), 0.0
        live = [gg for gg, rl in enumerate(role) if rl == "L"]
        if live:
            top = max(live, key=lambda gg: pm[gg, r])
            pm[top, r] = base
            contrib = live
        else:
            contrib = [gg for gg, rl in enumerate(role) if rl == "D"]
            top = contrib[0]
        mx = pm[contrib, r].max()
        w = {gg: (2.0 ** (pm[gg, r] - mx).item() if gg in live else 1.0) for gg in contrib}
        rest = sum(pl[gg, r].item() * w[gg] for gg in contrib if gg != top)
        p2 = 1.0
        while p2 < rest + 1:
            p2 *= 2
        pl[top, r] = (p2 - rest) / w[top]
    return po.float(), pm.float(), pl.float()


def merge_reference(po, pm, pl):
    """fp64 merge (acc, m, l) with the rule of merge_weights."""
    po, pm, pl = po.double(), pm.double(), pl.double()
    m = pm.amax(0)
    w = torch.where(pm == float("-inf"), torch.zeros_like(pm), torch.exp2(pm - m))
    return (po * w[..., None]).sum(0), m, (pl * w).sum(0)


def random_states(G, rows, dv, seed, kinds=("live", "dead_live", "live_inf")):
    """Random fp32 partial states: live parts with m in [-30, 30], l in [1, 100) and o normal with standard deviation
    l; filled and -inf parts as in dyadic_states."""
    g = torch.Generator().manual_seed(seed)
    po, pm, pl = dyadic_states(G, rows, dv, seed, kinds)
    live = torch.isfinite(pm)
    pm = torch.where(live, torch.rand(G, rows, generator=g) * 60 - 30, pm)
    l_r = 1 + torch.rand(G, rows, generator=g) * 99
    pl = torch.where(live, l_r, pl)
    po = torch.where(live[..., None], torch.randn(G, rows, dv, generator=g) * l_r[..., None], po)
    return po, pm, pl


def merge_element_bound(po, pm, pl, dtype):
    """(bound, ref) of the merge kernels' element-wise gate, in the form of gpu_util.decode_element_bound: the output is
    rounded to 16 bits once (u |ref|); before that every term passes through exp2f (2 ulp = 2^-22), G fma roundings on
    the numerator and on the denominator, the reciprocal and the product: 2 (G + 2) (2^-24 + 2^-22) sum_g |o_g| w_g / l.
    Twice the sum, plus one fp16 subnormal spacing."""
    acc, m, l = merge_reference(po, pm, pl)
    ref = acc / l[..., None]
    w = torch.where(pm.double() == float("-inf"), torch.zeros_like(pm.double()), torch.exp2(pm.double() - m))
    mag = (po.double().abs() * w[..., None]).sum(0) / l[..., None]
    G = po.shape[0]
    e32 = 2.0 * (G + 2) * (2.0 ** -24 + 2.0 ** -22) * mag
    u = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}[dtype]
    sp = 2.0 ** -24 if dtype == torch.float16 else 0.0
    return 2.0 * (u * ref.abs() + e32) + sp, ref


# ---- combine_peers and rescale restated, with mutants ----
PEER_MUTANTS = ("fast_path_at_dv132", "row_begin_ignored", "only_own_out")
RESCALE_MUTANTS = ("new_m_not_stored", "l_not_rescaled")


def peers_emulate(po, pm, pl, outs, row_begin, row_end, rank, dtype, mut=None):
    """One combine_peers call (pcv_aux.cu:80-156) on the CPU: rows [row_begin, row_end) of the (G, rows, dv) states
    merged and written into every outs[g] (rows, dv).  Mutants: the fast path taken whenever dv % 4 == 0 (lanes cover
    only 4 * 32 channels); r counted from 0 instead of row_begin; only outs[rank] written."""
    dv = po.shape[-1]
    rows = range(0, row_end - row_begin) if mut == "row_begin_ignored" else range(row_begin, row_end)
    rows = torch.tensor(list(rows), dtype=torch.long)
    if rows.numel() == 0:
        return
    vals = combine_emulate(po[:, rows], pm[:, rows], pl[:, rows], dtype)
    cols = dv
    if mut == "fast_path_at_dv132" and dv % 4 == 0:
        cols = min(dv, 4 * 32)
    targets = [outs[rank]] if mut == "only_own_out" else outs
    for o in targets:
        o[rows, :cols] = vals[:, :cols]


def rescale_emulate(po, pm, pl, new_m, mut=None):
    """rescale (pcv_aux.cu:161-183) in torch fp32 -> new (po, pm, pl)."""
    w = torch.where(pm == float("-inf"), torch.zeros_like(pm), torch.exp2(pm - new_m))
    return (po * w[..., None], pm if mut == "new_m_not_stored" else new_m.clone(),
            pl if mut == "l_not_rescaled" else pl * w)


def rescale_states(rows, dv, seed):
    """Dyadic states for rescale: live rows with integer m and new_m = m + e (e in 0..100, so w = 2^-e, o and l keep every
    bit), filled rows with new_m = -FLT_MAX (w = 1) or a finite new_m (w = 0), and -inf rows (w = 0)."""
    g = torch.Generator().manual_seed(seed)
    po, pm, pl = dyadic_states(1, rows, dv, seed, kinds=("live", "dead", "live", "dead_inf"))
    po, pm, pl = po[0], pm[0], pl[0]
    e = torch.randint(0, 101, (rows,), generator=g).float()
    e[::7] = 0
    new_m = torch.where(pm == -FLT_MAX, torch.where(torch.arange(rows) // 4 % 2 == 0, pm, torch.full_like(pm, 3.0)), pm + e)
    pm = torch.where(torch.arange(rows) % 11 == 5, torch.full_like(pm, float("-inf")), pm)
    inf = pm == float("-inf")
    po = torch.where(inf[:, None], torch.zeros_like(po), po)
    pl = torch.where(inf, torch.zeros_like(pl), pl)
    new_m = torch.where(inf, torch.full_like(new_m, 2.0), new_m)
    return po, pm, pl, new_m


def all_cases_variants():
    return {c.variant for c in SIMT_CASES}


def reachable_variants():
    return set(itertools.product(DTYPES, DVWS, MODES))
