"""Variant matrix, schedule rules and exact probes of the streaming decode kernel (perceiver_io_b200/csrc/
pcv_attn_decode.cu), shared by its GPU tests (test_gpu_decode_variants.py) and their CPU companion
(test_decode_variants_cpu.py).  Nothing here needs a GPU.

launch_attn_decode instantiates attn_decode_kernel<T, LPK, NQ, FP8, WIN> (pcv_attn_decode.cu:72-74, :346-363):
  - T: bf16 or fp16 (the dtype of q and out);
  - LPK, lanes per key: the 16-byte chunks of the longer head row rounded up to a power of two, at least 4; e4m3 rows
    (16 channels a chunk, head dims <= 256) take at most 16;
  - NQ: 1 for one query row, 4 for two to four;
  - FP8: e4m3 K / V rows (pcv_attn_decode_fp8, _window_fp8);
  - WIN: the key window read from device memory (pcv_attn_decode_window, _window_fp8).
Each rule below cites the line of pcv_attn_decode.cu (or pcv_api.cu) it restates."""
import itertools

import torch

BF16, FP16 = "bf16", "fp16"
DTYPES = (BF16, FP16)
WARPS = 4                 # kDecWarps (:29)
SMS = 132                 # the H100 SXM's SM count; choose_split also falls back to 132 without a device (:327)
SPLIT_ALIGN = 128         # choose_split: splits on 128-key boundaries (:337)
MAX_SPLITS = 256          # (:335)
MIN_KEYS_PER_CTA = 256    # max_by_keys = M / 256 (:334)
CTAS_PER_SM = 12          # (:333)
ROUTING_FLOOR = 1024      # use_decode: pcv_attn_fwd takes the 16-bit non-window decode only for M >= 1024 (pcv_api.cu:75)
FLT_MAX = torch.finfo(torch.float32).max


def device_sms():
    """The SM count choose_split plans with (:327-329): the current device's when there is one, else the fallback 132."""
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return SMS


# ---- the restated rules ----
def lanes_per_key(dqk, dv, fp8):
    """lanes_per_key (:370-376) and the dispatch of launch_decode (:356-363): lpk <= 4 collapses to 4; e4m3 rows stop at
    16 (`FP8 || lpk == 16`, and 256 e4m3 channels are 16 chunks)."""
    ch = 16 if fp8 else 8
    chunks = (max(dqk, dv) + ch - 1) // ch
    lpk = 1
    while lpk < chunks:
        lpk <<= 1
    return min(max(lpk, 4), 16 if fp8 else 32)


def nq_of(N):
    """launch_decode (:351-354): one query row takes NQ = 1, two to four share NQ = 4."""
    return 1 if N == 1 else 4


def unroll(fp8, nq):
    """kUnroll (:78): e4m3 rows with four query rows take 2 warp steps per block, every other variant 4 (Unroll<NQ>)."""
    return 2 if fp8 and nq > 1 else 4


def geometry(lpk, nq, fp8):
    """(KPW, KPB, warp stride): keys per warp step (:79), per warp block (:80), and the stride between one warp's blocks
    (kStride = kDecWarps * KPB, :206)."""
    kpw = 32 // lpk
    kpb = kpw * unroll(fp8, nq)
    return kpw, kpb, WARPS * kpb


def choose_split(B, H, M, sms=SMS):
    """choose_split (:326-341) -> (nsplit, keys_per_split): ~12 CTAs per SM, at least 256 keys per CTA, at most 256
    splits, on 128-key boundaries."""
    bh = B * H
    want = max(1, (CTAS_PER_SM * sms + bh - 1) // bh)
    want = min(want, max(1, M // MIN_KEYS_PER_CTA), MAX_SPLITS)
    kps = (M + want - 1) // want
    kps = (kps + SPLIT_ALIGN - 1) // SPLIT_ALIGN * SPLIT_ALIGN
    return (M + kps - 1) // kps, kps


def split_ranges(M, nsplit, kps):
    """[kb, ke) of every split of the non-window kernel (:98-99); the last split may be ragged."""
    return [(s * kps, min(M, s * kps + kps)) for s in range(nsplit)]


def window_ranges(win0, win1, M, nsplit):
    """[kb, ke) of every split of the window kernel (:92-96): the window clamped to [max(win0, 0), min(win1, M)), each
    split an equal share of ceil(len / nsplit) keys; a split past the window's end is empty (ke <= kb)."""
    w0, wend = max(win0, 0), min(win1, M)
    share = (max(wend - w0, 0) + nsplit - 1) // nsplit
    return [(w0 + s * share, min(wend, w0 + s * share + share)) for s in range(nsplit)]


def window_clamp(win0, win1, M):
    """(first key, end) of the window after the clamps; the causal mask is right-aligned to `end` (:133)."""
    return max(win0, 0), min(win1, M)


def workspace_bytes(B, H, N, M, dv, sms=SMS):
    """attn_decode_workspace_bytes (:416-423): ws_o, ws_m, ws_l of B*H*nsplit*NQ rows and B*H tickets, 256-aligned."""
    a256 = lambda x: (x + 255) // 256 * 256  # noqa: E731
    nsplit, _ = choose_split(B, H, M, sms)
    rows = B * H * nsplit * nq_of(N)
    return a256(rows * dv * 4) + 2 * a256(rows * 4) + a256(B * H * 4)


def serial_depth(kps, nsplit, lpk, nq, fp8):
    """The longest chain of fp32 roundings and ex2 factors one probability passes through (gpu_util.decode_element_bound):
    the keys and block rescales of one lane group (a lane group reads one key of every KPW, in every 4th block), the
    shuffle tree over the lane groups, the warps, the splits, and the descale, quotient and scale roundings."""
    kpw, kpb, _ = geometry(lpk, nq, fp8)
    keys = -(-kps // (WARPS * kpw))
    blocks = -(-kps // (WARPS * kpb))
    return keys + blocks + (kpw.bit_length() - 1) + WARPS + nsplit + 4


def partition(kb, ke, lpk, nq, fp8):
    """The warp loop (:205-218) and load_block (:149-161) of one split restated: {key: (warp, lane group, block, step)}
    for every key the split reads.  Warp w takes the blocks starting at kb + (w + 4 r) KPB; step u of a block holds keys
    j0 + u KPW + grp, and keys j >= ke are skipped."""
    kpw, kpb, stride = geometry(lpk, nq, fp8)
    owner = {}
    for w in range(WARPS):
        j0, r = kb + w * kpb, 0
        while j0 < ke:
            for u in range(unroll(fp8, nq)):
                for g in range(kpw):
                    j = j0 + u * kpw + g
                    if j < ke:
                        assert j not in owner, f"key {j} read twice: {owner[j]} and {(w, g, r, u)}"
                        owner[j] = (w, g, r, u)
            j0 += stride
            r += 1
    return owner


# ---- the instantiations ----
def variant_of(dt, fp8, win, dqk, dv, N):
    """The (T, LPK, NQ, FP8, WIN) instantiation one call launches."""
    return (dt, lanes_per_key(dqk, dv, fp8), nq_of(N), fp8, win)


def reachable_variants():
    """Every instantiation launch_attn_decode can reach: head dims 8..256 in multiples of 8 (16 for e4m3 rows,
    attn_decode_supported :397-400), 1..4 query rows, every dtype, with and without e4m3 rows and a window."""
    out = set()
    for dt, fp8, win, N in itertools.product(DTYPES, (False, True), (False, True), (1, 2, 3, 4)):
        step = 16 if fp8 else 8
        for dqk, dv in itertools.product(range(step, 257, step), repeat=2):
            out.add(variant_of(dt, fp8, win, dqk, dv, N))
    return out


# Head dims per (row kind, LPK): idle lanes (one chunk on a 4-lane group), dead chunks (dqk != dv both ways) and the
# widest rows.  Every pair has max(dqk, dv) reaching exactly that LPK.
HEAD_DIMS = {
    (False, 4): [(8, 8), (32, 16)],
    (False, 8): [(64, 40), (40, 64)],
    (False, 16): [(128, 72), (72, 128)],
    (False, 32): [(32, 160), (160, 32), (256, 256)],
    (True, 4): [(16, 16), (64, 32)],
    (True, 8): [(128, 80), (80, 128)],
    (True, 16): [(32, 160), (160, 32), (256, 256)],
}


def _matrix():
    cases = []
    for (fp8, lpk), dims in HEAD_DIMS.items():
        for dt, win, nq in itertools.product(DTYPES, (False, True), (1, 4)):
            for i, (dqk, dv) in enumerate(dims):
                N = 1 if nq == 1 else 2 + (i + len(cases)) % 3   # NQ = 4 at N = 2, 3 and 4
                cases.append((dt, fp8, win, dqk, dv, N))
    return cases


#: (dtype, e4m3 rows, window, dqk, dv, N)
VARIANT_CASES = _matrix()


def case_id(case):
    dt, fp8, win, dqk, dv, N = case
    return f"{dt}-{'e4m3' if fp8 else 'k16'}-{'win' if win else 'full'}-qk{dqk}-v{dv}-n{N}"


# ---- named edge shapes: (B, H, M) of the non-window kernel, and the structure check_schedule asserts ----
EDGE_SHAPES = {
    "ragged_one": (2, 2, 1153),         # 4 splits of 384 keys, the last holds exactly 1
    "ragged_mid_step": (2, 2, 1485),    # the last split holds 333 keys: it ends inside a warp block and a warp step
    "one_split": (4, 396, 1024),        # B*H = 12 * 132: one split of 1024 keys
    "middle": (1, 1, 5000),             # 14 splits of 384, the last of 8 keys
    "cap_256": (1, 1, 65536),           # the 256-split cap: 256 splits of 256 keys
}
#: one split for the e4m3 and window entry points, which take any M: fewer than 512 keys
SHORT_SHAPE = (2, 2, 500)


def check_schedule(shape, lpk, nq, fp8, sms=SMS):
    """Assert that EDGE_SHAPES[shape] has, for the variant geometry (lpk, nq, fp8), the structure it is named for.
    Returns a one-line description."""
    B, H, M = EDGE_SHAPES[shape]
    nsplit, kps = choose_split(B, H, M, sms)
    kpw, kpb, _ = geometry(lpk, nq, fp8)
    last = M - (nsplit - 1) * kps
    if shape == "ragged_one":
        assert nsplit > 1 and last == 1, (nsplit, kps, last)
    elif shape == "ragged_mid_step":
        assert nsplit > 1 and last % kpb != 0, (nsplit, kps, last, kpb)
        # some lane group's last step has no key (a step is one key at 32 lanes per key)
        assert kpw == 1 or last % kpw != 0, (last, kpw)
    elif shape == "one_split":
        assert nsplit == 1 and M == ROUTING_FLOOR, (nsplit, M)
    elif shape == "middle":
        assert 1 < nsplit < MAX_SPLITS and last < kps, (nsplit, kps, last)
    elif shape == "cap_256":
        assert nsplit == MAX_SPLITS, nsplit
    else:
        raise KeyError(shape)
    return f"{shape} (B={B}, H={H}, M={M}) LPK {lpk} NQ {nq}: {nsplit} splits of {kps} keys, the last of {last}; KPB {kpb}"


# ---- windows on one arena: (name, (win0, win1)) on CAPACITY rows, B*H = 12, planned at WIN_NSPLIT splits ----
WIN_B, WIN_H, CAPACITY = 3, 4, 3000
WIN_NSPLIT = choose_split(WIN_B, WIN_H, CAPACITY)[0]     # 8
WINDOWS = [
    ("len1", (1000, 1001)),
    ("nsplit_minus_1", (13, 13 + WIN_NSPLIT - 1)),       # one key per split, trailing splits empty
    ("nsplit", (101, 101 + WIN_NSPLIT)),
    ("nsplit_plus_1", (200, 200 + WIN_NSPLIT + 1)),
    ("mid_block", (517, 1518)),                          # shares of 126 keys: boundaries mid warp block; odd begin
    ("diag_at_share", (1001, 1066)),                     # 65 keys: shares of 9, the last of 2 (the diagonals straddle it)
    ("odd_begin", (3, 2000)),
    ("to_capacity", (2001, CAPACITY)),
    ("past_capacity", (2500, CAPACITY + 500)),           # clamped to capacity
    ("negative_begin", (-50, 700)),                      # clamped to 0
    ("shorter_than_n", (2200, 2202)),                    # causal: rows 0 and 1 of N = 4 have no live key
    ("empty", (40, 40)),
    ("negative_length", (50, 30)),
    ("begin_past_capacity", (CAPACITY + 100, CAPACITY + 200)),
]


def check_window(name, win, N=4, lpk=4, nq=4, fp8=False):
    """Assert the structure the window `name` is named for (on the arena of WINDOWS); returns a description."""
    w0, wend = window_clamp(*win, CAPACITY)
    length = wend - w0
    r = window_ranges(*win, CAPACITY, WIN_NSPLIT)
    sizes = [max(ke - kb, 0) for kb, ke in r]
    _kpw, kpb, _ = geometry(lpk, nq, fp8)
    assert sum(sizes) == max(length, 0)
    if name == "len1":
        assert length == 1
    elif name == "nsplit_minus_1":
        assert length == WIN_NSPLIT - 1 and sizes[-1] == 0
    elif name == "nsplit":
        assert length == WIN_NSPLIT and sizes == [1] * WIN_NSPLIT
    elif name == "nsplit_plus_1":
        assert length == WIN_NSPLIT + 1 and 0 in sizes and sizes[0] == 2
    elif name == "mid_block":
        assert sizes[0] % kpb != 0 and w0 % 2 == 1
    elif name == "diag_at_share":
        firsts = {kb for kb, ke in r if ke > kb}
        lasts = {ke - 1 for kb, ke in r if ke > kb}
        diags = {wend - N + i for i in range(N)}
        assert diags & firsts and diags & lasts, (diags, firsts, lasts)
    elif name == "odd_begin":
        assert w0 % 2 == 1
    elif name == "to_capacity":
        assert wend == CAPACITY and win[1] == CAPACITY
    elif name == "past_capacity":
        assert win[1] > CAPACITY and wend == CAPACITY
    elif name == "negative_begin":
        assert win[0] < 0 and w0 == 0
    elif name == "shorter_than_n":
        assert 0 < length < N
    elif name in ("empty", "negative_length", "begin_past_capacity"):
        assert length <= 0 and sum(sizes) == 0
        if name == "begin_past_capacity":
            assert win[0] >= CAPACITY
    else:
        raise KeyError(name)
    return f"window {name} {win} -> [{w0}, {wend}) on {WIN_NSPLIT} splits: shares {sizes}"


# ---- exact expectations (on the device of their tensors) ----
def key_sets(B, N, M, pad, causal, rng=None, m_total=None, m_offset=0, causal_end=None, device="cpu"):
    """(in_range (B, N, M), live (B, N, M)) bool: the keys a row reads and the ones not masked.  `rng` = (k0, kend) of
    a window (default all M keys); the causal mask is right-aligned to `causal_end` (the window's end, :133) or to
    m_total (the non-window kernel; key j of a shard is global key m_offset + j, :177)."""
    j = torch.arange(M, device=device)
    k0, kend = (0, M) if rng is None else rng
    in_range = ((j >= k0) & (j < kend))[None, None, :].expand(B, N, M)
    live = in_range.clone()
    if pad is not None:
        live = live & ~pad.to(device).bool()[:, None, :]
    if causal:
        end = (M if m_total is None else m_total) if causal_end is None else causal_end
        shift = end - N
        live = live & ((m_offset + j)[None, :] <= (torch.arange(N, device=device)[:, None] + shift))[None]
    return in_range, live


def count_state(v, H, in_range, live):
    """(S, L, any_live) of the count probe (q = 0: every live score is exactly 0, every masked one -FLT_MAX): S (B, H, N,
    dv) the fp64 sum of V over a row's live keys, or over every key it reads when none is live (the finite fill), L the
    number of those keys."""
    B, M = v.shape[0], v.shape[1]
    vh = v.double().reshape(B, M, H, -1).transpose(1, 2)                     # (B, H, M, dv)
    any_live = live.any(-1, keepdim=True)
    sel = torch.where(any_live, live, in_range).double()                      # (B, N, M)
    S = torch.einsum("bnm,bhmc->bhnc", sel, vh)
    L = sel.sum(-1)[:, None, :].expand(B, H, -1)
    return S, L, any_live[..., 0][:, None, :].expand(B, H, -1)


def _scaled(v, H, v_scale):
    if v_scale is None:
        return v.double()
    B, M = v.shape[0], v.shape[1]
    return (v.double().reshape(B, M, H, -1) * v_scale.to(v.device).double()[None, None]).reshape(B, M, -1)


def count_expect(v, H, in_range, live, dtype, v_scale=None):
    """The count probe's output bit for bit: RN16(RN32(S / L)), (B, N, H*dv) in `dtype`; a row that reads no key gives 0
    (the window kernel's empty-window guard, :309-311).  S is an integer sum (times the power-of-two v_descale of e4m3
    rows, `v_scale` (H, dv)), exact in fp32 below 2^24, so the one rounding before the output is the fp32 quotient."""
    S, L, _ = count_state(_scaled(v, H, v_scale), H, in_range, live)
    assert S.abs().max().item() < 2 ** 24
    Lf = L.float()[..., None]
    q = torch.where(Lf > 0, S.float() / Lf.clamp_min(1), torch.zeros((), dtype=torch.float32, device=S.device))
    B, _, N, dv = q.shape
    return q.to(dtype).transpose(1, 2).reshape(B, N, H * dv)


def needle_expect(v, H, in_range, live, needle, dtype, v_scale=None):
    """The needle probe's output bit for bit.  `needle` (B, H, N) long: the key whose score is >= 100 (log2 units) above
    every other key's 0 for that row.  Found (the needle is live): l rounds to 1 and the output is RN16(v[needle]).
    Not found (masked, or outside the window): the row is the count probe's."""
    B, M = v.shape[0], v.shape[1]
    N = needle.shape[2]
    dev = v.device
    vh = _scaled(v, H, v_scale).reshape(B, M, H, -1)
    nd = needle.to(dev)
    bi, hi, ni = (torch.arange(s, device=dev) for s in (B, H, N))
    vn = vh[bi[:, None, None], nd, hi[None, :, None]]                         # (B, H, N, dv)
    found = live[bi[:, None, None], ni[None, None, :], nd]                    # (B, H, N)
    base = count_expect(v, H, in_range, live, dtype, v_scale).reshape(B, N, H, -1)
    hit = vn.float().to(dtype).transpose(1, 2)                                # (B, N, H, dv)
    return torch.where(found.transpose(1, 2)[..., None], hit, base).reshape(B, N, -1)


def edge_keys(ranges, lpk, nq, fp8, extra=(), M=None, limit=60):
    """Keys under test for the count probe's sparse V: the first and last key of every split (or window share; of
    seven of them past eight) and of every warp's first and last block in the first and last non-empty split, plus
    `extra` (the diagonals, the keys next to a window).  Capped at `limit` so that S stays below 64 codes: then a change
    of S by one code moves S / L by more than a bf16 ulp.  Keys outside [0, M) are dropped."""
    _kpw, kpb, stride = geometry(lpk, nq, fp8)
    live_r = [(kb, ke) for kb, ke in ranges if ke > kb]
    marks = set(extra)
    picks = live_r if len(live_r) <= 8 else live_r[:3] + live_r[len(live_r) // 2:len(live_r) // 2 + 1] + live_r[-3:]
    for kb, ke in picks:
        marks |= {kb, ke - 1}
    for kb, ke in ({live_r[0], live_r[-1]} if live_r else ()):
        for w in range(WARPS):
            j0 = kb + w * kpb
            jl = j0 + max(0, (ke - 1 - j0) // stride) * stride
            for s in (j0, jl):
                if s < ke:
                    marks |= {s, min(s + kpb, ke) - 1}
    marks = sorted(m for m in marks if m >= 0 and (M is None or m < M))
    assert len(marks) <= limit, len(marks)
    return marks


# ---- probe operands (on `device`) ----
def v_descale(H, dv, device="cpu"):
    """The e4m3 probes' v_descale (H, dv): powers of two that differ from one channel to the next."""
    return (2.0 ** ((torch.arange(dv, device=device) % 5) - 2).float())[None].expand(H, dv).contiguous()


def _as(x, fp8, dtype):
    return x.to(torch.float8_e4m3fn) if fp8 else x.to(dtype)


def count_operands(B, Bq, N, M, H, dqk, dv, marks, pad, fp8, dtype, seed, device="cpu"):
    """(q, k, v) of the count probe: q = 0; K random (integer e4m3 codes); V = 2^(c % 3) at the keys under test, 8 at
    padded keys, else 0 (codes with |code| <= 16 are exact in e4m3)."""
    g = torch.Generator(device=device).manual_seed(seed)
    q = torch.zeros(Bq, N, H * dqk, device=device).to(dtype)
    k = (torch.randint(-8, 9, (B, M, H * dqk), generator=g, device=device).float() if fp8
         else torch.randn(B, M, H * dqk, generator=g, device=device))
    v = torch.zeros(B, M, H, dv, device=device)
    v[:, list(marks)] = (2.0 ** (torch.arange(dv, device=device) % 3)).float()
    v = torch.where(pad.to(device)[:, :, None, None], torch.full_like(v, 8.0), v)
    return q, _as(k, fp8, dtype), _as(v.reshape(B, M, H * dv), fp8, dtype)


NEEDLE_SCALE = 0.5   # a needle scores 16 * 16 * NEEDLE_SCALE * log2(e) = 184.7 (k_descale 1)


def needle_channels(N, dqk):
    """c_n: the one channel query row n sees; the last channel for row 0, spread over the chunks for the others."""
    return [dqk - 1 - n * (dqk // N) for n in range(N)]


def needle_operands(B, Bq, N, M, H, dqk, dv, needle, fp8, dtype, seed, device="cpu"):
    """(q, k, v) of the needle probe: q[n, h, c_n] = 16, K[:, :, h, c_n] = 0 but 16 at the needle of (b, h, n), V random
    integers in [-4, 4] and +-(9..14) at the needles."""
    g = torch.Generator(device=device).manual_seed(seed)
    cs = torch.tensor(needle_channels(N, dqk), device=device)
    q = torch.zeros(Bq, N, H, dqk, device=device)
    k = (torch.randint(-8, 9, (B, M, H, dqk), generator=g, device=device).float() if fp8
         else torch.randn(B, M, H, dqk, generator=g, device=device))
    v = torch.randint(-4, 5, (B, M, H, dv), generator=g, device=device).float()
    ni = torch.arange(N, device=device)
    q[:, ni, :, cs] = 16.0
    k[:, :, :, cs] = 0.0
    nd = needle.to(device)
    bi = torch.arange(B, device=device)[:, None, None].expand(B, H, N)
    hi = torch.arange(H, device=device)[None, :, None].expand(B, H, N)
    k[bi, nd, hi, cs[None, None, :].expand(B, H, N)] = 16.0
    mag = (9 + (ni[None, None, :] + hi + bi) % 6).float() * (1 - 2 * (nd % 2)).float()
    v[bi, nd, hi] = mag[..., None].expand(B, H, N, dv)
    return (q.reshape(Bq, N, -1).to(dtype), _as(k.reshape(B, M, -1), fp8, dtype), _as(v.reshape(B, M, -1), fp8, dtype))


def needle_candidates(N, k0, kend, ranges, pad, b, causal, lpk, nq, fp8):
    """Keys a needle of batch row b is placed on: the diagonal and the key past it (causal), the first and last padded
    key, split / share and warp-block edges, the first and the last key."""
    cand = [k0, kend - 1]
    if causal:
        for n in range(N):
            cand += [kend - N + n, kend - N + n + 1]
    padded = pad[b, k0:kend].nonzero()
    if padded.numel():
        cand += [k0 + int(padded[0]), k0 + int(padded[-1])]
    cand += edge_keys(ranges, lpk, nq, fp8)
    return sorted({c for c in cand if k0 <= c < kend})


def needles(B, H, N, cands, r):
    """(B, H, N) needle keys of round r: batch row b walks its own candidate list cands[b], H * N keys a round, so the
    first needle_rounds(cands, H, N) rounds put a needle on every candidate of every batch row."""
    out = torch.zeros(B, H, N, dtype=torch.long)
    for b, h, n in itertools.product(range(B), range(H), range(N)):
        c = cands[b]
        out[b, h, n] = c[(r * H * N + h * N + n) % len(c)]
    return out


def needle_rounds(cands, H, N):
    """Rounds of `needles` that cover every candidate of every batch row."""
    return max(-(-len(c) // (H * N)) for c in cands)
