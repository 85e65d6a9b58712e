// pcv_attn_cached.cu — attention of 1 to 64 bf16 / fp16 query rows over a KV cache on the Hopper tensor cores (sm_90a),
// in two forms of one kernel, attn_cached_kernel<BF16, FP8, WIN, NVB>:
//   - whole cache (WIN false, pcv_attn_cached_fp8): the e4m3 keys [0, M).  A cached step that appends several tokens at
//     once (a prompt fed in chunks, a run of new tokens, draft tokens verified in one call) reads the e4m3 codes once
//     and never materialises a 16-bit copy of the cache.
//   - window (WIN true, pcv_attn_cached_window (_fp8)): batch row b's window [w[0], w[1]), w = bounds +
//     b * bounds_stride_b, of an arena of bf16 / fp16 rows of q's type or e4m3 codes, read from device memory when the
//     kernel runs and clamped to [0, capacity), with an optional causal band: a k-token step of a graph-replayed decode
//     loop sees for every one of its tokens exactly the keys the one-token loop gives that token.
//
//   grid = B * nsplit * H CTAs, head index fastest (as attn_decode_kernel); CTA = one (b, h) and a contiguous range of
//   64-key tiles.  nsplit is planned on the host from M (the arena's capacity for a window), so for a window the grid
//   and the workspace are fixed for the life of a graph.  The whole cache's splits take tiles_per_split tiles each; a
//   window's tiles start at its begin (not tile-aligned) and every split takes an equal share of them.  256 threads:
//     warpgroup 1, the loader: e4m3 K and V rows are loaded with 16-byte loads (the next unit of 32 or 64 keys in
//       flight while one is converted), every code is converted to q's 16-bit type and the tile is stored into a ring
//       of converted stages in the SWIZZLE_128B layout that TMA writes for the forward kernel (K K-major, V MN-major,
//       64-channel boxes of 64 keys), so the pcv_sm90.cuh wgmma wrappers read it as they are.  16-bit rows go straight
//       into the stages with 16-byte cp.async (keys past the window's end and the channel tail of a k16 step are
//       zero-filled).  full / empty mbarriers guard the ring.
//     warpgroup 0, the consumer: one m64 query tile in shared memory (rows N .. 63 are zero and dropped), S = Q K^T
//       (m64n64k16, SS), the online softmax in registers, O += P V (m64n64k16, P from registers) per 64-channel box.
//   Split states go to the workspace; the last CTA of every (b, h) (atomic ticket) merges them in split order and
//   writes the output: one launch, bitwise reproducible.
//   The raw e4m3 tile is staged in registers, not in shared memory by a TMA producer warp: the converter has to read
//   every code into registers anyway, and the shared memory of a raw ring (16 KB a stage at head dims 128 / 128) goes to
//   converted stages instead.  This is a design choice from arithmetic, not a measured one.
//
// Masks (include/pcv_attn.h).  The pad mask is (B, M) bytes, indexed by the absolute key (arena) row.  Query i sits at
// row r_i = end - N + i, end = M for the whole cache.
//   - no band: the causal mask is right-aligned (query i sees keys j <= r_i); padded and causally masked keys take the
//     finite fill (a fully masked row is the uniform average of the keys);
//   - band W > 0 (window, causal only): query i sees exactly the keys [r_i + 1 - W, r_i] of the window.  Every other
//     key is excluded: it contributes nothing, like a key outside the window, and takes no fill.  Padded keys inside the
//     band take the fill, so a row whose band is all padding is the uniform average over its band.
//   In a window, a tile, or a whole split, can hold no key of a row: its running maximum stays -inf, the rescale of an
//   empty state is skipped, and an empty split state (m = -inf, l = 0) merges with weight 0.  A window of length <= 0
//   writes zeros.  These guards are compiled into the window kernels only: every whole-cache tile and split holds a
//   live or filled key of every row.
//
// Arithmetic contract (the tests derive their element-wise gate from it):
//   - 16-bit K / V enter the MMA as stored; e4m3 codes exactly: every e4m3 value is an fp16 and a bf16 value;
//     cvt.rn.f16x2.e4m3x2 gives fp16, bf16 goes through f32 (exact);
//   - q enters unrounded, in its own dtype; c = scale * log2(e) (times k_descale[h] for e4m3 rows) multiplies the fp32
//     score s once: the row maximum m is taken over round(s * c), and p = 2^(fma(s, c, -m)) (ex2.approx);
//   - the online softmax runs in fp32 in the log2 domain; P is rounded to q's 16-bit type before P V (as in
//     attn_fwd_kernel) while the denominators sum the fp32 p; for e4m3 rows v_descale[h, c] multiplies the fp32
//     accumulator once, before the merge (as in attn_decode_kernel).
//   With the window [0, capacity) and no band, the e4m3 window kernel computes what the whole-cache kernel computes,
//   bit for bit.
#include "pcv_common.cuh"
#include "pcv_sm90.cuh"

#include <algorithm>
#include <type_traits>

namespace pcv {
namespace {

using namespace sm90;

constexpr int kKeys = 64;               // keys per tile
constexpr int kMaxRows = 64;            // query rows: one m64 tile
constexpr int kBox = 64 * 128;          // one box: 64 rows x 64 16-bit channels, SWIZZLE_128B
constexpr int kThreads = 256;           // consumer warpgroup + loader warpgroup
constexpr int kMaxStages = 4;
constexpr int kSmemLimit = 227 * 1024 - 1024;  // dynamic bytes: the per-block limit less room for the static s_last
constexpr int kPairBudget = 110 * 1024; // per CTA when two share an SM (228 KB per SM, 1 KB reserved per CTA)

struct CachedParams {
  pcv_attn_params a;
  pcv_decode_fp8 f;             // e4m3 rows only
  const int32_t* win;           // window: device [begin, end) of batch row 0
  int win_stride_b;             // window: int32s between the windows of batch rows b and b + 1 (0: one shared window)
  int band;                     // window: > 0: query i sees keys [r_i + 1 - band, r_i] only
  int nsplit, tiles_per_split;  // whole cache: split s covers key tiles [s * tiles_per_split, min(+tiles_per_split, tiles))
  int nkb;                      // 64-channel boxes of a q / K row
  int stages;
  float* ws_o;                  // [B*H][nsplit][N][dv]
  float* ws_m;                  // [B*H][nsplit][N]
  float* ws_l;                  // [B*H][nsplit][N]
  unsigned int* tickets;        // [B*H], zero on entry; the last CTA of a (b, h) resets its ticket
};

// 16 e4m3 codes -> 16 16-bit values (two 16-byte chunks, lowest channel first), exact
template <bool BF16>
__device__ __forceinline__ void convert16(const uint4& u, uint4& lo, uint4& hi) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
  uint32_t h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint16_t pair = (uint16_t)(w[i >> 1] >> (16 * (i & 1)));
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h[i]) : "h"(pair));
    if constexpr (BF16) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h[i]));
      h[i] = pack2(f.x, f.y, true);
    }
  }
  lo = make_uint4(h[0], h[1], h[2], h[3]);
  hi = make_uint4(h[4], h[5], h[6], h[7]);
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// byte offset of 16-byte chunk `ch` (8 16-bit channels) of row r in a SWIZZLE_128B box
__device__ __forceinline__ uint32_t swz(int r, int ch) { return (uint32_t)(r * 128 + ((ch ^ (r & 7)) << 4)); }

// 16 bytes global -> shared, zero-filled when !live (nothing is read then)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool live) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(live ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// FP8: e4m3 rows, else rows of q's 16-bit type.  WIN: the window read from device memory, else the whole cache.  NVB:
// 64-channel boxes of a V row (ceil(dv / 64)).  Dynamic shared memory: [Q: nkb boxes][stage: nkb K boxes, NVB V boxes]
// x stages, then the barriers.  Watchdog sites: 61 / 62 for the whole cache, 63 / 64 for a window.
template <bool BF16, bool FP8, bool WIN, int NVB>
__global__ void __launch_bounds__(kThreads, NVB == 1 ? 2 : 1) attn_cached_kernel(const CachedParams p) {
  static_assert(WIN || FP8, "the whole-cache kernel reads e4m3 rows only");
  using T = typename std::conditional<BF16, __nv_bfloat16, __half>::type;
  const pcv_attn_params& a = p.a;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_u32 = smem_u32(smem_raw);
  const uint32_t base = (raw_u32 + 1023u) & ~1023u;
  const int nkb = p.nkb, S = p.stages;
  const uint32_t q_base = base;
  const uint32_t ring_base = base + nkb * kBox;
  const uint32_t stage_bytes = (nkb + NVB) * kBox;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + (ring_base - raw_u32) + S * stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kMaxStages;

  // blockIdx.x = (b * nsplit + split) * H + h
  const int h = blockIdx.x % a.H;
  const int split = (blockIdx.x / a.H) % p.nsplit;
  const int b = blockIdx.x / (a.H * p.nsplit);
  const int bh = b * a.H + h;
  // the keys [w0, wend); this split takes the tiles [t0, t1), tile t = keys w0 + 64 t .. (< wend)
  int w0 = 0, wlim = 0, t0, t1;
  if constexpr (WIN) {  // the window clamped to the arena
    const int32_t* win = p.win + (int64_t)b * p.win_stride_b;
    w0 = max(win[0], 0);
    wlim = min(win[1], a.M);
    const int ntiles = (max(wlim - w0, 0) + kKeys - 1) / kKeys;
    const int tps = (ntiles + p.nsplit - 1) / p.nsplit;
    t0 = min(ntiles, split * tps);
    t1 = min(ntiles, t0 + tps);
  } else {
    const int tiles = (a.M + kKeys - 1) / kKeys;
    t0 = split * p.tiles_per_split;
    t1 = min(tiles, t0 + p.tiles_per_split);
  }
  // the whole cache's end is M, read from the kernel parameters at each use: a register copy of it compiles the
  // converter's load loop to a different, untimed schedule
  const int& wend = WIN ? wlim : a.M;
  constexpr int kFree = WIN ? 63 : 61, kReady = WIN ? 64 : 62;  // watchdog sites

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 4);   // one arrive per loader warp
      mbar_init(&empty[s], 4);  // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x >= 128) {
    // ---- loader warpgroup ------------------------------------------------------------------------------------
    const int ct = threadIdx.x - 128;
    if constexpr (FP8) {
      const int kch = a.dqk / 16, vch = a.dv / 16;  // 16-byte e4m3 chunks of a K / V row
      const uint8_t* kp = reinterpret_cast<const uint8_t*>(a.k) + (int64_t)b * a.k_stride_b + (int64_t)h * a.k_stride_h;
      const uint8_t* vp = reinterpret_cast<const uint8_t*>(a.v) + (int64_t)b * a.v_stride_b + (int64_t)h * a.v_stride_h;
      // The tile is converted in units of U keys, two units in registers: one is stored while the next one's loads are
      // in flight.  Two CTAs per SM (NVB == 1) take half tiles to stay within 128 registers; one CTA per SM whole tiles,
      // so that as many bytes are in flight per SM.
      constexpr int U = NVB == 1 ? 32 : 64, P = kKeys / U;  // keys per unit, units per tile
      constexpr int KU = U / 8, VU = U * NVB / 32;          // chunks per thread of a unit: K U * 16 / 128, V U * 4 NVB / 128
      // chunk u of this thread in unit z (tile z / P, part z % P): key U (z % P) + idx / ch, chunk idx % ch, idx = ct + 128 u
      auto load = [&](uint4 (&kr)[KU], uint4 (&vr)[VU], int z) {
        const int j0 = w0 + (z / P) * kKeys + U * (z % P);
#pragma unroll
        for (int u = 0; u < KU; ++u) {
          const int idx = ct + 128 * u, key = idx / kch;
          kr[u] = make_uint4(0, 0, 0, 0);
          if (idx < U * kch && j0 + key < wend)
            kr[u] = __ldcs(reinterpret_cast<const uint4*>(kp + (int64_t)(j0 + key) * a.k_stride_m + (idx - key * kch) * 16));
        }
#pragma unroll
        for (int u = 0; u < VU; ++u) {
          const int idx = ct + 128 * u, key = idx / vch;
          vr[u] = make_uint4(0, 0, 0, 0);
          if (idx < U * vch && j0 + key < wend)
            vr[u] = __ldcs(reinterpret_cast<const uint4*>(vp + (int64_t)(j0 + key) * a.v_stride_m + (idx - key * vch) * 16));
        }
      };
      auto store = [&](const uint4 (&kr)[KU], const uint4 (&vr)[VU], uint32_t st, int part) {
#pragma unroll
        for (int u = 0; u < KU; ++u) {
          const int idx = ct + 128 * u, key = idx / kch;
          if (idx < U * kch) {
            const int ci = idx - key * kch, r = U * part + key;
            const uint32_t box = st + (ci >> 2) * kBox;
            uint4 lo, hi;
            convert16<BF16>(kr[u], lo, hi);
            st_shared_v4(box + swz(r, 2 * (ci & 3)), lo);
            st_shared_v4(box + swz(r, 2 * (ci & 3) + 1), hi);
          }
        }
#pragma unroll
        for (int u = 0; u < VU; ++u) {
          const int idx = ct + 128 * u, key = idx / vch;
          if (idx < U * vch) {
            const int ci = idx - key * vch, r = U * part + key;
            const uint32_t box = st + (nkb + (ci >> 2)) * kBox;
            uint4 lo, hi;
            convert16<BF16>(vr[u], lo, hi);
            st_shared_v4(box + swz(r, 2 * (ci & 3)), lo);
            st_shared_v4(box + swz(r, 2 * (ci & 3) + 1), hi);
          }
        }
      };
      // unit z: the first part of a tile waits for its stage, the last one publishes it
      auto put = [&](const uint4 (&kr)[KU], const uint4 (&vr)[VU], int z) {
        const int i = z / P - t0, slot = i % S, part = z % P;
        const uint32_t st = ring_base + slot * stage_bytes;
        if (part == 0) mbar_wait(&empty[slot], ((i / S) & 1) ^ 1, kFree);
        store(kr, vr, st, part);
        if (part == P - 1) {
          fence_proxy_async_smem();  // the generic-proxy stores, before the wgmma (async proxy) reads them
          warp_arrive(&full[slot]);
        }
      };
      uint4 ka[KU], va[VU], kb[KU], vb[VU];
      const int z1 = t1 * P;
      if (!WIN || t0 < t1) load(ka, va, t0 * P);  // a whole-cache split is never empty
      for (int z = t0 * P; z < z1; z += 2) {
        if (z + 1 < z1) load(kb, vb, z + 1);
        put(ka, va, z);
        if (z + 2 < z1) load(ka, va, z + 2);
        if (z + 1 < z1) put(kb, vb, z + 1);
      }
    } else {
      // 16-byte chunks of a K row in shared memory (the tail of the last k16 step zero-filled) and of a V row; V
      // channels past dv in the last box only feed output channels that are dropped
      const int kc = (a.dqk + 15) / 16 * 2, vc = a.dv / 8;
      const int nk = kKeys * kc, nall = kKeys * (kc + vc);
      const T* kp = reinterpret_cast<const T*>(a.k) + (int64_t)b * a.k_stride_b + (int64_t)h * a.k_stride_h;
      const T* vp = reinterpret_cast<const T*>(a.v) + (int64_t)b * a.v_stride_b + (int64_t)h * a.v_stride_h;
      // one tile's cp.async group stays in flight while the next one is issued (stages >= 2: the slot of tile i was
      // released by the consumer before it waits for tile i - 1)
      for (int t = t0; t < t1; ++t) {
        const int i = t - t0, slot = i % S;
        const uint32_t st = ring_base + slot * stage_bytes;
        mbar_wait(&empty[slot], ((i / S) & 1) ^ 1, kFree);
        const int j0 = w0 + t * kKeys;
        for (int idx = ct; idx < nall; idx += 128) {
          const bool isk = idx < nk;
          const int e = isk ? idx : idx - nk, cpr = isk ? kc : vc;
          const int key = e / cpr, ch = e - key * cpr;
          const int j = j0 + key;
          const bool live = j < wend && 8 * ch < (isk ? a.dqk : a.dv);
          const T* src = isk ? kp + (live ? (int64_t)j * a.k_stride_m + 8 * ch : 0)
                             : vp + (live ? (int64_t)j * a.v_stride_m + 8 * ch : 0);
          cp_async16(st + ((isk ? 0 : nkb) + (ch >> 3)) * kBox + swz(key, ch & 7), src, live);
        }
        cp_async_commit();
        if (i > 0) {
          cp_async_wait<1>();
          fence_proxy_async_smem();
          warp_arrive(&full[(i - 1) % S]);
        }
      }
      if (t1 > t0) {
        cp_async_wait<0>();
        fence_proxy_async_smem();
        warp_arrive(&full[(t1 - t0 - 1) % S]);
      }
    }
  } else {
    // ---- consumer warpgroup ----------------------------------------------------------------------------------
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, cq = 2 * (lane & 3);
    const int rloc = 16 * w + (lane >> 2);  // this thread's rows: rloc and rloc + 8
    const int kw = (a.dqk + 15) / 16;  // a window's k16 steps: head dims are multiples of 8, the last step's tail is zero
    {  // q -> shared memory, rows N .. 63 (and in a window the channel tail of the last k16 step) zero
      const int nq8 = a.dqk / 8, qc = WIN ? 2 * kw : nq8;  // 16-byte chunks of a q row: in memory, in shared memory
      const T* qp = reinterpret_cast<const T*>(a.q) + (a.q_stride_b ? (int64_t)b * a.q_stride_b : 0) + (int64_t)h * a.q_stride_h;
      for (int idx = threadIdx.x; idx < kMaxRows * qc; idx += 128) {
        const int r = idx / qc, c8 = idx - (WIN ? r * 2 * kw : r * nq8);
        uint4 x = make_uint4(0, 0, 0, 0);
        if (r < a.N && (!WIN || c8 < nq8)) x = *reinterpret_cast<const uint4*>(qp + (int64_t)r * a.q_stride_n + 8 * c8);
        st_shared_v4(q_base + (c8 >> 3) * kBox + swz(r, c8 & 7), x);
      }
      fence_proxy_async_smem();
      named_bar_sync<1, 128>();
    }
    const int ksteps = WIN ? kw : a.dqk / 16;  // k16 steps of a q / K row
    float c = a.scale * kLog2e;  // fp32 score -> log2 domain
    if constexpr (FP8) c = a.scale * kLog2e * p.f.k_descale[h];
    const int cshift = wend - a.N;  // query n sits at row n + cshift: key j masked for it iff j > n + cshift
    const int band = WIN ? p.band : 0;
    const uint8_t* pad = a.pad_mask ? a.pad_mask + (int64_t)b * a.pad_stride_b : nullptr;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float o[NVB][32];
#pragma unroll
    for (int v = 0; v < NVB; ++v)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[v][i] = 0.f;

    for (int t = t0; t < t1; ++t) {
      const int i = t - t0, slot = i % S;
      const uint32_t st = ring_base + slot * stage_bytes;
      mbar_wait(&full[slot], (i / S) & 1, kReady);
      float s[32];
      wgmma_fence();
      for (int kk = 0; kk < ksteps; ++kk)
        wgmma_ss<64, BF16>(s, make_desc(q_base + (kk >> 2) * kBox + (kk & 3) * 32),
                           make_desc(st + (kk >> 2) * kBox + (kk & 3) * 32), kk != 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);

      // scores -> probabilities: element 4 g + e is row rloc + 8 (e >> 1), key j0 + 8 g + cq + (e & 1)
      const int j0 = w0 + t * kKeys;
      uint32_t live = 0, filled = 0;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int g = 0; g < 8; ++g)
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
          const int j = j0 + 8 * g + cq + e2;
          if (j >= wend) continue;
          const bool padded = pad != nullptr && pad[j] != 0;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int e = 4 * g + 2 * r + e2;
            const int row = rloc + 8 * r + cshift;
            if (band > 0 && (j > row || j <= row - band)) continue;  // outside the band: excluded
            if (padded || (a.causal && j > row)) {
              filled |= 1u << e;
              mx[r] = fmaxf(mx[r], kMaskedScore);
            } else {
              live |= 1u << e;
              mx[r] = fmaxf(mx[r], s[e] * c);
            }
          }
        }
      float alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float mn = fmaxf(m_run[r], mx[r]);
        alpha[r] = WIN && mn == -INFINITY ? 1.f : ex2(m_run[r] - mn);  // no key of this row yet: nothing to rescale
        m_run[r] = mn;
        l_run[r] *= alpha[r];
      }
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int r = (e >> 1) & 1;
        const float pe = ((live >> e) & 1u) ? ex2(fmaf(s[e], c, -m_run[r]))
                         : ((filled >> e) & 1u) ? ex2(kMaskedScore - m_run[r]) : 0.f;
        l_run[r] += pe;
        s[e] = pe;
      }
#pragma unroll
      for (int v = 0; v < NVB; ++v)
#pragma unroll
        for (int e = 0; e < 32; ++e) o[v][e] *= alpha[(e >> 1) & 1];
      uint32_t pa[4][4];
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        pa[g >> 1][(g & 1) * 2 + 0] = pack2(s[4 * g + 0], s[4 * g + 1], BF16);
        pa[g >> 1][(g & 1) * 2 + 1] = pack2(s[4 * g + 2], s[4 * g + 3], BF16);
      }
      wgmma_fence();
#pragma unroll
      for (int v = 0; v < NVB; ++v)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_rs<64, BF16>(o[v], pa[kk], make_desc(st + (nkb + v) * kBox + kk * 2048));
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int v = 0; v < NVB; ++v) fence_regs(o[v]);
      warp_arrive(&empty[slot]);
    }

    // this split's state -> workspace (an empty window split writes m = -inf, l = 0, o = 0)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float* vd = FP8 ? p.f.v_descale + (int64_t)h * a.dv : nullptr;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int n = rloc + 8 * r;
      if (n >= a.N) continue;
      const int64_t row = ((int64_t)bh * p.nsplit + split) * a.N + n;
#pragma unroll
      for (int v = 0; v < NVB; ++v)
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const int ch = 64 * v + 8 * g + cq;  // dv is a multiple of 8: ch and ch + 1 are both in or both out
          if (ch < a.dv) {
            float2 x = make_float2(o[v][4 * g + 2 * r], o[v][4 * g + 2 * r + 1]);
            if constexpr (FP8) x = make_float2(x.x * vd[ch], x.y * vd[ch + 1]);
            *reinterpret_cast<float2*>(p.ws_o + row * a.dv + ch) = x;
          }
        }
      if ((lane & 3) == 0) {
        p.ws_m[row] = m_run[r];
        p.ws_l[row] = l_run[r];
      }
    }
  }

  // ---- the last CTA of this (b, h) merges the splits in split order ------------------------------------------------
  __shared__ unsigned int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int tk = atomicAdd(p.tickets + bh, 1u);
    s_last = (tk == (unsigned int)p.nsplit - 1) ? 1u : 0u;
    if (s_last) p.tickets[bh] = 0u;  // ready for the next launch on this workspace
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int idx = threadIdx.x; idx < a.N * a.dv; idx += kThreads) {
    const int n = idx / a.dv, ch = idx - n * a.dv;
    const int64_t sb = (int64_t)bh * p.nsplit * a.N + n;
    float mm = -INFINITY;
    for (int sp = 0; sp < p.nsplit; ++sp) mm = fmaxf(mm, __ldcg(p.ws_m + sb + (int64_t)sp * a.N));
    float ov = 0.f, ll = 0.f;
    for (int sp = 0; sp < p.nsplit; ++sp) {
      const float ms = __ldcg(p.ws_m + sb + (int64_t)sp * a.N);
      const float wt = WIN && ms == -INFINITY ? 0.f : exp2f(ms - mm);  // an empty split state has weight 0
      ov = fmaf(__ldcg(p.ws_o + (sb + (int64_t)sp * a.N) * a.dv + ch), wt, ov);
      ll = fmaf(__ldcg(p.ws_l + sb + (int64_t)sp * a.N), wt, ll);
    }
    T* out = reinterpret_cast<T*>(a.out) + (int64_t)b * a.o_stride_b + (int64_t)n * a.o_stride_n + (int64_t)h * a.o_stride_h;
    out[ch] = Elem<T>::from_f(!WIN || ll > 0.f ? ov / ll : 0.f);  // an empty window writes zeros
  }
}

int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

struct CachedPlan {
  int nkb, nvb;
  int ctas_per_sm;      // 2 when two CTAs fit (dv <= 64, dqk <= 192: registers and shared memory), else 1
  int stages;           // >= 2 for every head dim up to 256
  int smem;             // dynamic shared memory bytes
  int nsplit, tiles_per_split;  // tiles_per_split: the whole cache's split; a window splits its own tiles
};

// About two waves of resident CTAs over all (b, h), at least 4 tiles (256 keys) of M (a window: of the arena) per
// split, at most 256 splits.
CachedPlan plan_cached(const pcv_attn_params& a, int sms) {
  CachedPlan pl;
  pl.nkb = (a.dqk + 63) / 64;
  pl.nvb = (a.dv + 63) / 64;
  pl.ctas_per_sm = (pl.nvb == 1 && pl.nkb <= 3) ? 2 : 1;
  const int budget = pl.ctas_per_sm == 2 ? kPairBudget : kSmemLimit;
  const int fixed = pl.nkb * kBox + 1024 + 2 * kMaxStages * 8;  // q, alignment slack, barriers
  pl.stages = std::min(kMaxStages, (budget - fixed) / ((pl.nkb + pl.nvb) * kBox));
  pl.smem = fixed + pl.stages * (pl.nkb + pl.nvb) * kBox;
  const int64_t tiles = (a.M + kKeys - 1) / kKeys;
  const int64_t bh = (int64_t)a.B * a.H;
  int64_t want = std::max<int64_t>(1, (2LL * pl.ctas_per_sm * sms + bh - 1) / bh);
  want = std::min<int64_t>(std::min<int64_t>(want, std::max<int64_t>(1, tiles / 4)), 256);
  const int64_t tps = (tiles + want - 1) / want;
  pl.tiles_per_split = (int)tps;
  pl.nsplit = (int)((tiles + tps - 1) / tps);
  return pl;
}

size_t align256(size_t x) { return (x + 255) / 256 * 256; }

size_t workspace_of(const pcv_attn_params& a, const CachedPlan& pl, size_t* off_m, size_t* off_l, size_t* off_t) {
  const size_t rows = (size_t)a.B * a.H * pl.nsplit * a.N;
  *off_m = align256(rows * a.dv * 4);
  *off_l = *off_m + align256(rows * 4);
  *off_t = *off_l + align256(rows * 4);
  return *off_t + align256((size_t)a.B * a.H * 4);
}

}  // namespace

bool attn_cached_supported(const pcv_attn_params& a, const pcv_decode_fp8* f, const pcv_dev_rows* rows, int band,
                           const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (rows != nullptr) {
    if (rows->bounds == nullptr) return fail("rows->bounds is NULL");
    if (rows->capacity < 1) return fail("rows->capacity must be >= 1");
    if (rows->capacity != a.M) return fail("M must equal rows->capacity (k / v / pad_mask point at arena row 0)");
    if (rows->bounds_stride_b < 0) return fail("rows->bounds_stride_b must be >= 0");
  } else if (f == nullptr || band != 0) {
    return fail("the whole-cache attention takes e4m3 rows and no band");
  }
  if (a.dtype != PCV_BF16 && a.dtype != PCV_F16)
    return fail(f != nullptr ? "dtype (of q and out) must be bf16 or fp16"
                             : "dtype (of q, the K / V arenas and out) must be bf16 or fp16");
  if (a.impl != PCV_IMPL_AUTO) return fail("impl must be AUTO");
  if (a.N > kMaxRows) return fail("more than 64 query rows");
  if (band < 0) return fail("band must be >= 0");
  if (band > 0 && !a.causal) return fail("a band needs the causal mask");
  if (a.write_partial)
    return fail(rows != nullptr ? "the window attention writes the normalised output only (no write_partial)"
                                : "the cached e4m3 attention writes the normalised output only (no write_partial)");
  if (a.m_total != a.M || a.m_offset != 0)
    return fail(rows != nullptr ? "the window attention takes no key shard (m_total != M or m_offset != 0)"
                                : "the cached e4m3 attention takes no key shard (m_total != M or m_offset != 0)");
  const int kv = f != nullptr ? 16 : 8;  // K / V elements per 16-byte chunk
  if ((a.dqk % kv) || (a.dv % kv))
    return fail(f != nullptr ? "head dims must be multiples of 16" : "head dims must be multiples of 8");
  if (a.dqk > 256 || a.dv > 256) return fail("head dim > 256");
  if (f != nullptr && (f->k_descale == nullptr || f->v_descale == nullptr)) return fail("k_descale / v_descale are NULL");
  if (!al16(a.q) || !al16(a.k) || !al16(a.v)) return fail("q/k/v must be 16-byte aligned");
  if ((a.q_stride_n % 8) || (a.q_stride_h % 8) || (a.q_stride_b % 8))
    return fail("q strides must be multiples of 8 elements");
  if ((a.k_stride_m % kv) || (a.v_stride_m % kv) || (a.k_stride_h % kv) || (a.v_stride_h % kv) ||
      (a.k_stride_b % kv) || (a.v_stride_b % kv))
    return fail(f != nullptr ? "e4m3 k/v strides must be multiples of 16 elements"
                             : "k/v strides must be multiples of 8 elements");
  return true;
}

int attn_cached_workspace_bytes(const pcv_attn_params& a, size_t* bytes) {
  size_t om, ol, ot;
  *bytes = workspace_of(a, plan_cached(a, sm_count()), &om, &ol, &ot);
  return PCV_OK;
}

int launch_attn_cached(const pcv_attn_params& a, const pcv_decode_fp8* f, const pcv_dev_rows* rows, int band,
                       cudaStream_t stream) {
  const char* what = rows != nullptr ? "window attention" : "cached e4m3 attention";
  const CachedPlan pl = plan_cached(a, sm_count());
  size_t om, ol, ot;
  const size_t need = workspace_of(a, pl, &om, &ol, &ot);
  PCV_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= need, PCV_ERR_WORKSPACE,
              "%s: workspace of %zu bytes required, %zu given", what, need, a.workspace_bytes);
  if (const char* dp = device_problem()) {
    set_error("%s: %s", what, dp);
    return PCV_ERR_UNSUPPORTED;
  }
  CachedParams p{};
  p.a = a;
  if (f != nullptr) p.f = *f;
  if (rows != nullptr) {
    p.win = rows->bounds;
    p.win_stride_b = rows->bounds_stride_b;
    p.band = band;
  }
  p.nsplit = pl.nsplit;
  p.tiles_per_split = pl.tiles_per_split;
  p.nkb = pl.nkb;
  p.stages = pl.stages;
  char* ws = reinterpret_cast<char*>(a.workspace);
  p.ws_o = reinterpret_cast<float*>(ws);
  p.ws_m = reinterpret_cast<float*>(ws + om);
  p.ws_l = reinterpret_cast<float*>(ws + ol);
  p.tickets = reinterpret_cast<unsigned int*>(ws + ot);
  int rc = attach_wait_diag(&g_wait_diag);
  if (rc != PCV_OK) return rc;
  // the workspace is caller memory with arbitrary contents: the tickets must start at zero
  PCV_CHECK_CUDA(cudaMemsetAsync(p.tickets, 0, (size_t)a.B * a.H * 4, stream));
  const dim3 grid((unsigned)((int64_t)pl.nsplit * a.B * a.H));
  auto run = [&](auto kernel) {
    // one limit for every head dim of the instantiation: the dynamic size varies with dqk
    const int r = set_smem_limit(reinterpret_cast<const void*>(kernel), kSmemLimit);
    return r != PCV_OK ? r : launch_kernel(kernel, grid, kThreads, pl.smem, 0, stream, p);
  };
  auto pick = [&](auto bf16, auto fp8, auto win) {
    constexpr bool BF16 = decltype(bf16)::value, FP8 = decltype(fp8)::value, WIN = decltype(win)::value;
    switch (pl.nvb) {
      case 1: return run(attn_cached_kernel<BF16, FP8, WIN, 1>);
      case 2: return run(attn_cached_kernel<BF16, FP8, WIN, 2>);
      case 3: return run(attn_cached_kernel<BF16, FP8, WIN, 3>);
      default: return run(attn_cached_kernel<BF16, FP8, WIN, 4>);
    }
  };
  // rows == nullptr: the whole e4m3 cache; else the window of an e4m3 (f) or 16-bit arena
  auto kind = [&](auto bf16) {
    if (rows == nullptr) return pick(bf16, std::true_type{}, std::false_type{});
    return f != nullptr ? pick(bf16, std::true_type{}, std::true_type{}) : pick(bf16, std::false_type{}, std::true_type{});
  };
  prof_mark_begin(stream);
  rc = a.dtype == PCV_BF16 ? kind(std::true_type{}) : kind(std::false_type{});
  prof_mark_end(stream);
  return rc;
}

}  // namespace pcv
