// pcv_attn_window.cu — attention of 1 to 64 bf16 / fp16 query rows over a device-resident key window of a KV arena on
// the Hopper tensor cores (sm_90a), with an optional causal band: a k-token step of a graph-replayed decode loop
// (draft tokens verified in one replay, a chunk of known tokens) sees for every one of its tokens exactly the keys the
// one-token loop gives that token.  The arena holds bf16 / fp16 rows of q's type or e4m3 codes.
//
//   grid = B * nsplit * H CTAs, head index fastest; nsplit is planned on the host from the arena's capacity (as
//   pcv_attn_cached_fp8 plans it from M), so the grid and the workspace are fixed for the life of a graph.  Batch row
//   b's window [w[0], w[1]), w = bounds + b * bounds_stride_b, is read from device memory when the kernel runs and
//   clamped to [0, capacity); its 64-key tiles start at its begin (not tile-aligned) and every split takes an equal
//   share of them.  256 threads:
//     warpgroup 1, the loader: 16-bit rows go straight into a ring of SWIZZLE_128B stages with 16-byte cp.async (keys
//       past the window's end and the channel tail of a k16 step are zero-filled); e4m3 rows are loaded into registers
//       and converted exactly to q's type, as attn_cached_fp8_kernel does.  full / empty mbarriers guard the ring.
//     warpgroup 0, the consumer: one m64 query tile (rows N .. 63 zero and dropped), S = Q K^T (m64n64k16, SS), the
//       online softmax in registers, O += P V (m64n64k16, P from registers) per 64-channel box.
//   Split states go to the workspace; the last CTA of every (b, h) merges them in split order: one launch, bitwise
//   reproducible.
//
// Masks.  Query i sits at arena row r_i = end - N + i.  Pad bytes are indexed by the absolute arena row.
//   - band W == 0: masks as pcv_attn_cached_fp8 on the window: the causal mask is right-aligned to the window's end,
//     padded and causally masked keys take the finite fill (a fully masked row is the uniform average of the window);
//   - band W > 0 (causal only): query i sees exactly the keys [r_i + 1 - W, r_i] of the window.  Every other key is
//     excluded: it contributes nothing, like a key outside the window, and takes no fill.  Padded keys inside the band
//     take the fill, so a row whose band is all padding is the uniform average over its band.
//   A tile, or a whole split, can hold no key of a row: its running maximum stays -inf, the rescale of an empty state
//   is skipped, and an empty split state (m = -inf, l = 0) merges with weight 0.  A window of length <= 0 writes zeros.
//
// Arithmetic contract (that of pcv_attn_cached.cu; the tests derive their element-wise gate from it):
//   - 16-bit K / V enter the MMA as stored; e4m3 codes exactly (every e4m3 value is an fp16 and a bf16 value);
//   - q enters unrounded, in its own dtype; c = scale * log2(e) (times k_descale[h] for e4m3 rows) multiplies the fp32
//     score s once: the row maximum m is taken over round(s * c), and p = 2^(fma(s, c, -m)) (ex2.approx);
//   - the online softmax runs in fp32 in the log2 domain; P is rounded to q's 16-bit type before P V while the
//     denominators sum the fp32 p; for e4m3 rows v_descale[h, c] multiplies the fp32 accumulator once, before the merge.
//   With the window [0, capacity) and no band, the e4m3 kernel computes what attn_cached_fp8_kernel computes, bit for
//   bit.
#include "pcv_common.cuh"
#include "pcv_sm90.cuh"
#include "pcv_cached_tile.cuh"

#include <algorithm>
#include <type_traits>

namespace pcv {
namespace {

using namespace sm90;
using namespace cached_tile;

constexpr int kKeys = 64;               // keys per tile
constexpr int kMaxRows = 64;            // query rows: one m64 tile
constexpr int kBox = 64 * 128;          // one box: 64 rows x 64 16-bit channels, SWIZZLE_128B
constexpr int kThreads = 256;           // consumer warpgroup + loader warpgroup
constexpr int kMaxStages = 4;
constexpr int kSmemLimit = 227 * 1024 - 1024;  // dynamic bytes: the per-block limit less room for the static s_last
constexpr int kPairBudget = 110 * 1024; // per CTA when two share an SM (228 KB per SM, 1 KB reserved per CTA)

struct WindowParams {
  pcv_attn_params a;
  pcv_decode_fp8 f;             // e4m3 rows only
  const int32_t* win;           // device: [begin, end) of the window
  int band;                     // > 0: query i sees keys [r_i + 1 - band, r_i] only
  int nsplit;
  int nkb;                      // 64-channel boxes of a q / K row
  int stages;
  float* ws_o;                  // [B*H][nsplit][N][dv]
  float* ws_m;                  // [B*H][nsplit][N]
  float* ws_l;                  // [B*H][nsplit][N]
  unsigned int* tickets;        // [B*H], zero on entry; the last CTA of a (b, h) resets its ticket
  int win_stride_b;             // int32s between the windows of batch rows b and b + 1 (0: one shared window)
};

// 16 bytes global -> shared, zero-filled when !live (nothing is read then)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool live) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(live ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// FP8: e4m3 arena rows, else rows of q's 16-bit type.  NVB: 64-channel boxes of a V row (ceil(dv / 64)).  Dynamic
// shared memory: [Q: nkb boxes][stage: nkb K boxes, NVB V boxes] x stages, then the barriers.
template <bool BF16, bool FP8, int NVB>
__global__ void __launch_bounds__(kThreads, NVB == 1 ? 2 : 1) attn_window_kernel(const WindowParams p) {
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
  // the window clamped to the arena; this split takes its tiles [t0, t1), tile t = keys w0 + 64 t .. (< wend)
  const int32_t* win = p.win + (int64_t)b * p.win_stride_b;
  const int w0 = max(win[0], 0), wend = min(win[1], a.M);
  const int ntiles = (max(wend - w0, 0) + kKeys - 1) / kKeys;
  const int tps = (ntiles + p.nsplit - 1) / p.nsplit;
  const int t0 = min(ntiles, split * tps), t1 = min(ntiles, t0 + tps);

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
      // units of U keys, two in registers (one stored while the next one's loads are in flight), as in
      // attn_cached_fp8_kernel
      constexpr int U = NVB == 1 ? 32 : 64, P = kKeys / U;
      constexpr int KU = U / 8, VU = U * NVB / 32;
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
      auto put = [&](const uint4 (&kr)[KU], const uint4 (&vr)[VU], int z) {
        const int i = z / P - t0, slot = i % S, part = z % P;
        const uint32_t st = ring_base + slot * stage_bytes;
        if (part == 0) mbar_wait(&empty[slot], ((i / S) & 1) ^ 1, 63);
        store(kr, vr, st, part);
        if (part == P - 1) {
          fence_proxy_async_smem();  // the generic-proxy stores, before the wgmma (async proxy) reads them
          warp_arrive(&full[slot]);
        }
      };
      uint4 ka[KU], va[VU], kb[KU], vb[VU];
      const int z1 = t1 * P;
      if (t0 < t1) load(ka, va, t0 * P);
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
        mbar_wait(&empty[slot], ((i / S) & 1) ^ 1, 63);
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
    const int ksteps = (a.dqk + 15) / 16;
    {  // q -> shared memory, rows N .. 63 and the channel tail of the last k16 step zero
      const int nq8 = a.dqk / 8;
      const T* qp = reinterpret_cast<const T*>(a.q) + (a.q_stride_b ? (int64_t)b * a.q_stride_b : 0) + (int64_t)h * a.q_stride_h;
      for (int idx = threadIdx.x; idx < kMaxRows * 2 * ksteps; idx += 128) {
        const int r = idx / (2 * ksteps), c8 = idx - r * 2 * ksteps;
        uint4 x = make_uint4(0, 0, 0, 0);
        if (r < a.N && c8 < nq8) x = *reinterpret_cast<const uint4*>(qp + (int64_t)r * a.q_stride_n + 8 * c8);
        st_shared_v4(q_base + (c8 >> 3) * kBox + swz(r, c8 & 7), x);
      }
      fence_proxy_async_smem();
      named_bar_sync<1, 128>();
    }
    float c = a.scale * kLog2e;  // fp32 score -> log2 domain
    if constexpr (FP8) c = a.scale * kLog2e * p.f.k_descale[h];
    const int cshift = wend - a.N;  // query n sits at row n + cshift
    const int band = p.band;
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
      mbar_wait(&full[slot], (i / S) & 1, 64);
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
        alpha[r] = mn == -INFINITY ? 1.f : ex2(m_run[r] - mn);  // no key of this row yet: nothing to rescale
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

    // this split's state -> workspace (an empty split writes m = -inf, l = 0, o = 0)
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
      const float wt = ms == -INFINITY ? 0.f : exp2f(ms - mm);  // an empty split state has weight 0
      ov = fmaf(__ldcg(p.ws_o + (sb + (int64_t)sp * a.N) * a.dv + ch), wt, ov);
      ll = fmaf(__ldcg(p.ws_l + sb + (int64_t)sp * a.N), wt, ll);
    }
    T* out = reinterpret_cast<T*>(a.out) + (int64_t)b * a.o_stride_b + (int64_t)n * a.o_stride_n + (int64_t)h * a.o_stride_h;
    out[ch] = Elem<T>::from_f(ll > 0.f ? ov / ll : 0.f);  // an empty window writes zeros
  }
}

int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

struct WindowPlan {
  int nkb, nvb;
  int ctas_per_sm;      // 2 when two CTAs fit (dv <= 64, dqk <= 192: registers and shared memory), else 1
  int stages;           // >= 2 for every head dim up to 256
  int smem;             // dynamic shared memory bytes
  int nsplit;
};

// pcv_attn_cached_fp8's plan on M = capacity: about two waves of resident CTAs over all (b, h), at least 4 tiles (256
// keys) of the arena per split, at most 256 splits.
WindowPlan plan_window(const pcv_attn_params& a, int sms) {
  WindowPlan pl;
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
  pl.nsplit = (int)((tiles + tps - 1) / tps);
  return pl;
}

size_t align256(size_t x) { return (x + 255) / 256 * 256; }

size_t workspace_of(const pcv_attn_params& a, const WindowPlan& pl, size_t* off_m, size_t* off_l, size_t* off_t) {
  const size_t rows = (size_t)a.B * a.H * pl.nsplit * a.N;
  *off_m = align256(rows * a.dv * 4);
  *off_l = *off_m + align256(rows * 4);
  *off_t = *off_l + align256(rows * 4);
  return *off_t + align256((size_t)a.B * a.H * 4);
}

}  // namespace

bool attn_window_supported(const pcv_attn_params& a, const pcv_decode_fp8* f, const pcv_dev_rows& rows, int band,
                           const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (rows.bounds == nullptr) return fail("rows->bounds is NULL");
  if (rows.capacity < 1) return fail("rows->capacity must be >= 1");
  if (rows.capacity != a.M) return fail("M must equal rows->capacity (k / v / pad_mask point at arena row 0)");
  if (rows.bounds_stride_b < 0) return fail("rows->bounds_stride_b must be >= 0");
  if (a.dtype != PCV_BF16 && a.dtype != PCV_F16)
    return fail(f != nullptr ? "dtype (of q and out) must be bf16 or fp16"
                             : "dtype (of q, the K / V arenas and out) must be bf16 or fp16");
  if (a.impl != PCV_IMPL_AUTO) return fail("impl must be AUTO");
  if (a.N > kMaxRows) return fail("more than 64 query rows");
  if (band < 0) return fail("band must be >= 0");
  if (band > 0 && !a.causal) return fail("a band needs the causal mask");
  if (a.write_partial) return fail("the window attention writes the normalised output only (no write_partial)");
  if (a.m_total != a.M || a.m_offset != 0)
    return fail("the window attention takes no key shard (m_total != M or m_offset != 0)");
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

int attn_window_workspace_bytes(const pcv_attn_params& a, size_t* bytes) {
  size_t om, ol, ot;
  *bytes = workspace_of(a, plan_window(a, sm_count()), &om, &ol, &ot);
  return PCV_OK;
}

int launch_attn_window(const pcv_attn_params& a, const pcv_decode_fp8* f, const pcv_dev_rows& rows, int band,
                       cudaStream_t stream) {
  const WindowPlan pl = plan_window(a, sm_count());
  size_t om, ol, ot;
  const size_t need = workspace_of(a, pl, &om, &ol, &ot);
  PCV_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= need, PCV_ERR_WORKSPACE,
              "window attention: workspace of %zu bytes required, %zu given", need, a.workspace_bytes);
  if (const char* dp = device_problem()) {
    set_error("window attention: %s", dp);
    return PCV_ERR_UNSUPPORTED;
  }
  WindowParams p{};
  p.a = a;
  if (f != nullptr) p.f = *f;
  p.win = rows.bounds;
  p.win_stride_b = rows.bounds_stride_b;
  p.band = band;
  p.nsplit = pl.nsplit;
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
  auto pick = [&](auto bf16, auto fp8) {
    constexpr bool BF16 = decltype(bf16)::value, FP8 = decltype(fp8)::value;
    switch (pl.nvb) {
      case 1: return run(attn_window_kernel<BF16, FP8, 1>);
      case 2: return run(attn_window_kernel<BF16, FP8, 2>);
      case 3: return run(attn_window_kernel<BF16, FP8, 3>);
      default: return run(attn_window_kernel<BF16, FP8, 4>);
    }
  };
  prof_mark_begin(stream);
  if (a.dtype == PCV_BF16)
    rc = f != nullptr ? pick(std::true_type{}, std::true_type{}) : pick(std::true_type{}, std::false_type{});
  else
    rc = f != nullptr ? pick(std::false_type{}, std::true_type{}) : pick(std::false_type{}, std::false_type{});
  prof_mark_end(stream);
  return rc;
}

}  // namespace pcv
