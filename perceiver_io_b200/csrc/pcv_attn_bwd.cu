// pcv_attn_bwd.cu — training kernels of the fused attention core on the Hopper tensor cores (SURVEY.md §8(f)2):
// backward (C ABI pcv_attn_bwd, with attention-probability dropout) and the dropout mask export (pcv_attn_dropout_mask).
//
// Reference: autograd through perceiver/model/core/modules.py:141-167 (einsum scores, masked_fill_ with the finite
// fill, softmax, dropout, einsum with V).  With P = softmax(scale * Q K^T + fill), O = P V and the saved row statistics
// (m, l) of the forward kernel (log2 domain: P = 2^(t - m) / l, t = scale*log2(e) * q.k):
//     delta_q = sum_c dO[q,c] O[q,c]            dP = dO V^T            dS = P * (dP - delta)   (0 where filled)
//     dV = P^T dO            dK = scale * dS^T Q            dQ = scale * dS K
// The shape of the path is asymmetric (N = a few hundred latent queries, M >> N keys), so the work is split into two
// kernels that never hold the (B, H, N, M) score tensor and need no atomics on the large axis:
//
//   bwd_dkdv_kernel  key-tile outer, persistent.  One CTA owns a 128-key tile (K, V resident in shared memory) and walks
//                    the queries in sub-steps of 64.  Scores are computed TRANSPOSED, S^T = K Q^T and dP^T = V dO^T
//                    (wgmma SS, accumulator rows = keys), so P^T and dS^T, rounded to bf16/fp16, stay in registers and
//                    feed dV += P^T dO and dK += dS^T Q as the A operand (wgmma RS, B = dO / Q stage read MN-major).
//   bwd_dq_kernel    query-tile outer.  A work item is (b, h, 128 queries) and a range of key tiles (K and V streamed
//                    through a TMA ring in stages of KS keys); S = Q K^T, dP = dO V^T, dS in registers, dQ += dS K (K
//                    stage read MN-major, as V is in the forward).  dQ accumulates in registers over the item's key
//                    range and leaves once per item: added into an fp32 buffer (KS = 128), or stored as an ordered
//                    fp32 partial (KS = 64).
//
// Head dims above 128 (up to 192: a third 64-channel box) run the dK/dV kernel as a dV pass and a dK pass and the dQ
// kernel on 64-key stages; see dq_ordered_partials.
//
// Warpgroup 0 is the TMA producer (one lane), warpgroups 1 and 2 each own 64 rows of the tile.
#include "pcv_common.cuh"
#include "pcv_dropout.cuh"
#include "pcv_sm90.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <type_traits>

namespace pcv {
namespace {

using namespace sm90;

constexpr int kT = 128;                 // tile rows (queries or keys)
constexpr int kBoxBytes = kT * 128;     // one TMA box: 128 rows x 64 16-bit channels, SWIZZLE_128B
constexpr int kThreads = 384;
constexpr int kSmemLimit = 227 * 1024;
constexpr int kStatsBytes = 64 * 12;    // row statistics of one block of 64 queries (see bwd_prep_kernel)
constexpr int kBox64 = 64 * 128;        // a 64-row TMA box (the dK/dV kernel stages Q / dO in 64-query pieces)

struct BwdParams {
  int B, H, N, M, dqk, dv;
  int Npad, nq, nk;          // query rows padded to tiles, query tiles, key tiles
  int q_bcast;               // q has one batch row shared by all b (latents)
  float scale, scale_log2;
  int causal, cshift;        // local key j masked for query n iff j > n + cshift   (right aligned over all keys:
                             // cshift = (m_total - N) - key_base)
  const uint32_t* pad_bits;  // (B, pad_wpr) bit set = padding key; nullptr if none
  int pad_wpr;
  const float* stats;        // (B, H, 2*nq) blocks of kStatsBytes (layout: see bwd_prep_kernel)
  float* dq32;               // (Bq, N, H*dqk) fp32, zero-initialised, that CTAs reduce into; or the dQ partials
  void* dk;
  void* dv_out;
  int64_t dk_sb, dk_sm, dk_sh, dv_sb, dv_sm, dv_sh;
  uint32_t drop_thresh;      // attention dropout: element kept iff its random byte >= drop_thresh (0 = no dropout)
  uint32_t seed_lo, seed_hi;
  int key_base;              // global index of local key 0 (even; 0 unless key-sharded): the mask hashes key_base + j
  float drop_rp;             // 1 / (1 - drop_thresh / 256)
  int total_tiles;           // dkdv kernel: B*H*nk
  int splits, tiles_per_split;  // dq kernel
};

// keep mask of keys [key_begin, key_begin + W) (tests / the backward shim): keep[b][h][q][k - key_begin] = 1 if the
// element survives
__global__ void __launch_bounds__(256) drop_mask_kernel(uint8_t* __restrict__ keep, int B, int H, int N, int key_begin,
                                                        int W, uint32_t thresh, uint32_t seed_lo, uint32_t seed_hi) {
  const int64_t total = (int64_t)B * H * N * W;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t k = (uint32_t)(key_begin + idx % W);
    const int64_t r = idx / W;
    const uint32_t q = (uint32_t)(r % N), bh = (uint32_t)(r / N);
    keep[idx] = drop_keep(drop_bits(seed_lo, seed_hi, bh, q, k), q, k, thresh) ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Row statistics, one 768-byte block per (b, h, 64 queries): 32 x float4 {nlse[2c], nlse[2c+1], delta[2c], delta[2c+1]}
// then 64 x float fillp.   nlse = -(m + log2 l) so that P = 2^(t + nlse); delta = sum_c dO*O; fillp = the probability
// of a FILLED score: 1/l on a row whose scores are all filled (uniform attention), else 0.  Rows beyond N (tile
// padding) and fully filled rows get nlse = -inf (their live P is exactly 0).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int stat_nlse_idx(int r) { return (r >> 1) * 4 + (r & 1); }
__device__ __forceinline__ int stat_delta_idx(int r) { return (r >> 1) * 4 + 2 + (r & 1); }
__device__ __forceinline__ int stat_fillp_idx(int r) { return 128 + r; }

template <typename T>
__global__ void __launch_bounds__(256) bwd_prep_kernel(const T* __restrict__ out, const T* __restrict__ dout,
                                                       const float* __restrict__ stat_m,
                                                       const float* __restrict__ stat_l, float* __restrict__ stats,
                                                       int B, int H, int N, int Npad, int dv, int64_t o_sb,
                                                       int64_t o_sn, int64_t o_sh, int64_t g_sb, int64_t g_sn,
                                                       int64_t g_sh) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (int64_t)B * H * Npad) return;
  const int n = (int)(row % Npad);
  const int64_t bh = row / Npad;
  const int h = (int)(bh % H), b = (int)(bh / H);
  float nlse = -INFINITY, delta = 0.f, fillp = 0.f;
  if (n < N) {
    const T* o = out + b * o_sb + (int64_t)n * o_sn + h * o_sh;
    const T* g = dout + b * g_sb + (int64_t)n * g_sn + h * g_sh;
    float acc = 0.f;
    for (int c = lane; c < dv; c += 32) acc += Elem<T>::to_f(o[c]) * Elem<T>::to_f(g[c]);
    delta = warp_sum(acc);
    const int64_t r = bh * N + n;
    const float m = stat_m[r], l = stat_l[r];
    if (m <= -1e37f)
      fillp = 1.f / l;  // every score of the row is the finite fill: uniform over the l filled keys
    else
      nlse = -(m + log2f(l));
  }
  if (lane == 0) {
    float* blk = stats + (bh * (Npad / 64) + n / 64) * (kStatsBytes / 4);
    const int r = n % 64;
    blk[stat_nlse_idx(r)] = nlse;
    blk[stat_delta_idx(r)] = delta;
    blk[stat_fillp_idx(r)] = fillp;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// kernel 1: dK, dV.  CTA = one 128-key tile (K, V resident in shared memory; persistent over tiles), warpgroups 1-2
// own 64 keys each and walk the queries in sub-steps of 64 (Q / dO pieces through a TMA ring).
// ---------------------------------------------------------------------------------------------------------------
template <int NQB, int NVB>
struct Cfg1 {
  static constexpr int kKVBytes = (NQB + NVB) * kBoxBytes;
  static constexpr int kStage = (NQB + NVB) * kBox64;
  static constexpr int kSlots = (kSmemLimit - kKVBytes - 2048) / kStage > 8 ? 8 : (kSmemLimit - kKVBytes - 2048) / kStage;
  static constexpr int kSmem = kKVBytes + kSlots * kStage + 2048;
};

// kernel 2 (dQ): work item = (b, h, 128 queries, key range); warpgroups 1-2 own 64 queries each; Q and dO stay
// resident per item, K / V stream through a TMA ring in stages of KS keys (a KS-row box per 64 channels).
template <int NQB, int NVB, int KS>
struct Cfg2 {
  static constexpr int kQBytes = (NQB + NVB) * kBoxBytes;
  static constexpr int kKSBox = KS * 128;
  static constexpr int kStage = (NQB + NVB) * kKSBox;
  static constexpr int kSlots = (kSmemLimit - kQBytes - 2048) / kStage > 4 ? 4 : (kSmemLimit - kQBytes - 2048) / kStage;
  static constexpr int kSmem = kQBytes + kSlots * kStage + 2048;
  static_assert(kSlots >= 2, "shared memory budget");
};

struct BwdBarriers {
  uint64_t full[8], empty[8];
  uint64_t fix_full, fix_empty;
};

__device__ __forceinline__ bool filled_key(const BwdParams& p, int b, int j, int n) {
  if (p.pad_bits != nullptr && ((p.pad_bits[(int64_t)b * p.pad_wpr + (j >> 5)] >> (j & 31)) & 1u)) return true;
  return p.causal && j > n + p.cshift;
}

// The score-gradient rule of one element (query n, local key j, score s = q.k, dP = dO.v) with the row statistics of
// query n: P = 2^(s * scale_log2 + nlse), fillp on a filled key, 0 outside the problem; pd = P after dropout (the dV
// operand) and ds = P (dP' - delta) with dP' = dP after dropout, 0 on filled keys and outside the problem.  A caller
// that uses one of the two lets the compiler drop the other.  Without dropout neither is scaled (drop_rp would be
// exactly 1: dropout_rule).  bwd_dkdv_kernel writes the same rule out in its element loop: through this helper its
// wide dV and dK passes ran about 10 % slower on an H100 SXM (700 W).
struct ScoreGrad {
  float pd, ds;
};

__device__ __forceinline__ ScoreGrad score_grad(const BwdParams& p, int b, int bh, int n, int j, float s, float dP,
                                                float nlse, float delta, float fillp) {
  const bool oob = j >= p.M || n >= p.N;
  const bool filled = !oob && filled_key(p, b, j, n);
  const float P = oob ? 0.f : (filled ? fillp : ex2(fmaf(s, p.scale_log2, nlse)));
  float pd = P;
  if (p.drop_thresh) {
    const uint32_t jg = (uint32_t)(p.key_base + j);
    const bool keep = drop_keep(drop_bits(p.seed_lo, p.seed_hi, (uint32_t)bh, (uint32_t)n, jg), n, jg, p.drop_thresh);
    dP = keep ? dP * p.drop_rp : 0.f;
    pd = keep ? P * p.drop_rp : 0.f;
  }
  return {pd, (oob || filled) ? 0.f : P * (dP - delta)};
}

// Outputs of one bwd_dkdv_kernel launch.  With a head dim above 128 (a third 64-channel box) the dK and dV accumulators
// do not fit the consumer registers beside S^T, dP^T and the packed operands without spilling (ptxas spills already at
// (1, 3) and (3, 1)), so the backward runs the kernel twice: a dV pass (K resident, no dP^T GEMM, no dS) and a dK pass
// (K and V resident).  Each pass computes S^T = K Q^T: one extra GEMM of dqk channels per (key, query) pair.
enum DkdvOut : int { kOutBoth = 0, kOutDV = 1, kOutDK = 2 };

template <int NQB, int NVB, bool BF16, int OUT = kOutBoth>
__global__ void __launch_bounds__(kThreads, 1)
bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tq64, const __grid_constant__ CUtensorMap tk,
                const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap tdo64, const BwdParams p) {
  using C = Cfg1<NQB, NVB>;
  constexpr int NS = C::kSlots;
  constexpr bool kDK = OUT != kOutDV, kDV = OUT != kOutDK;
  constexpr int kResident = kDK ? C::kKVBytes : NQB * kBoxBytes;  // the dV pass leaves V's boxes empty
  using T = typename std::conditional<BF16, __nv_bfloat16, __half>::type;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = smem + NQB * kBoxBytes;
  uint8_t* sRing = smem + C::kKVBytes;
  BwdBarriers& bar = *reinterpret_cast<BwdBarriers*>(sRing + NS * C::kStage);
  const int wg = threadIdx.x / 128;
  const int nq64 = (p.N + 63) / 64;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&bar.full[s], 1);
      mbar_init(&bar.empty[s], 8);
    }
    mbar_init(&bar.fix_full, 1);
    mbar_init(&bar.fix_empty, 8);
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0, tl = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++tl) {
        const int bh = tile / p.nk, kt = tile % p.nk, b = bh / p.H, h = bh % p.H;
        mbar_wait(&bar.fix_empty, (tl & 1) ^ 1, 21);
        mbar_arrive_expect_tx(&bar.fix_full, kResident);
        for (int c = 0; c < NQB; ++c) tma_load_4d(sK + c * kBoxBytes, &tk, &bar.fix_full, c * 64, kt * kT, h, b);
        if constexpr (kDK)
          for (int c = 0; c < NVB; ++c) tma_load_4d(sV + c * kBoxBytes, &tv, &bar.fix_full, c * 64, kt * kT, h, b);
        for (int qs = 0; qs < nq64; ++qs, ++it) {
          const uint32_t s = it % NS;
          mbar_wait(&bar.empty[s], ((it / NS) & 1) ^ 1, 22);
          mbar_arrive_expect_tx(&bar.full[s], C::kStage);
          uint8_t* st = sRing + s * C::kStage;
          for (int c = 0; c < NQB; ++c)
            tma_load_4d(st + c * kBox64, &tq64, &bar.full[s], c * 64, qs * 64, h, p.q_bcast ? 0 : b);
          for (int c = 0; c < NVB; ++c)
            tma_load_4d(st + (NQB + c) * kBox64, &tdo64, &bar.full[s], c * 64, qs * 64, h, b);
        }
      }
    }
    return;
  }

  reg_alloc<232>();
  const int cw = wg - 1;
  const int tid = threadIdx.x - 128 * wg;
  const int warp = tid >> 5, lane = tid & 31;
  const int kloc = 64 * cw + 16 * warp + (lane >> 2);  // key rows kloc, kloc + 8 of the tile
  const int cq = 2 * (lane & 3);
  const uint32_t k_base = smem_u32(sK) + cw * 64 * 128, v_base = smem_u32(sV) + cw * 64 * 128;
  const uint32_t ring = smem_u32(sRing);
  uint32_t it = 0, tl = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++tl) {
    const int bh = tile / p.nk, kt = tile % p.nk, b = bh / p.H, h = bh % p.H;
    mbar_wait(&bar.fix_full, tl & 1, 23);
    constexpr int NK = kDK ? NQB : 0, NV = kDV ? NVB : 0;  // accumulator boxes of this launch
    float dk[kDK ? NQB : 1][32], dv[kDV ? NVB : 1][32];
#pragma unroll
    for (int c = 0; c < NK; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) dk[c][i] = 0.f;
#pragma unroll
    for (int c = 0; c < NV; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) dv[c][i] = 0.f;
    const int jrow[2] = {kt * kT + kloc, kt * kT + kloc + 8};
    for (int qs = 0; qs < nq64; ++qs, ++it) {
      const uint32_t s = it % NS;
      const uint32_t stq = ring + s * C::kStage, stdo = stq + NQB * kBox64;
      mbar_wait(&bar.full[s], (it / NS) & 1, 24);
      float st[32], dpt[kDK ? 32 : 1];
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < NQB; ++c)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_ss<64, BF16>(st, make_desc(k_base + c * kBoxBytes + kk * 32), make_desc(stq + c * kBox64 + kk * 32), (c | kk) != 0);
      if constexpr (kDK) {
#pragma unroll
        for (int c = 0; c < NVB; ++c)
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
            wgmma_ss<64, BF16>(dpt, make_desc(v_base + c * kBoxBytes + kk * 32), make_desc(stdo + c * kBox64 + kk * 32), (c | kk) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(st);
      if constexpr (kDK) fence_regs(dpt);
      const float* blk = p.stats + ((int64_t)bh * (p.Npad / 64) + qs) * (kStatsBytes / 4);
      uint32_t pa[kDV ? 4 : 1][4], da[kDK ? 4 : 1][4];
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        float pv[4], dsv[4];
#pragma unroll
        for (int e4 = 0; e4 < 4; ++e4) {
          const int i = e4 >> 1, e = e4 & 1;
          const int qc = 8 * g + cq + e;
          const int n = qs * 64 + qc, j = jrow[i];
          const float nlse = blk[stat_nlse_idx(qc)], delta = blk[stat_delta_idx(qc)], fillp = blk[stat_fillp_idx(qc)];
          const bool oob = j >= p.M || n >= p.N;
          const bool filled = !oob && filled_key(p, b, j, n);
          float P = oob ? 0.f : (filled ? fillp : ex2(fmaf(st[4 * g + e4], p.scale_log2, nlse)));
          const uint32_t jg = (uint32_t)(p.key_base + j);
          if constexpr (kDK) {
            float dP = dpt[4 * g + e4];
            if (p.drop_thresh) {
              const bool keep = drop_keep(drop_bits(p.seed_lo, p.seed_hi, (uint32_t)bh, (uint32_t)n, jg), n, jg, p.drop_thresh);
              dP = keep ? dP * p.drop_rp : 0.f;
              pv[e4] = keep ? P * p.drop_rp : 0.f;
            } else {
              pv[e4] = P;
            }
            dsv[e4] = (oob || filled) ? 0.f : P * (dP - delta);
          } else {
            (void)delta;  // the dV pass needs no dS
            if (p.drop_thresh) {
              const bool keep = drop_keep(drop_bits(p.seed_lo, p.seed_hi, (uint32_t)bh, (uint32_t)n, jg), n, jg, p.drop_thresh);
              pv[e4] = keep ? P * p.drop_rp : 0.f;
            } else {
              pv[e4] = P;
            }
          }
        }
        if constexpr (kDV) {
          pa[g >> 1][(g & 1) * 2 + 0] = pack2(pv[0], pv[1], BF16);
          pa[g >> 1][(g & 1) * 2 + 1] = pack2(pv[2], pv[3], BF16);
        }
        if constexpr (kDK) {
          da[g >> 1][(g & 1) * 2 + 0] = pack2(dsv[0], dsv[1], BF16);
          da[g >> 1][(g & 1) * 2 + 1] = pack2(dsv[2], dsv[3], BF16);
        }
      }
      wgmma_fence();
      if constexpr (kDV) {
#pragma unroll
        for (int c = 0; c < NVB; ++c)
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_rs<64, BF16>(dv[c], pa[kk], make_desc(stdo + c * kBox64 + kk * 2048));
      }
      if constexpr (kDK) {
#pragma unroll
        for (int c = 0; c < NQB; ++c)
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_rs<64, BF16>(dk[c], da[kk], make_desc(stq + c * kBox64 + kk * 2048));
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < NV; ++c) fence_regs(dv[c]);
#pragma unroll
      for (int c = 0; c < NK; ++c) fence_regs(dk[c]);
      warp_arrive(&bar.empty[s]);
    }
    warp_arrive(&bar.fix_empty);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int j = jrow[i];
      if (j >= p.M) continue;
      T* krow = reinterpret_cast<T*>(p.dk) + (int64_t)b * p.dk_sb + (int64_t)j * p.dk_sm + (int64_t)h * p.dk_sh;
      T* vrow = reinterpret_cast<T*>(p.dv_out) + (int64_t)b * p.dv_sb + (int64_t)j * p.dv_sm + (int64_t)h * p.dv_sh;
#pragma unroll
      for (int c = 0; c < NK; ++c)
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const int col = c * 64 + 8 * g + cq;
          if (col < p.dqk)
            *reinterpret_cast<uint32_t*>(krow + col) = pack2(dk[c][4 * g + 2 * i] * p.scale, dk[c][4 * g + 2 * i + 1] * p.scale, BF16);
        }
#pragma unroll
      for (int c = 0; c < NV; ++c)
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const int col = c * 64 + 8 * g + cq;
          if (col < p.dv) *reinterpret_cast<uint32_t*>(vrow + col) = pack2(dv[c][4 * g + 2 * i], dv[c][4 * g + 2 * i + 1], BF16);
        }
    }
  }
}

// The dQ epilogue of KS-key stages.  Head dims above 128 run the dQ kernel on 64-key stages: S and dP then take 32
// registers each beside the three dQ accumulator boxes, and that is what keeps those instantiations spill-free (a
// 128-key stage needs 64 + 64).  Their work items store their dQ share (already scaled) as one fp32 partial
// (Bq, N, H*dqk) per (batch contribution, split), partial index (q_bcast ? b : 0) * splits + split, and
// bwd_sum_dq_kernel adds the partials in index order, so the wide dQ is bitwise reproducible.  128-key stages add their
// share into the zeroed fp32 p.dq32 with atomics.
constexpr bool dq_ordered_partials(int ks) { return ks == 64; }

// dQ += scale * dS K.  CTAs walk the work items (b, h, query tile, split) persistently, as the dK/dV kernel walks its
// key tiles; with 128-key stages the grid is one CTA per item.  A split covers tiles_per_split tiles of 128 keys, i.e.
// tiles_per_split * 128 / KS stages.
template <int NQB, int NVB, bool BF16, int KS>
__global__ void __launch_bounds__(kThreads, 1)
bwd_dq_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
              const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap tdo, const BwdParams p) {
  using C = Cfg2<NQB, NVB, KS>;
  constexpr int NS = C::kSlots;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sdO = smem + NQB * kBoxBytes;
  uint8_t* sRing = smem + C::kQBytes;
  BwdBarriers& bar = *reinterpret_cast<BwdBarriers*>(sRing + NS * C::kStage);
  const int wg = threadIdx.x / 128;
  const int total = p.B * p.H * p.nq * p.splits;  // work items (b, h, query tile, split)
  const int nks = (p.M + KS - 1) / KS, per_split = p.tiles_per_split * (kT / KS);  // stages in all, per split
  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&bar.full[s], 1);
      mbar_init(&bar.empty[s], 8);
    }
    mbar_init(&bar.fix_full, 1);
    mbar_init(&bar.fix_empty, 8);
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0, wl = 0;
      for (int w = blockIdx.x; w < total; w += gridDim.x, ++wl) {
        const int unit = w / p.splits, split = w % p.splits;
        const int bh = unit / p.nq, qt = unit % p.nq, b = bh / p.H, h = bh % p.H;
        const int kt0 = split * per_split, kt1 = min(nks, kt0 + per_split);
        mbar_wait(&bar.fix_empty, (wl & 1) ^ 1, 34);
        mbar_arrive_expect_tx(&bar.fix_full, C::kQBytes);
        for (int c = 0; c < NQB; ++c)
          tma_load_4d(sQ + c * kBoxBytes, &tq, &bar.fix_full, c * 64, qt * kT, h, p.q_bcast ? 0 : b);
        for (int c = 0; c < NVB; ++c) tma_load_4d(sdO + c * kBoxBytes, &tdo, &bar.fix_full, c * 64, qt * kT, h, b);
        for (int kt = kt0; kt < kt1; ++kt, ++it) {
          const uint32_t s = it % NS;
          mbar_wait(&bar.empty[s], ((it / NS) & 1) ^ 1, 31);
          mbar_arrive_expect_tx(&bar.full[s], C::kStage);
          uint8_t* st = sRing + s * C::kStage;
          for (int c = 0; c < NQB; ++c) tma_load_4d(st + c * C::kKSBox, &tk, &bar.full[s], c * 64, kt * KS, h, b);
          for (int c = 0; c < NVB; ++c)
            tma_load_4d(st + (NQB + c) * C::kKSBox, &tv, &bar.full[s], c * 64, kt * KS, h, b);
        }
      }
    }
    return;
  }

  reg_alloc<232>();
  const int cw = wg - 1;
  const int tid = threadIdx.x - 128 * wg;
  const int warp = tid >> 5, lane = tid & 31;
  const int qloc = 64 * cw + 16 * warp + (lane >> 2);
  const int r0 = 16 * warp + (lane >> 2);  // this thread's rows r0, r0 + 8 of its warpgroup's 64-query statistics block
  const int cq = 2 * (lane & 3);
  const uint32_t q_base = smem_u32(sQ) + cw * 64 * 128, do_base = smem_u32(sdO) + cw * 64 * 128;
  const uint32_t ring = smem_u32(sRing);
  uint32_t it = 0, wl = 0;
  for (int w = blockIdx.x; w < total; w += gridDim.x, ++wl) {
    const int unit = w / p.splits, split = w % p.splits;
    const int bh = unit / p.nq, qt = unit % p.nq, b = bh / p.H, h = bh % p.H;
    const int kt0 = split * per_split, kt1 = min(nks, kt0 + per_split);
    const float* blk = p.stats + ((int64_t)bh * (p.Npad / 64) + 2 * qt + cw) * (kStatsBytes / 4);
    mbar_wait(&bar.fix_full, wl & 1, 32);
    float acc[NQB][32];
#pragma unroll
    for (int c = 0; c < NQB; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
    for (int kt = kt0; kt < kt1; ++kt, ++it) {
      const uint32_t s = it % NS;
      const uint32_t stk = ring + s * C::kStage, stv = stk + NQB * C::kKSBox;
      mbar_wait(&bar.full[s], (it / NS) & 1, 33);
      float sc[KS / 2], dp[KS / 2];
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < NQB; ++c)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_ss<KS, BF16>(sc, make_desc(q_base + c * kBoxBytes + kk * 32), make_desc(stk + c * C::kKSBox + kk * 32), (c | kk) != 0);
#pragma unroll
      for (int c = 0; c < NVB; ++c)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_ss<KS, BF16>(dp, make_desc(do_base + c * kBoxBytes + kk * 32), make_desc(stv + c * C::kKSBox + kk * 32), (c | kk) != 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(sc);
      fence_regs(dp);
      uint32_t a[KS / 16][4];
#pragma unroll
      for (int g = 0; g < KS / 8; ++g) {
        float val[4];
#pragma unroll
        for (int e4 = 0; e4 < 4; ++e4) {
          const int i = e4 >> 1, e = e4 & 1;
          const int r = r0 + 8 * i;
          val[e4] = score_grad(p, b, bh, qt * kT + qloc + 8 * i, kt * KS + 8 * g + cq + e, sc[4 * g + e4], dp[4 * g + e4],
                               blk[stat_nlse_idx(r)], blk[stat_delta_idx(r)], blk[stat_fillp_idx(r)]).ds;
        }
        a[g >> 1][(g & 1) * 2 + 0] = pack2(val[0], val[1], BF16);
        a[g >> 1][(g & 1) * 2 + 1] = pack2(val[2], val[3], BF16);
      }
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < NQB; ++c)
#pragma unroll
        for (int kk = 0; kk < KS / 16; ++kk) wgmma_rs<64, BF16>(acc[c], a[kk], make_desc(stk + c * C::kKSBox + kk * 2048));
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < NQB; ++c) fence_regs(acc[c]);
      warp_arrive(&bar.empty[s]);
    }
    warp_arrive(&bar.fix_empty);
    const int Bq = p.q_bcast ? 1 : p.B, bq = p.q_bcast ? 0 : b;
    const int64_t part = dq_ordered_partials(KS) ? (int64_t)(p.q_bcast ? b : 0) * p.splits + split : 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int n = qt * kT + qloc + 8 * i;
      if (n >= p.N) continue;
      float* dst = p.dq32 + (((part * Bq + bq) * p.N + n) * p.H + h) * p.dqk;
#pragma unroll
      for (int c = 0; c < NQB; ++c)
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const int col = c * 64 + 8 * g + cq;
          if (col >= p.dqk) continue;
          const float x = acc[c][4 * g + 2 * i] * p.scale, y = acc[c][4 * g + 2 * i + 1] * p.scale;
          if constexpr (dq_ordered_partials(KS)) {  // every element of the partial is written by exactly one item
            *reinterpret_cast<float2*>(dst + col) = make_float2(x, y);
          } else {
            atomicAdd(dst + col, x);
            atomicAdd(dst + col + 1, y);
          }
        }
    }
  }
}

// the dQ partials (nparts x (Bq, N, H*dqk) fp32; one, the atomics' buffer, up to head dim 128), added in partial order
// from 0.f -> dq (bf16, fp16 or fp32) with its own strides
template <typename T>
__global__ void __launch_bounds__(256) bwd_sum_dq_kernel(const float* __restrict__ part, int nparts, T* __restrict__ dq,
                                                         int Bq, int N, int H, int dqk, int64_t sb, int64_t sn, int64_t sh) {
  const int64_t total = (int64_t)Bq * N * H * dqk;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int i = 0; i < nparts; ++i) s += part[i * total + idx];
    const int c = (int)(idx % dqk);
    int64_t r = idx / dqk;
    const int h = (int)(r % H);
    r /= H;
    const int n = (int)(r % N);
    const int b = (int)(r / N);
    dq[b * sb + (int64_t)n * sn + h * sh + c] = Elem<T>::from_f(s);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------
inline size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

void set_dropout(BwdParams& p, float dropout_p, uint64_t seed) {
  const DropoutRule r = dropout_rule(dropout_p, seed);
  p.drop_thresh = r.thresh;
  p.drop_rp = r.scale;
  p.seed_lo = r.seed_lo;
  p.seed_hi = r.seed_hi;
}

// Split of the dq kernel's key tiles over CTAs: aim at ~64 key tiles per CTA (launch + Q/dO load amortised) but at
// least ~4 CTAs per SM in total
void dq_split(int units, int nk, int sms, int& tiles_per_split, int& splits) {
  int s = std::max(1, (nk + 63) / 64);
  while (units * s < 4 * sms && s < nk && (nk + s - 1) / s > 4) ++s;
  tiles_per_split = (nk + s - 1) / s;
  splits = (nk + tiles_per_split - 1) / tiles_per_split;
}

// Head dims above 128 take the wide variants: the dK/dV kernel with a third box as a dV and a dK pass, and the dQ
// kernel on 64-key stages with its ordered dQ partials (dq_ordered_partials).
constexpr bool wide_bwd(int dqk, int dv) { return dqk > 128 || dv > 128; }

// The wide dQ split is planned for a fixed SM count (the H100 SXM's 132), not the device's: the number of dQ partials,
// and so the workspace size, follow from the problem alone, and so does the order in which dQ is summed.
constexpr int kWideSplitSms = 132;

// Workspace of the backward: the row-statistics blocks, an fp32 dQ accumulator of acc_bytes (zeroed before the
// kernels; none for a key shard's or the wide backward), the pad bits, then part_bytes of dQ partials (the wide
// backward; written whole by its dQ kernel, so not zeroed).
struct BwdLayout {
  int Npad, nq, nk;
  int dq_splits, dq_tiles_per_split, dq_parts;  // the wide backward's dQ split and partial count (else 0)
  size_t acc_bytes, off_acc, off_pad, part_bytes, off_part, total;  // the statistics start at offset 0
};

// shard != nullptr: a key shard's backward, whose dQ kernel up to head dim 128 accumulates straight into the caller's
// fp32 grad_q32 (no accumulator in the workspace)
BwdLayout bwd_layout(const pcv_attn_bwd_params& a, const pcv_key_shard* shard) {
  const int Bq = a.q_stride_b == 0 ? 1 : a.B;
  const size_t dq_bytes = sizeof(float) * (size_t)Bq * a.N * a.H * a.dqk;
  const bool wide = wide_bwd(a.dqk, a.dv);
  BwdLayout L;
  L.nq = (a.N + kT - 1) / kT;
  L.nk = (a.M + kT - 1) / kT;
  L.Npad = L.nq * kT;
  L.dq_splits = L.dq_tiles_per_split = L.dq_parts = 0;
  L.acc_bytes = wide || shard != nullptr ? 0 : dq_bytes;
  L.off_acc = align256((size_t)kStatsBytes * a.B * a.H * 2 * L.nq);
  L.off_pad = L.off_acc + align256(L.acc_bytes);
  L.part_bytes = 0;
  L.off_part = L.total =
      L.off_pad + (a.pad_mask != nullptr ? align256(sizeof(uint32_t) * (size_t)a.B * pad_words_per_row(a.M)) : 0);
  if (!wide) return L;
  dq_split(a.B * a.H * L.nq, L.nk, kWideSplitSms, L.dq_tiles_per_split, L.dq_splits);
  L.dq_parts = (Bq == 1 ? a.B : 1) * L.dq_splits;  // a batch-1 q receives one contribution per batch row and split
  L.part_bytes = dq_bytes * L.dq_parts;
  L.total = L.off_part + align256(L.part_bytes);
  return L;
}

// Key rows of the dQ kernel's ring stages: 64 for the wide head dims (see dq_ordered_partials), else a whole tile.
constexpr int dq_stage_keys(int dqk, int dv) { return wide_bwd(dqk, dv) ? 64 : kT; }

// The tensor maps of one backward: Q and dO resident in the dQ kernel (128-row boxes) and staged by the dK/dV kernel
// (64-row boxes); K and V resident in the dK/dV kernel (128-row boxes) and staged by the dQ kernel (KS-row boxes).
struct BwdMaps {
  CUtensorMap q, dout, q64, dout64;
  CUtensorMap k, v, k_dq, v_dq;
};

// Fills the BwdParams core and the dq-kernel split, zeroes the fp32 accumulator, writes the row statistics, packs the
// pad mask and encodes the tensor maps.  The call's keys are [m_offset, m_offset + M) of m_total (the causal
// diagonal and the dropout hash use global key indices).
int bwd_setup(const pcv_attn_bwd_params& a, const BwdLayout& L, int m_total, int m_offset, cudaStream_t stream,
              BwdParams& p, BwdMaps& m, int& sms) {
  int dev = 0;
  PCV_CHECK_CUDA(cudaGetDevice(&dev));
  PCV_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  int rc = attach_wait_diag(&g_wait_diag);
  if (rc != PCV_OK) return rc;

  uint8_t* ws = reinterpret_cast<uint8_t*>(a.workspace);
  p.B = a.B; p.H = a.H; p.N = a.N; p.M = a.M; p.dqk = a.dqk; p.dv = a.dv;
  p.Npad = L.Npad; p.nq = L.nq; p.nk = L.nk;
  p.q_bcast = (a.q_stride_b == 0 && a.B > 1) ? 1 : 0;
  p.scale = a.scale;
  p.scale_log2 = a.scale * kLog2e;
  p.causal = a.causal;
  p.cshift = (m_total - a.N) - m_offset;
  p.key_base = m_offset;
  p.stats = reinterpret_cast<const float*>(ws);
  set_dropout(p, a.dropout_p, a.dropout_seed);
  if (L.dq_splits > 0) {
    p.tiles_per_split = L.dq_tiles_per_split;
    p.splits = L.dq_splits;
  } else {
    dq_split(a.B * a.H * L.nq, L.nk, sms, p.tiles_per_split, p.splits);
  }

  PCV_CHECK_CUDA(cudaMemsetAsync(ws + L.off_acc, 0, L.acc_bytes, stream));
  {
    const int64_t rows = (int64_t)a.B * a.H * L.Npad;
    const int blocks = (int)((rows + 7) / 8);
    float* stats = reinterpret_cast<float*>(ws);
    if (a.dtype == PCV_BF16)
      bwd_prep_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(
          reinterpret_cast<const __nv_bfloat16*>(a.out), reinterpret_cast<const __nv_bfloat16*>(a.grad_out), a.stat_m,
          a.stat_l, stats, a.B, a.H, a.N, L.Npad, a.dv, a.o_stride_b, a.o_stride_n, a.o_stride_h, a.go_stride_b,
          a.go_stride_n, a.go_stride_h);
    else
      bwd_prep_kernel<__half><<<blocks, 256, 0, stream>>>(
          reinterpret_cast<const __half*>(a.out), reinterpret_cast<const __half*>(a.grad_out), a.stat_m, a.stat_l,
          stats, a.B, a.H, a.N, L.Npad, a.dv, a.o_stride_b, a.o_stride_n, a.o_stride_h, a.go_stride_b, a.go_stride_n,
          a.go_stride_h);
    PCV_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  if (a.pad_mask != nullptr) {
    uint32_t* bits = reinterpret_cast<uint32_t*>(ws + L.off_pad);
    rc = launch_pack_pad(a.pad_mask, a.pad_stride_b, a.B, a.M, bits, stream);
    if (rc != PCV_OK) return rc;
    p.pad_bits = bits;
    p.pad_wpr = pad_words_per_row(a.M);
  }

  const int Bq = a.q_stride_b == 0 ? 1 : a.B, ks = dq_stage_keys(a.dqk, a.dv);
  const struct {
    CUtensorMap* map;
    const void* base;
    int channels, rows, batch;
    int64_t s_row, s_h, s_b;
    int box;
  } maps[] = {
      {&m.q, a.q, a.dqk, a.N, Bq, a.q_stride_n, a.q_stride_h, a.q_stride_b, kT},
      {&m.q64, a.q, a.dqk, a.N, Bq, a.q_stride_n, a.q_stride_h, a.q_stride_b, 64},
      {&m.dout, a.grad_out, a.dv, a.N, a.B, a.go_stride_n, a.go_stride_h, a.go_stride_b, kT},
      {&m.dout64, a.grad_out, a.dv, a.N, a.B, a.go_stride_n, a.go_stride_h, a.go_stride_b, 64},
      {&m.k, a.k, a.dqk, a.M, a.B, a.k_stride_m, a.k_stride_h, a.k_stride_b, kT},
      {&m.k_dq, a.k, a.dqk, a.M, a.B, a.k_stride_m, a.k_stride_h, a.k_stride_b, ks},
      {&m.v, a.v, a.dv, a.M, a.B, a.v_stride_m, a.v_stride_h, a.v_stride_b, kT},
      {&m.v_dq, a.v, a.dv, a.M, a.B, a.v_stride_m, a.v_stride_h, a.v_stride_b, ks},
  };
  for (const auto& t : maps) {
    rc = make_tmap_4d(t.map, t.base, a.dtype, t.channels, t.rows, a.H, t.batch, t.s_row, t.s_h, t.s_b, t.box);
    if (rc != PCV_OK) return rc;
  }
  return PCV_OK;
}

// One backward of NQB x NVB boxes: the dK/dV kernel (a dV and a dK pass for the wide head dims), then the dQ kernel on
// its KS-key stages, one CTA per work item on 128-key stages and persistent on at most one CTA per SM on 64-key ones.
template <int NQB, int NVB, bool BF16>
int launch_shape(const BwdMaps& m, const BwdParams& p, int sms, cudaStream_t stream) {
  constexpr int KS = dq_stage_keys(NQB * 64, NVB * 64);
  const dim3 grid1(std::min(p.total_tiles, sms));
  constexpr int smem1 = Cfg1<NQB, NVB>::kSmem;
  int rc;
  if constexpr (wide_bwd(NQB * 64, NVB * 64)) {
    rc = launch_kernel(bwd_dkdv_kernel<NQB, NVB, BF16, kOutDV>, grid1, kThreads, smem1, 0, stream, m.q64, m.k, m.v,
                       m.dout64, p);
    if (rc == PCV_OK)
      rc = launch_kernel(bwd_dkdv_kernel<NQB, NVB, BF16, kOutDK>, grid1, kThreads, smem1, 0, stream, m.q64, m.k, m.v,
                         m.dout64, p);
  } else {
    rc = launch_kernel(bwd_dkdv_kernel<NQB, NVB, BF16>, grid1, kThreads, smem1, 0, stream, m.q64, m.k, m.v, m.dout64, p);
  }
  if (rc != PCV_OK) return rc;
  const int items = p.B * p.H * p.nq * p.splits;
  return launch_kernel(bwd_dq_kernel<NQB, NVB, BF16, KS>, dim3(KS == kT ? items : std::min(items, sms)), kThreads,
                       Cfg2<NQB, NVB, KS>::kSmem, 0, stream, m.q, m.k_dq, m.v_dq, m.dout, p);
}

template <int NQB, bool BF16>
int launch_nvb(int nvb, const BwdMaps& m, const BwdParams& p, int sms, cudaStream_t stream) {
  return nvb == 1 ? launch_shape<NQB, 1, BF16>(m, p, sms, stream)
         : nvb == 2 ? launch_shape<NQB, 2, BF16>(m, p, sms, stream)
                    : launch_shape<NQB, 3, BF16>(m, p, sms, stream);
}

// (NQB, NVB) in {1, 2, 3}^2: the 64-channel boxes of head dims up to 192
template <bool BF16>
int launch_dispatch(const BwdMaps& m, const BwdParams& p, int sms, cudaStream_t stream) {
  const int nqb = (p.dqk + 63) / 64, nvb = (p.dv + 63) / 64;
  return nqb == 1 ? launch_nvb<1, BF16>(nvb, m, p, sms, stream)
         : nqb == 2 ? launch_nvb<2, BF16>(nvb, m, p, sms, stream)
                    : launch_nvb<3, BF16>(nvb, m, p, sms, stream);
}

// the dQ partials, summed in order -> dq (dtype: bf16, fp16 or fp32) with its own strides
int launch_sum_dq(int dtype, const float* part, int nparts, void* dst, int Bq, int N, int H, int dqk, int64_t sb,
                  int64_t sn, int64_t sh, cudaStream_t stream) {
  const int64_t total = (int64_t)Bq * N * H * dqk;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, 4096);
  if (dtype == PCV_BF16)
    bwd_sum_dq_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(part, nparts, reinterpret_cast<__nv_bfloat16*>(dst), Bq,
                                                                 N, H, dqk, sb, sn, sh);
  else if (dtype == PCV_F32)
    bwd_sum_dq_kernel<float><<<blocks, 256, 0, stream>>>(part, nparts, reinterpret_cast<float*>(dst), Bq, N, H, dqk, sb,
                                                         sn, sh);
  else
    bwd_sum_dq_kernel<__half><<<blocks, 256, 0, stream>>>(part, nparts, reinterpret_cast<__half*>(dst), Bq, N, H, dqk, sb,
                                                          sn, sh);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

}  // namespace

bool attn_bwd_supported(const pcv_attn_bwd_params& a, const pcv_key_shard* shard, const char** why) {
  auto no = [&](const char* w) {
    if (why) *why = w;
    return false;
  };
  if (a.dtype != PCV_BF16 && a.dtype != PCV_F16) return no("dtype must be bf16 or fp16");
  if (a.B < 1 || a.H < 1 || a.N < 1 || a.M < 1) return no("empty problem");
  if (shard != nullptr) {
    if (shard->grad_q32 == nullptr) return no("key shard: grad_q32 is NULL");
    if (!al16(shard->grad_q32)) return no("key shard: grad_q32 must be 16-byte aligned");
    if (shard->m_offset < 0 || (int64_t)shard->m_offset + a.M > shard->m_total)
      return no("key shard: keys [m_offset, m_offset + M) outside m_total");
    // the dropout hash covers key pairs (k >> 1): an odd base would pair a shard's keys differently from the mask
    if (shard->m_offset % 2) return no("key shard: m_offset must be even");
    if (a.causal && shard->m_total < a.N) return no("key shard: causal attention needs m_total >= N");
  }
  if (a.dqk < 8 || a.dv < 8) return no("head dims must be in [8, 192]");
  if (a.dqk % 8 || a.dv % 8) return no("head dims must be multiples of 8");
  if (a.dqk > 192 || a.dv > 192) return no("head dims must be in [8, 192]");
  if (!(a.dropout_p >= 0.f && a.dropout_p < 1.f)) return no("dropout_p must be in [0, 1)");
  if (!al16(a.q) || !al16(a.k) || !al16(a.v) || !al16(a.out) || !al16(a.grad_out) || !al16(a.grad_q) ||
      !al16(a.grad_k) || !al16(a.grad_v))
    return no("tensors must be 16-byte aligned");
  const int64_t strides[] = {a.q_stride_b, a.q_stride_n, a.q_stride_h, a.k_stride_b, a.k_stride_m, a.k_stride_h,
                             a.v_stride_b, a.v_stride_m, a.v_stride_h, a.go_stride_b, a.go_stride_n, a.go_stride_h,
                             a.gk_stride_b, a.gk_stride_m, a.gk_stride_h, a.gv_stride_b, a.gv_stride_m, a.gv_stride_h};
  for (int64_t s : strides)
    if (s % 8) return no("strides must be multiples of 8 elements");
  if ((int64_t)a.M >= (int64_t)1 << 30 || (int64_t)a.N >= (int64_t)1 << 24) return no("N or M too large");
  if (const char* w = device_problem()) return no(w);
  return true;
}

int attn_bwd_workspace_bytes(const pcv_attn_bwd_params& a, const pcv_key_shard* shard, size_t* bytes) {
  PCV_REQUIRE(bytes != nullptr, PCV_ERR_INVALID, "attn_bwd_workspace_bytes: bytes is NULL");
  *bytes = bwd_layout(a, shard).total;
  return PCV_OK;
}

int launch_attn_bwd(const pcv_attn_bwd_params& a, const pcv_key_shard* shard, cudaStream_t stream) {
  const char* why = "";
  PCV_REQUIRE(attn_bwd_supported(a, shard, &why), PCV_ERR_UNSUPPORTED, "attn_bwd: %s", why);
  PCV_REQUIRE(a.stat_m != nullptr && a.stat_l != nullptr, PCV_ERR_INVALID, "attn_bwd: forward statistics are NULL");
  const BwdLayout L = bwd_layout(a, shard);
  PCV_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= L.total, PCV_ERR_INVALID,
              "attn_bwd: workspace too small (%zu < %zu)", a.workspace_bytes, L.total);
  PCV_REQUIRE((reinterpret_cast<uintptr_t>(a.workspace) & 255u) == 0, PCV_ERR_INVALID,
              "attn_bwd: workspace must be 256-byte aligned");
  BwdParams p{};
  BwdMaps m;
  int sms = 0;
  const int m_total = shard != nullptr ? shard->m_total : a.M, m_offset = shard != nullptr ? shard->m_offset : 0;
  int rc = bwd_setup(a, L, m_total, m_offset, stream, p, m, sms);
  if (rc != PCV_OK) return rc;
  const bool wide = wide_bwd(a.dqk, a.dv);
  const int Bq = a.q_stride_b == 0 ? 1 : a.B;
  p.dq32 = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(a.workspace) + (wide ? L.off_part : L.off_acc));
  if (shard != nullptr && !wide) {  // the dQ kernel reduces straight into the caller's fp32 contribution
    p.dq32 = shard->grad_q32;
    PCV_CHECK_CUDA(cudaMemsetAsync(p.dq32, 0, sizeof(float) * (size_t)Bq * a.N * a.H * a.dqk, stream));
  }
  p.dk = a.grad_k; p.dv_out = a.grad_v;
  p.dk_sb = a.gk_stride_b; p.dk_sm = a.gk_stride_m; p.dk_sh = a.gk_stride_h;
  p.dv_sb = a.gv_stride_b; p.dv_sm = a.gv_stride_m; p.dv_sh = a.gv_stride_h;
  p.total_tiles = a.B * a.H * L.nk;

  rc = a.dtype == PCV_BF16 ? launch_dispatch<true>(m, p, sms, stream) : launch_dispatch<false>(m, p, sms, stream);
  if (rc != PCV_OK) return rc;
  // dQ in the caller's dtype and strides: the partials in order, or the one fp32 buffer of the atomics up to head dim
  // 128; a key shard's grad_q32 already holds the latter and takes the former as it is, fp32 (Bq, N, H*dqk) dense
  if (shard != nullptr)
    return wide ? launch_sum_dq(PCV_F32, p.dq32, L.dq_parts, shard->grad_q32, Bq, a.N, a.H, a.dqk,
                                (int64_t)a.N * a.H * a.dqk, (int64_t)a.H * a.dqk, a.dqk, stream)
                : PCV_OK;
  return launch_sum_dq(a.dtype, p.dq32, wide ? L.dq_parts : 1, a.grad_q, Bq, a.N, a.H, a.dqk, a.gq_stride_b,
                       a.gq_stride_n, a.gq_stride_h, stream);
}

// ---- dropout mask export ---------------------------------------------------------------------------------------
int launch_dropout_mask(uint8_t* keep, int B, int H, int N, int key_begin, int key_end, float dropout_p, uint64_t seed,
                        cudaStream_t stream) {
  PCV_REQUIRE(keep != nullptr && B > 0 && H > 0 && N > 0 && key_begin >= 0 && key_end > key_begin, PCV_ERR_INVALID,
              "dropout_mask: bad arguments (B=%d H=%d N=%d keys [%d, %d))", B, H, N, key_begin, key_end);
  PCV_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, PCV_ERR_INVALID, "dropout_mask: dropout_p must be in [0, 1)");
  const DropoutRule r = dropout_rule(dropout_p, seed);
  const int W = key_end - key_begin;
  const int64_t total = (int64_t)B * H * N * W;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, 8192);
  drop_mask_kernel<<<blocks, 256, 0, stream>>>(keep, B, H, N, key_begin, W, r.thresh, r.seed_lo, r.seed_hi);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

}  // namespace pcv