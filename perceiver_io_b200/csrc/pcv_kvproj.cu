// pcv_kvproj.cu — fused K/V producer of the cross-attention module (SURVEY.md §8(f)1): LayerNorm of the
// (rows, C) input and BOTH projections in one pass over the input, on the Hopper tensor cores (wgmma).
//
// Reference (perceiver/model/core/modules.py): kv_norm(x_kv) :226, then k_proj / v_proj :114-115, i.e.
//     K = LN(x) Wk^T + bk,   V = LN(x) Wv^T + bv,   LN(x) = (x - mu) / sigma * gamma + beta.
// LayerNorm is folded around the GEMM instead of being materialised:
//     LN(x) W^T + b = rstd * ( x (gamma.W)^T  -  mu * s )  +  t,      s_n = sum_c gamma_c W_nc,
//                                                                     t_n = sum_c beta_c  W_nc + b_n
// so the kernel multiplies the RAW input tile (TMA -> shared memory -> wgmma, fp32 accumulators in registers)
// with the pre-scaled weights W' = [gamma.Wk ; gamma.Wv] and applies the per-row (mu, rstd) and per-column (s, t)
// terms in the epilogue.  s is computed from the ROUNDED W' (host side), so the mu*s cancellation is exact with
// respect to the operands the tensor core actually sees.  Row statistics come from ln_stats_kernel (one HBM pass
// over x, 8 bytes out per row) or, with FUSE, from the staged input tiles inside the GEMM.
//
// Kernel shape: CTA = 128 rows x 128 output columns, 384 threads: warpgroup 0 is the TMA producer (one lane;
// A box 128 x 64 and B box 128 x 64 per stage, SWIZZLE_128B, mbarrier ring), warpgroups 1-2 each own 64 rows.
// The column tile is the fastest grid index, so the column tiles of a row block run together and meet in L2.
// CG = 2 (cta_group = 2) runs two adjacent row blocks of the same column tile as a 2-CTA cluster: each CTA loads one
// 64-row half of every weight box and multicasts it to both, which halves the weight traffic into shared memory.
#include "pcv_common.cuh"
#include "pcv_sm90.cuh"

#include <algorithm>
#include <cstdlib>

namespace pcv {
namespace {

using namespace sm90;

constexpr int kBM = 128;   // rows per CTA
constexpr int kBN = 128;   // output columns per CTA
constexpr int kBK = 64;    // channels per pipeline stage (one 128-byte swizzle atom of 16-bit elements)
constexpr int kGemmThreads = 384;
constexpr int kStages = 6;
constexpr int kBoxBytes = 128 * 128;
constexpr int kStageBytes = 2 * kBoxBytes;
constexpr int kSmemBytes = kStages * kStageBytes + 2048 + 1024;  // ring + barriers / row statistics + alignment slack

struct GemmParams {
  const float2* stats;   // per row (mean, rstd); nullptr = no LayerNorm or statistics computed in the kernel
  const float2* col_st;  // per output column (s, t)
  void* k_out;
  void* v_out;
  const void* x;         // raw input (first element of each row: shift of the in-kernel statistics)
  int64_t x_stride, k_stride, v_stride;
  int64_t rows;
  int n_k, n_total;      // columns [0, n_k) go to K, [n_k, n_total) to V
  int num_kb;            // ceil(C / 64)
  int tiles_n;           // ceil(n_total / 128)
  int C;                 // input channels
  float eps;             // LayerNorm epsilon of the in-kernel statistics
};

// e4m3 outputs of kvproj_fp8_kernel (its own argument, so that kvproj_kernel's parameters are unchanged): column n is
// multiplied by inv_scale[n] and rounded to e4m3 (satfinite); K columns go to k_out as e4m3 rows, V columns to vt_out
// transposed, (B, H, dv, keys), row r being key r % keys_per_batch of batch row r / keys_per_batch (a 128-row tile
// may cross a batch boundary)
struct Fp8Out {
  const float* inv_scale;
  void* vt_out;
  int64_t vt_sb, vt_sh, vt_sc;
  int64_t keys_per_batch;
  int v_dv;              // channels per V head
};

struct GemmSmem {
  uint64_t full[kStages], empty[kStages];
  float2 row_st[kBM];
};

// The body of kvproj_kernel (F8 = false: 16-bit outputs) and kvproj_fp8_kernel (F8 = true: e4m3 outputs, see Fp8Out)
template <bool BF16, bool FUSE, int CG, bool F8>
__device__ __forceinline__ void kvproj_body(const CUtensorMap& tx, const CUtensorMap& tw, const GemmParams& p,
                                            const Fp8Out& f8) {
  static_assert(!F8 || CG == 1, "the e4m3 producer runs one CTA per tile");
  using T = typename std::conditional<BF16, __nv_bfloat16, __half>::type;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  GemmSmem& sh = *reinterpret_cast<GemmSmem*>(smem + kStages * kStageBytes);
  const int wg = threadIdx.x / 128;
  const uint32_t rank = CG == 2 ? cluster_ctarank() : 0u;
  const int64_t cid = blockIdx.x / CG;
  const int n_blk = (int)(cid % p.tiles_n);
  const int64_t m_blk = (cid / p.tiles_n) * CG + rank;
  const int64_t row0 = m_blk * kBM;
  const int col0 = n_blk * kBN;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&sh.full[s], 1);
      mbar_init(&sh.empty[s], CG == 2 ? 16 : 8);  // one arrive per consumer warp (of both CTAs of a pair)
    }
    fence_mbar_init();
  }
  if (CG == 2)
    cluster_sync_all();
  else
    __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < p.num_kb; ++kb) {
        const int s = kb % kStages;
        mbar_wait(&sh.empty[s], ((kb / kStages) & 1) ^ 1, 11);
        mbar_arrive_expect_tx(&sh.full[s], kStageBytes);
        tma_load_2d(smem + s * kStageBytes, &tx, &sh.full[s], kb * kBK, (int)row0);
        if (CG == 2)
          tma_load_2d_mc(smem + s * kStageBytes + kBoxBytes + rank * (kBoxBytes / 2), &tw, &sh.full[s], kb * kBK,
                         col0 + 64 * (int)rank, 0x3);
        else
          tma_load_2d(smem + s * kStageBytes + kBoxBytes, &tw, &sh.full[s], kb * kBK, col0);
      }
    }
    if (CG == 2) {
      __syncwarp();
      cluster_sync_all();  // the peer may still multicast into / arrive on this CTA's shared memory until here
    }
    return;
  }

  reg_alloc<232>();
  const int cw = wg - 1;
  const int tid = threadIdx.x - 128 * wg;
  const int warp = tid >> 5, lane = tid & 31;
  const int rloc = 64 * cw + 16 * warp + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t base = smem_u32(smem);
  // in-kernel statistics: two threads per row, each reads half of the row's 128-byte line of every A box;
  // shifted sums (by the row's first element) keep the one-pass variance free of cancellation
  const int srow = 64 * cw + (tid >> 1), shalf = tid & 1;
  float x0 = 0.f, s1 = 0.f, s2 = 0.f;
  if (FUSE && row0 + srow < p.rows)
    x0 = Elem<T>::to_f(*(reinterpret_cast<const T*>(p.x) + (row0 + srow) * p.x_stride));

  float acc[64];
  for (int kb = 0; kb < p.num_kb; ++kb) {
    const int s = kb % kStages;
    mbar_wait(&sh.full[s], (kb / kStages) & 1, 12);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      wgmma_ss<128, BF16>(acc, make_desc(base + s * kStageBytes + cw * 64 * 128 + kk * 32),
                          make_desc(base + s * kStageBytes + kBoxBytes + kk * 32), (kb | kk) != 0);
    wgmma_commit();
    if (FUSE) {
      const uint8_t* line = smem + s * kStageBytes + srow * 128;
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        const int lc = shalf * 4 + ch;  // logical 16-byte chunk of the row
        const uint4 u = *reinterpret_cast<const uint4*>(line + ((lc ^ (srow & 7)) * 16));
        const typename Elem<T>::T2* h2 = reinterpret_cast<const typename Elem<T>::T2*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int c = kb * kBK + lc * 8 + 2 * e;
          const float2 f = Elem<T>::to_f2(h2[e]);
          if (c < p.C) {
            const float d = f.x - x0;
            s1 += d;
            s2 = fmaf(d, d, s2);
          }
          if (c + 1 < p.C) {
            const float d = f.y - x0;
            s1 += d;
            s2 = fmaf(d, d, s2);
          }
        }
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (CG == 2) warp_arrive_pair(&sh.empty[s]);
    else warp_arrive(&sh.empty[s]);
  }

  if (FUSE) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
    if (shalf == 0) {
      const float inv_c = 1.f / (float)p.C;
      const float dm = s1 * inv_c;
      const float var = fmaxf(s2 * inv_c - dm * dm, 0.f);
      // a constant row (every shifted element is 0) has x_hat == 0: rstd = 0 makes the epilogue write t exactly
      // instead of amplifying the fp32 residue of x.w' - mean * s by eps^-1/2
      sh.row_st[srow] = make_float2(x0 + dm, var > 0.f ? rsqrtf(var + p.eps) : 0.f);
    }
    asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
  }

  // given statistics of eps = p.eps > 0: rstd == 1 / sqrtf(0 + eps), the value pcv_ln_stats writes for a zero-variance
  // row, marks x_hat == 0 (the statistics themselves stay as pcv_ln_linear_bwd reads them)
  const float rstd_flat = p.eps > 0.f ? 1.f / sqrtf(p.eps) : -1.f;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int64_t row = row0 + rloc + 8 * r;
    if (row >= p.rows) continue;
    float2 st = make_float2(0.f, 1.f);
    const bool ln = FUSE || p.stats != nullptr;
    if (FUSE) {
      st = sh.row_st[rloc + 8 * r];
    } else if (p.stats != nullptr) {
      st = p.stats[row];
      if (st.y == rstd_flat) st.y = 0.f;
    }
#pragma unroll
    for (int g = 0; g < 16; ++g) {
      const int n = col0 + 8 * g + cq;
      if (n >= p.n_total) continue;
      const float2 c0 = p.col_st[n], c1 = p.col_st[n + 1];
      float a0 = acc[4 * g + 2 * r], a1 = acc[4 * g + 2 * r + 1];
      if (ln) {
        a0 = st.y * (a0 - st.x * c0.x);
        a1 = st.y * (a1 - st.x * c1.x);
      }
      if constexpr (F8) {
        const uint32_t w8 = cvt_e4m3x2((a0 + c0.y) * f8.inv_scale[n], (a1 + c1.y) * f8.inv_scale[n + 1]);
        if (n < p.n_k) {
          *reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(p.k_out) + row * p.k_stride + n) = (uint16_t)w8;
        } else {  // channels c and c + 1 of one head (dv is even): two rows of V^T, key m
          const int c = n - p.n_k, h = c / f8.v_dv;
          const int64_t b = row / f8.keys_per_batch, m = row - b * f8.keys_per_batch;
          uint8_t* dst = reinterpret_cast<uint8_t*>(f8.vt_out) + b * f8.vt_sb + h * f8.vt_sh +
                         (int64_t)(c - h * f8.v_dv) * f8.vt_sc + m;
          dst[0] = (uint8_t)(w8 & 0xffu);
          dst[f8.vt_sc] = (uint8_t)(w8 >> 8);
        }
      } else {
        const uint32_t w = pack2(a0 + c0.y, a1 + c1.y, BF16);
        if (n < p.n_k)
          *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(p.k_out) + row * p.k_stride + n) = w;
        else
          *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(p.v_out) + row * p.v_stride + (n - p.n_k)) = w;
      }
    }
  }
  if (CG == 2) cluster_sync_all();
}

template <bool BF16, bool FUSE, int CG>
__global__ void __launch_bounds__(kGemmThreads, 1)
kvproj_kernel(const __grid_constant__ CUtensorMap tx, const __grid_constant__ CUtensorMap tw, const GemmParams p) {
  kvproj_body<BF16, FUSE, CG, false>(tx, tw, p, Fp8Out{});
}

// LayerNorm-folded projection with e4m3 outputs (pcv_kv_project_fp8): a separate kernel, one CTA per tile
template <bool BF16, bool FUSE>
__global__ void __launch_bounds__(kGemmThreads, 1)
kvproj_fp8_kernel(const __grid_constant__ CUtensorMap tx, const __grid_constant__ CUtensorMap tw, const GemmParams p,
                  const Fp8Out f8) {
  kvproj_body<BF16, FUSE, 1, true>(tx, tw, p, f8);
}


// --------------------------------------------------------------------------------------------------
// LayerNorm row statistics: one warp per row, (mean, 1/sqrt(var + eps)) with the biased variance of
// nn.LayerNorm, two-pass in fp32 (mean first, then the centred second moment: no cancellation however large
// |mean| / sigma is).  HBM-bound: rows * C * 2 bytes in, 8 bytes per row out.  Rows of up to 2048 16-bit
// channels (a multiple of 256) are held in registers between the passes (NCH 16-byte chunks per lane, all loads
// of a row in flight at once, two rows per warp iteration); other widths re-read the row from L1.
// --------------------------------------------------------------------------------------------------
template <typename T, int NCH>
__global__ void __launch_bounds__(256) ln_stats_reg_kernel(const T* __restrict__ x, int64_t stride_row, int64_t rows,
                                                            float eps, float2* __restrict__ stats) {
  constexpr int C = NCH * 256;
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t w0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  for (int64_t r = w0 * 2; r < rows; r += warps * 2) {
    uint4 u[2][NCH];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const bool live = r + k < rows;
      const uint4* xr = reinterpret_cast<const uint4*>(x + (r + k) * stride_row);
#pragma unroll
      for (int i = 0; i < NCH; ++i) u[k][i] = live ? __ldcs(xr + lane + 32 * i) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        const typename Elem<T>::T2* h = reinterpret_cast<const typename Elem<T>::T2*>(&u[k][i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = Elem<T>::to_f2(h[j]);
          sum += f.x + f.y;
        }
      }
      // divided, not multiplied by RN(1 / C): for C = 1792 that reciprocal is off by more than 2^-25, so a constant
      // row's mean would land one ulp off its value, give var > 0 and escape the producer's zero-variance rule
      const float mean = warp_sum(sum) / (float)C;
      float sq = 0.f;
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        const typename Elem<T>::T2* h = reinterpret_cast<const typename Elem<T>::T2*>(&u[k][i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = Elem<T>::to_f2(h[j]);
          const float d0 = f.x - mean, d1 = f.y - mean;
          sq = fmaf(d0, d0, sq);
          sq = fmaf(d1, d1, sq);
        }
      }
      const float var = warp_sum(sq) * (1.f / (float)C);
      if (lane == 0 && r + k < rows) stats[r + k] = make_float2(mean, 1.f / sqrtf(var + eps));
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) ln_stats_kernel(const T* __restrict__ x, int64_t stride_row, int64_t rows, int C,
                                                        float eps, float2* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += warps) {
    const T* xr = x + r * stride_row;
    const bool vec = ((reinterpret_cast<uintptr_t>(xr) & 15) == 0) && (C % 8 == 0);
    float sum = 0.f;
    if (vec) {
      for (int c = lane * 8; c < C; c += 256) {
        const uint4 u = *reinterpret_cast<const uint4*>(xr + c);
        const typename Elem<T>::T2* h = reinterpret_cast<const typename Elem<T>::T2*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = Elem<T>::to_f2(h[i]);
          sum += f.x + f.y;
        }
      }
    } else {
      for (int c = lane; c < C; c += 32) sum += Elem<T>::to_f(xr[c]);
    }
    const float mean = warp_sum(sum) / (float)C;
    float sq = 0.f;
    if (vec) {
      for (int c = lane * 8; c < C; c += 256) {
        const uint4 u = *reinterpret_cast<const uint4*>(xr + c);
        const typename Elem<T>::T2* h = reinterpret_cast<const typename Elem<T>::T2*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = Elem<T>::to_f2(h[i]);
          const float d0 = f.x - mean, d1 = f.y - mean;
          sq = fmaf(d0, d0, sq);
          sq = fmaf(d1, d1, sq);
        }
      }
    } else {
      for (int c = lane; c < C; c += 32) {
        const float d = Elem<T>::to_f(xr[c]) - mean;
        sq = fmaf(d, d, sq);
      }
    }
    const float var = warp_sum(sq) / (float)C;
    if (lane == 0) stats[r] = make_float2(mean, 1.f / sqrtf(var + eps));
  }
}

template <typename T>
int launch_ln_stats_t(const pcv_ln_stats_params& p, cudaStream_t stream) {
  const T* x = reinterpret_cast<const T*>(p.x);
  float2* st = reinterpret_cast<float2*>(p.stats);
  const bool reg_ok = (p.C % 256 == 0) && p.C <= 2048 && (p.x_stride_row % 8 == 0) &&
                      ((reinterpret_cast<uintptr_t>(p.x) & 15) == 0);
  if (reg_ok) {
    const int blocks = (int)std::min<int64_t>((p.rows + 15) / 16, 132 * 8);
#define PCV_LN_CASE(N)                                                                               \
  case N:                                                                                            \
    ln_stats_reg_kernel<T, N><<<blocks, 256, 0, stream>>>(x, p.x_stride_row, p.rows, p.eps, st);     \
    break;
    switch (p.C / 256) {
      PCV_LN_CASE(1) PCV_LN_CASE(2) PCV_LN_CASE(3) PCV_LN_CASE(4) PCV_LN_CASE(5) PCV_LN_CASE(6) PCV_LN_CASE(7)
      PCV_LN_CASE(8)
    }
#undef PCV_LN_CASE
  } else {
    const int blocks = (int)std::min<int64_t>((p.rows + 7) / 8, 132 * 8);
    ln_stats_kernel<T><<<blocks, 256, 0, stream>>>(x, p.x_stride_row, p.rows, p.C, p.eps, st);
  }
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

template <bool BF16, bool FUSE, int CG, bool F8 = false>
int launch_gemm(const CUtensorMap& tx, const CUtensorMap& tw, const GemmParams& gp, cudaStream_t stream,
                const Fp8Out& f8 = Fp8Out{}) {
  const int64_t m_blocks = (gp.rows + kBM * CG - 1) / (kBM * CG) * CG;  // whole pairs; a pair's spare block is all padding
  const int64_t tiles = m_blocks * gp.tiles_n;
  PCV_REQUIRE(tiles <= 0x7fffffff, PCV_ERR_UNSUPPORTED, "kv_project: %lld tiles exceed the grid limit", (long long)tiles);
  prof_mark_begin(stream);
  int rc;
  if constexpr (F8)
    rc = launch_kernel(kvproj_fp8_kernel<BF16, FUSE>, dim3((unsigned)tiles), kGemmThreads, kSmemBytes, 0, stream, tx, tw,
                       gp, f8);
  else
    rc = launch_kernel(kvproj_kernel<BF16, FUSE, CG>, dim3((unsigned)tiles), kGemmThreads, kSmemBytes, CG, stream,
                       tx, tw, gp);
  prof_mark_end(stream);
  return rc;
}

}  // namespace

int launch_ln_stats(const pcv_ln_stats_params& p, cudaStream_t stream) {
  PCV_REQUIRE(p.x != nullptr && p.stats != nullptr, PCV_ERR_INVALID, "ln_stats: NULL pointer");
  PCV_REQUIRE(p.rows >= 0 && p.C >= 1, PCV_ERR_INVALID, "ln_stats: rows=%lld C=%d", (long long)p.rows, p.C);
  PCV_REQUIRE(p.dtype == PCV_BF16 || p.dtype == PCV_F16, PCV_ERR_INVALID, "ln_stats: dtype must be bf16/fp16");
  if (p.rows == 0) return PCV_OK;
  return p.dtype == PCV_BF16 ? launch_ln_stats_t<__nv_bfloat16>(p, stream) : launch_ln_stats_t<__half>(p, stream);
}

bool kv_project_supported(const pcv_kvproj_params& p, const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (p.dtype != PCV_BF16 && p.dtype != PCV_F16) return fail("dtype must be bf16 or fp16");
  if (p.C < 8 || (p.C % 8)) return fail("input channels must be a multiple of 8 (16-byte TMA strides)");
  if (p.n_k < 0 || p.n_v < 0 || p.n_k + p.n_v < 1) return fail("no output columns");
  if ((p.n_k % 64) != 0) return fail("K width must be a multiple of 64");
  if ((p.n_v % 8) != 0) return fail("V width must be a multiple of 8");
  if (!al16(p.x) || !al16(p.w) || (p.n_k && !al16(p.k_out)) || (p.n_v && !al16(p.v_out)))
    return fail("x / w / k_out / v_out must be 16-byte aligned");
  if ((p.x_stride_row % 8) || (p.k_stride_row % 8) || (p.v_stride_row % 8)) return fail("row strides must be multiples of 8 elements");
  if (p.rows < 1 || p.rows > (int64_t)0x7fffff00) return fail("row count out of range");
  if (p.cta_group < 0 || p.cta_group > 2) return fail("cta_group must be 0, 1 or 2");
  if (const char* w = device_problem()) return fail(w);
  return true;
}

bool kv_project_fp8_supported(const pcv_kvproj_params& p, const pcv_kvproj_fp8& f, const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (f.inv_scale == nullptr) return fail("inv_scale is NULL");
  if (p.cta_group == 2) return fail("the e4m3 producer runs one CTA per tile (cta_group 0 or 1)");
  if (p.n_k % 16) return fail("K width must be a multiple of 16");
  if (p.n_v > 0) {
    if (f.vt_out == nullptr) return fail("vt_out is NULL");
    if (f.v_head_dim < 16 || (f.v_head_dim % 16) || (p.n_v % f.v_head_dim)) return fail("v_head_dim must be a multiple of 16 dividing n_v");
    if (f.keys_per_batch < 1 || (p.rows % f.keys_per_batch)) return fail("keys_per_batch must divide the row count");
    if (f.vt_stride_c < f.keys_per_batch || (f.vt_stride_c % 16) || (f.vt_stride_h % 16) || (f.vt_stride_b % 16))
      return fail("v^T strides must be multiples of 16 bytes and cover keys_per_batch keys");
  }
  if (p.n_k > 0 && (p.k_stride_row % 16)) return fail("the e4m3 K row stride must be a multiple of 16 bytes");
  // the 16-bit conditions of pcv_kv_project (v_out / v_stride_row are unused here)
  pcv_kvproj_params q = p;
  q.v_out = q.k_out != nullptr ? q.k_out : const_cast<void*>(q.x);
  q.v_stride_row = 0;
  q.k_stride_row = 0;
  return kv_project_supported(q, why);
}

int launch_kv_project_fp8(const pcv_kvproj_params& p, const pcv_kvproj_fp8& f, cudaStream_t stream) {
  const char* why = "";
  PCV_REQUIRE(p.x && p.w && p.col_st, PCV_ERR_INVALID, "kv_project_fp8: NULL pointer");
  PCV_REQUIRE(kv_project_fp8_supported(p, f, &why), PCV_ERR_UNSUPPORTED, "kv_project_fp8: %s", why);
  const int n_total = p.n_k + p.n_v;
  GemmParams gp{};
  gp.stats = reinterpret_cast<const float2*>(p.row_stats);
  gp.col_st = reinterpret_cast<const float2*>(p.col_st);
  gp.k_out = p.k_out;
  gp.x = p.x;
  gp.x_stride = p.x_stride_row;
  gp.k_stride = p.k_stride_row;
  gp.rows = p.rows;
  gp.n_k = p.n_k;
  gp.n_total = n_total;
  gp.num_kb = (p.C + kBK - 1) / kBK;
  gp.tiles_n = (n_total + kBN - 1) / kBN;
  gp.C = p.C;
  gp.eps = p.ln_eps;
  Fp8Out f8{};
  f8.inv_scale = f.inv_scale;
  f8.vt_out = f.vt_out;
  f8.vt_sb = f.vt_stride_b; f8.vt_sh = f.vt_stride_h; f8.vt_sc = f.vt_stride_c;
  f8.keys_per_batch = f.keys_per_batch > 0 ? f.keys_per_batch : p.rows;
  f8.v_dv = f.v_head_dim > 0 ? f.v_head_dim : 16;
  const bool fuse = p.row_stats == nullptr && p.ln_eps > 0.f;
  int rc = attach_wait_diag(&g_wait_diag);
  if (rc != PCV_OK) return rc;
  CUtensorMap tx, tw;
  rc = make_tmap_2d(&tx, p.x, p.dtype, p.C, p.rows, p.x_stride_row, kBM);
  if (rc != PCV_OK) return rc;
  rc = make_tmap_2d(&tw, p.w, p.dtype, p.C, n_total, p.C, kBN);
  if (rc != PCV_OK) return rc;
  const bool bf = p.dtype == PCV_BF16;
  if (fuse)
    return bf ? launch_gemm<true, true, 1, true>(tx, tw, gp, stream, f8) : launch_gemm<false, true, 1, true>(tx, tw, gp, stream, f8);
  return bf ? launch_gemm<true, false, 1, true>(tx, tw, gp, stream, f8) : launch_gemm<false, false, 1, true>(tx, tw, gp, stream, f8);
}

int launch_kv_project(const pcv_kvproj_params& p, cudaStream_t stream) {
  const char* why = "";
  PCV_REQUIRE(p.x && p.w && p.col_st, PCV_ERR_INVALID, "kv_project: NULL pointer");
  PCV_REQUIRE(kv_project_supported(p, &why), PCV_ERR_UNSUPPORTED, "kv_project: %s", why);
  const int n_total = p.n_k + p.n_v;
  GemmParams gp{};
  gp.stats = reinterpret_cast<const float2*>(p.row_stats);
  gp.col_st = reinterpret_cast<const float2*>(p.col_st);
  gp.k_out = p.k_out;
  gp.v_out = p.v_out;
  gp.x = p.x;
  gp.x_stride = p.x_stride_row;
  gp.k_stride = p.k_stride_row;
  gp.v_stride = p.v_stride_row;
  gp.rows = p.rows;
  gp.n_k = p.n_k;
  gp.n_total = n_total;
  gp.num_kb = (p.C + kBK - 1) / kBK;
  gp.tiles_n = (n_total + kBN - 1) / kBN;
  gp.C = p.C;
  gp.eps = p.ln_eps;
  const bool fuse = p.row_stats == nullptr && p.ln_eps > 0.f;

  int rc = attach_wait_diag(&g_wait_diag);
  if (rc != PCV_OK) return rc;
  CUtensorMap tx, tw;
  rc = make_tmap_2d(&tx, p.x, p.dtype, p.C, p.rows, p.x_stride_row, kBM);
  if (rc != PCV_OK) return rc;
  // one CTA per tile by default; cta_group = 2 asks for the 2-CTA clusters (each CTA loads half of the weight box)
  const int cg = p.cta_group == 2 ? 2 : 1;
  rc = make_tmap_2d(&tw, p.w, p.dtype, p.C, n_total, p.C, kBN / cg);
  if (rc != PCV_OK) return rc;
  const bool bf = p.dtype == PCV_BF16;
#define PCV_GEMM_CASE(G)                                                                                   \
  if (fuse) return bf ? launch_gemm<true, true, G>(tx, tw, gp, stream) : launch_gemm<false, true, G>(tx, tw, gp, stream); \
  return bf ? launch_gemm<true, false, G>(tx, tw, gp, stream) : launch_gemm<false, false, G>(tx, tw, gp, stream);
  if (cg == 2) {
    PCV_GEMM_CASE(2)
  }
  PCV_GEMM_CASE(1)
#undef PCV_GEMM_CASE
}

}  // namespace pcv
