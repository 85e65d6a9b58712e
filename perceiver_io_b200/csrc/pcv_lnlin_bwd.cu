// pcv_lnlin_bwd.cu — backward of the LayerNorm -> Linear chain of the fused producer (pcv_kvproj.cu), for training
// through kv_norm -> k_proj / v_proj, q_norm -> q_proj and norm -> q/k/v_proj.
//
// With x_hat = (x - mean) * rstd, y = x_hat * gamma + beta, out = y W^T + b and the incoming gradient G (rows, n):
//     db = G^T 1,   P = G^T x_hat,   dW = P diag(gamma) + db beta^T,
//     dy = G W,     dgamma = sum_rows dy * x_hat,   dbeta = sum_rows dy,
//     dx = rstd * (dx_hat - (a + x_hat * b) / C),   dx_hat = gamma * dy,   a = sum_c dx_hat,   b = sum_c dx_hat * x_hat.
// y is never stored: both GEMMs rebuild x_hat from x and the row statistics.  b comes from dy (not from the saved
// outputs, which hold the folded bias), and dW multiplies a 16-bit x_hat rounded AFTER normalising (not x with a
// rank-1 mean correction, which cancels badly for rows with a large mean).
//
// Kernels (CTA = 384 threads: warpgroup 0 is the TMA producer, warpgroups 1-2 each own 64 rows of a 128 x 128 tile):
//   lnlin_dx_kernel    dy = G W: A = G boxes (K-major), B = W boxes (MN-major, as stored).  The epilogue forms x_hat
//                      from x and the statistics, writes dx_hat (rounded) to grad_x, and fp32 partials: per (row,
//                      128-column tile) (sum dx_hat, sum dx_hat * x_hat), per (128-row block, column) (sum dy * x_hat,
//                      sum dy).
//   lnlin_dx_fixup_kernel  dx = rstd * (dx_hat - (a + x_hat b) / C) in place, a and b summed in column-tile order.
//   lnlin_dw_kernel    P^T = x_hat^T G: A from registers (x tile by ldmatrix.trans, normalised, rounded to 16 bits),
//                      B = G boxes (MN-major).  The rows are split by a plan fixed for 132 SMs into fp32 partials; the
//                      CTAs of the first channel tile also sum the columns of G (db partials) in row order.
//   lnlin_dw_finish_kernel / lnlin_colsum_kernel  sum the partials in index order and write the parameter gradients.
// No atomics: every gradient is bitwise reproducible.
#include "pcv_common.cuh"
#include "pcv_sm90.cuh"

#include <algorithm>

namespace pcv {
namespace {

using namespace sm90;

constexpr int kBM = 128;          // dx: rows per CTA; dw: channels per CTA
constexpr int kBN = 128;          // dx: channels per CTA; dw: output columns per CTA
constexpr int kBK = 64;           // reduction step per pipeline stage
constexpr int kThreads = 384;
constexpr int kStages = 6;
constexpr int kStageBytes = 32768;
constexpr int kSmemBytes = kStages * kStageBytes + 256 + 8 * kBN * 8 + 1024;  // ring, barriers, column sums, alignment
// SMs of an H100 SXM.  The dW kernel runs one CTA per SM (its ring takes most of the shared memory), and the row-split
// plan aims at about 2 x kWorkers CTAs: two waves.
constexpr int kWorkers = 132;
constexpr int kMaxSplits = 32;

struct Plan {
  int64_t rows, m_blocks, kb_rows;
  int C, n_k, n_v, n_total, tiles_c, tiles_n, splits;
  size_t off_col, off_p, off_db, bytes;
};

size_t up256(size_t b) { return (b + 255) / 256 * 256; }

// Fixed by (rows, C, n_k, n_v) alone, so the workspace size does not depend on the device
Plan make_plan(int64_t rows, int C, int n_k, int n_v) {
  Plan pl{};
  pl.rows = rows;
  pl.C = C;
  pl.n_k = n_k;
  pl.n_v = n_v;
  pl.n_total = n_k + n_v;
  pl.m_blocks = (rows + kBM - 1) / kBM;
  pl.kb_rows = (rows + kBK - 1) / kBK;
  pl.tiles_c = (C + kBN - 1) / kBN;
  pl.tiles_n = (pl.n_total + kBN - 1) / kBN;
  const int tiles = pl.tiles_c * pl.tiles_n;
  pl.splits = (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)(2 * kWorkers / tiles), (int64_t)kMaxSplits, pl.kb_rows}));
  const size_t row_bytes = (size_t)pl.tiles_c * rows * 8;
  const size_t col_bytes = (size_t)pl.m_blocks * C * 8;
  const size_t p_bytes = (size_t)pl.splits * pl.n_total * C * 4;
  const size_t db_bytes = (size_t)pl.splits * pl.n_total * 4;
  pl.off_col = up256(row_bytes);
  pl.off_p = pl.off_col + up256(col_bytes);
  pl.off_db = pl.off_p + up256(p_bytes);
  pl.bytes = pl.off_db + up256(db_bytes);
  return pl;
}

struct DxParams {
  const void* x;
  const float2* stats;
  const void* gamma;     // nullptr = 1
  void* grad_x;          // (rows, C) contiguous: dx_hat; nullptr = not needed
  float2* row_part;      // (tiles_c, rows)
  float2* col_part;      // (m_blocks, C); nullptr = not needed
  int64_t x_stride, rows;
  int C, kb_k, num_kb, tiles_c;
};

struct DwParams {
  const float2* stats;
  float* p_part;         // (splits, n_total, C)
  float* db_part;        // (splits, n_total)
  int64_t rows, kb_rows;
  int C, n_k, n_v, n_total, tiles_c, tiles_n, splits;
};

__device__ __forceinline__ uint8_t* aligned_smem() {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
}

__device__ __forceinline__ void init_ring(uint64_t* full, uint64_t* empty) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);  // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
}

// dy = G W for a 128-row x 128-channel tile; stage = G box (128 rows x 64 columns of n) + W boxes (64 rows of n x
// 2 x 64 channels)
template <bool BF16>
__global__ void __launch_bounds__(kThreads, 1)
lnlin_dx_kernel(const __grid_constant__ CUtensorMap tgk, const __grid_constant__ CUtensorMap tgv,
                const __grid_constant__ CUtensorMap tw, const DxParams p) {
  using T = typename std::conditional<BF16, __nv_bfloat16, __half>::type;
  using T2 = typename Elem<T>::T2;
  uint8_t* smem = aligned_smem();
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty = full + kStages;
  float2* colsm = reinterpret_cast<float2*>(smem + kStages * kStageBytes + 256);  // [8 warps][128 channels]
  const int wg = threadIdx.x / 128;
  const int n_blk = (int)(blockIdx.x % p.tiles_c);
  const int64_t m_blk = blockIdx.x / p.tiles_c;
  const int row0 = (int)(m_blk * kBM);
  const int col0 = n_blk * kBN;
  init_ring(full, empty);

  if (wg == 0) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < p.num_kb; ++kb) {
        const int s = kb % kStages;
        uint8_t* st = smem + s * kStageBytes;
        mbar_wait(&empty[s], ((kb / kStages) & 1) ^ 1, 51);
        mbar_arrive_expect_tx(&full[s], kStageBytes);
        if (kb < p.kb_k) tma_load_2d(st, &tgk, &full[s], kb * kBK, row0);
        else tma_load_2d(st, &tgv, &full[s], (kb - p.kb_k) * kBK, row0);
        tma_load_2d(st + 16384, &tw, &full[s], col0, kb * kBK);
        tma_load_2d(st + 16384 + 8192, &tw, &full[s], col0 + 64, kb * kBK);
      }
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

  float acc[64];
  for (int kb = 0; kb < p.num_kb; ++kb) {
    const int s = kb % kStages;
    mbar_wait(&full[s], (kb / kStages) & 1, 52);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      wgmma_ss_bmn_n128<BF16>(acc, make_desc(base + s * kStageBytes + cw * 64 * 128 + kk * 32),
                              make_desc(base + s * kStageBytes + 16384 + kk * 2048, 8192, 1024), (kb | kk) != 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc);
    warp_arrive(&empty[s]);
  }

  const bool want_x = p.grad_x != nullptr, want_col = p.col_part != nullptr;
  const T* x = reinterpret_cast<const T*>(p.x);
  const T* gamma = reinterpret_cast<const T*>(p.gamma);
  T* gx = reinterpret_cast<T*>(p.grad_x);
  float2 st[2];
  bool live[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int64_t row = (int64_t)row0 + rloc + 8 * r;
    live[r] = row < p.rows;
    st[r] = live[r] ? p.stats[row] : make_float2(0.f, 0.f);
  }
  float ra[2] = {0.f, 0.f}, rb[2] = {0.f, 0.f};
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    const int c = col0 + 8 * g + cq;
    float cx0 = 0.f, cx1 = 0.f, cy0 = 0.f, cy1 = 0.f;  // this thread's rows of columns c, c + 1
    if (c < p.C) {
      float g0 = 1.f, g1 = 1.f;
      if (gamma != nullptr) {
        const float2 f = Elem<T>::to_f2(*reinterpret_cast<const T2*>(gamma + c));
        g0 = f.x;
        g1 = f.y;
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (!live[r]) continue;
        const int64_t row = (int64_t)row0 + rloc + 8 * r;
        const float2 xf = Elem<T>::to_f2(*reinterpret_cast<const T2*>(x + row * p.x_stride + c));
        const float xh0 = (xf.x - st[r].x) * st[r].y, xh1 = (xf.y - st[r].x) * st[r].y;
        const float dy0 = acc[4 * g + 2 * r], dy1 = acc[4 * g + 2 * r + 1];
        cx0 = fmaf(dy0, xh0, cx0);
        cx1 = fmaf(dy1, xh1, cx1);
        cy0 += dy0;
        cy1 += dy1;
        if (want_x) {
          const float d0 = g0 * dy0, d1 = g1 * dy1;
          *reinterpret_cast<uint32_t*>(gx + row * p.C + c) = pack2(d0, d1, BF16);
          ra[r] += d0 + d1;
          rb[r] = fmaf(d0, xh0, fmaf(d1, xh1, rb[r]));
        }
      }
    }
    if (want_col) {
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        cx0 += __shfl_xor_sync(0xffffffffu, cx0, o);
        cx1 += __shfl_xor_sync(0xffffffffu, cx1, o);
        cy0 += __shfl_xor_sync(0xffffffffu, cy0, o);
        cy1 += __shfl_xor_sync(0xffffffffu, cy1, o);
      }
      if (lane < 4) {
        colsm[(4 * cw + warp) * kBN + 8 * g + cq] = make_float2(cx0, cy0);
        colsm[(4 * cw + warp) * kBN + 8 * g + cq + 1] = make_float2(cx1, cy1);
      }
    }
  }
  if (want_x) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float a = ra[r], b = rb[r];
      a += __shfl_xor_sync(0xffffffffu, a, 1);
      b += __shfl_xor_sync(0xffffffffu, b, 1);
      a += __shfl_xor_sync(0xffffffffu, a, 2);
      b += __shfl_xor_sync(0xffffffffu, b, 2);
      const int64_t row = (int64_t)row0 + rloc + 8 * r;
      if ((lane & 3) == 0 && live[r]) p.row_part[(int64_t)n_blk * p.rows + row] = make_float2(a, b);
    }
  }
  if (want_col) {
    named_bar_sync<1, 256>();
    const int t = threadIdx.x - 128;
    if (t < kBN && col0 + t < p.C) {
      float2 s = make_float2(0.f, 0.f);
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        s.x += colsm[w * kBN + t].x;
        s.y += colsm[w * kBN + t].y;
      }
      p.col_part[m_blk * p.C + col0 + t] = s;
    }
  }
}

// dx = rstd * (dx_hat - (a + x_hat * b) / C) over grad_x in place; one warp per row
template <typename T>
__global__ void __launch_bounds__(256) lnlin_dx_fixup_kernel(const T* __restrict__ x, int64_t x_stride,
                                                             const float2* __restrict__ stats,
                                                             const float2* __restrict__ row_part, int tiles_c,
                                                             T* __restrict__ gx, int64_t rows, int C) {
  using T2 = typename Elem<T>::T2;
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const float inv_c = 1.f / (float)C;
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += warps) {
    float a = 0.f, b = 0.f;
    for (int t = 0; t < tiles_c; ++t) {
      const float2 v = row_part[(int64_t)t * rows + r];
      a += v.x;
      b += v.y;
    }
    const float2 st = stats[r];
    for (int c = lane * 8; c < C; c += 256) {
      const uint4 xv = *reinterpret_cast<const uint4*>(x + r * x_stride + c);
      uint4 dv = *reinterpret_cast<const uint4*>(gx + r * C + c);
      const T2* xh = reinterpret_cast<const T2*>(&xv);
      uint32_t* d = reinterpret_cast<uint32_t*>(&dv);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 xf = Elem<T>::to_f2(xh[i]);
        const float2 df = Elem<T>::to_f2(*reinterpret_cast<const T2*>(&d[i]));
        const float h0 = (xf.x - st.x) * st.y, h1 = (xf.y - st.x) * st.y;
        d[i] = pack2(st.y * (df.x - (a + h0 * b) * inv_c), st.y * (df.y - (a + h1 * b) * inv_c),
                     std::is_same<T, __nv_bfloat16>::value);
      }
      *reinterpret_cast<uint4*>(gx + r * C + c) = dv;
    }
  }
}

// P^T = x_hat^T G for a 128-channel x 128-column tile over one split of the rows; stage = x boxes (64 rows x 2 x 64
// channels) + G boxes (64 rows x 2 x 64 columns)
template <bool BF16>
__global__ void __launch_bounds__(kThreads, 1)
lnlin_dw_kernel(const __grid_constant__ CUtensorMap tx, const __grid_constant__ CUtensorMap tgk,
                const __grid_constant__ CUtensorMap tgv, const DwParams p) {
  using T = typename std::conditional<BF16, __nv_bfloat16, __half>::type;
  using T2 = typename Elem<T>::T2;
  uint8_t* smem = aligned_smem();
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty = full + kStages;
  float* dbsm = reinterpret_cast<float*>(smem + kStages * kStageBytes + 256);  // [256 consumer threads]
  const int wg = threadIdx.x / 128;
  const int ct = (int)(blockIdx.x % p.tiles_c);
  const int nt = (int)((blockIdx.x / p.tiles_c) % p.tiles_n);
  const int split = (int)(blockIdx.x / ((unsigned)p.tiles_c * p.tiles_n));
  const int64_t kb0 = p.kb_rows * split / p.splits, kb1 = p.kb_rows * (split + 1) / p.splits;
  const int nkb = (int)(kb1 - kb0);
  init_ring(full, empty);

  if (wg == 0) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % kStages;
        uint8_t* st = smem + s * kStageBytes;
        const int r = (int)((kb0 + i) * kBK);
        mbar_wait(&empty[s], ((i / kStages) & 1) ^ 1, 53);
        mbar_arrive_expect_tx(&full[s], kStageBytes);
        tma_load_2d(st, &tx, &full[s], ct * kBM, r);
        tma_load_2d(st + 8192, &tx, &full[s], ct * kBM + 64, r);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int n = nt * kBN + 64 * j;
          if (n < p.n_k || p.n_v == 0) tma_load_2d(st + 16384 + 8192 * j, &tgk, &full[s], n, r);
          else tma_load_2d(st + 16384 + 8192 * j, &tgv, &full[s], n - p.n_k, r);
        }
      }
    }
    return;
  }

  reg_alloc<232>();
  const int cw = wg - 1;
  const int tid = threadIdx.x - 128 * wg;
  const int warp = tid >> 5, lane = tid & 31;
  const int q = lane & 3;
  const uint32_t base = smem_u32(smem);
  // ldmatrix.trans: lane i addresses row i % 8 of matrix i / 8; matrix j covers channels +8 (j & 1), rows +8 (j >> 1)
  const int lm_row = (lane & 7) + 8 * (lane >> 4);
  const int lm_chunk = 2 * warp + ((lane >> 3) & 1);
  // column sums of G (db) by the CTAs of the first channel tile: consumer thread t sums column t % 128 over
  // rows 32 (t / 128) .. + 31 of every stage
  const bool do_db = ct == 0;
  const int t = threadIdx.x - 128;
  const int db_col = t & 127, db_r0 = 32 * (t >> 7);
  const uint32_t db_off = 16384 + 8192 * (db_col >> 6) + 2 * (db_col & 7);
  const int db_chunk = (db_col & 63) >> 3;
  float dbs = 0.f;

  float acc0[32], acc1[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc0[i] = acc1[i] = 0.f;
  for (int i = 0; i < nkb; ++i) {
    const int s = i % kStages;
    const int64_t r0 = (kb0 + i) * kBK;
    float2 sts[4][4];  // [kk][row 2q, 2q + 1, 2q + 8, 2q + 9 of the k16 step]
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t row = r0 + 16 * kk + 2 * q + (e & 1) + 8 * (e >> 1);
        sts[kk][e] = row < p.rows ? p.stats[row] : make_float2(0.f, 0.f);
      }
    mbar_wait(&full[s], (i / kStages) & 1, 54);
    const uint32_t xa = base + s * kStageBytes + cw * 8192;
    uint32_t a[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const int kr = 16 * kk + lm_row;
      ldsm_x4_trans(a[kk], xa + kr * 128 + ((lm_chunk ^ (kr & 7)) << 4));
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int h = j >> 1;
        const float2 f = Elem<T>::to_f2(*reinterpret_cast<const T2*>(&a[kk][j]));
        a[kk][j] = pack2((f.x - sts[kk][2 * h].x) * sts[kk][2 * h].y, (f.y - sts[kk][2 * h + 1].x) * sts[kk][2 * h + 1].y,
                         BF16);
      }
    }
    const uint32_t gb = base + s * kStageBytes + 16384;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      wgmma_rs<64, BF16>(acc0, a[kk], make_desc(gb + kk * 2048));
      wgmma_rs<64, BF16>(acc1, a[kk], make_desc(gb + 8192 + kk * 2048));
    }
    wgmma_commit();
    if (do_db) {
      const uint8_t* sb = smem + s * kStageBytes + db_off;
#pragma unroll 8
      for (int rr = db_r0; rr < db_r0 + 32; ++rr)
        dbs += Elem<T>::to_f(*reinterpret_cast<const T*>(sb + rr * 128 + ((db_chunk ^ (rr & 7)) << 4)));
    }
    wgmma_wait<0>();
    fence_regs(acc0);
    fence_regs(acc1);
    warp_arrive(&empty[s]);
  }

  // accumulator register 4j + 2i + e: channel 16 warp + lane / 4 + 8i, column 8j + 2q + e of the 64-column half
  const int m_base = ct * kBM + 64 * cw + 16 * warp + (lane >> 2);
  float* part = p.p_part + (int64_t)split * p.n_total * p.C;
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int m = m_base + 8 * i;
        const int n0 = nt * kBN + 8 * j + 2 * q + e;
        if (m >= p.C) continue;
        if (n0 < p.n_total) part[(int64_t)n0 * p.C + m] = acc0[4 * j + 2 * i + e];
        if (n0 + 64 < p.n_total) part[(int64_t)(n0 + 64) * p.C + m] = acc1[4 * j + 2 * i + e];
      }
  if (do_db) {
    dbsm[t] = dbs;
    named_bar_sync<1, 256>();
    const int n = nt * kBN + t;
    if (t < kBN && n < p.n_total) p.db_part[(int64_t)split * p.n_total + n] = dbsm[t] + dbsm[t + 128];
  }
}

// db partials without the dW GEMM (grad_b requested, grad_w not): thread n sums column n of G over the rows of split
// blockIdx.y in row order, the same row ranges as lnlin_dw_kernel
template <typename T>
__global__ void __launch_bounds__(256) lnlin_db_kernel(const T* __restrict__ gk, int64_t gk_stride,
                                                       const T* __restrict__ gv, int64_t gv_stride, int n_k, int n_total,
                                                       int64_t rows, int64_t kb_rows, int splits,
                                                       float* __restrict__ db_part) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int split = blockIdx.y;
  if (n >= n_total) return;
  const int64_t r0 = kb_rows * split / splits * kBK, r1 = std::min<int64_t>(kb_rows * (split + 1) / splits * kBK, rows);
  const T* col = n < n_k ? gk + n : gv + (n - n_k);
  const int64_t stride = n < n_k ? gk_stride : gv_stride;
  float s = 0.f;
  for (int64_t r = r0; r < r1; ++r) s += Elem<T>::to_f(col[r * stride]);
  db_part[(int64_t)split * n_total + n] = s;
}

// dW = P diag(gamma) + db beta^T and db, from the split partials summed in split order (grad_w == nullptr: db only)
template <typename T>
__global__ void __launch_bounds__(256) lnlin_dw_finish_kernel(const float* __restrict__ p_part,
                                                              const float* __restrict__ db_part, const T* gamma,
                                                              const T* beta, T* grad_w, T* grad_b, int splits,
                                                              int n_total, int C) {
  const int cols = grad_w != nullptr ? C : 1;
  const int64_t total = (int64_t)n_total * cols;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / cols), c = (int)(idx - (int64_t)n * cols);
    float db = 0.f;
    for (int s = 0; s < splits; ++s) db += db_part[(int64_t)s * n_total + n];
    if (grad_w != nullptr) {
      float pv = 0.f;
      for (int s = 0; s < splits; ++s) pv += p_part[((int64_t)s * n_total + n) * C + c];
      const float g = gamma != nullptr ? Elem<T>::to_f(gamma[c]) : 1.f;
      const float b = beta != nullptr ? Elem<T>::to_f(beta[c]) : 0.f;
      grad_w[idx] = Elem<T>::from_f(fmaf(pv, g, db * b));
    }
    if (grad_b != nullptr && c == 0) grad_b[n] = Elem<T>::from_f(db);
  }
}

// dgamma / dbeta: the (sum dy * x_hat, sum dy) row-block partials of 32 channels per CTA, summed by 8 threads per
// channel over consecutive ranges of row blocks and then in range order
template <typename T>
__global__ void __launch_bounds__(256) lnlin_colsum_kernel(const float2* __restrict__ col_part, int64_t m_blocks,
                                                           int C, T* grad_gamma, T* grad_beta) {
  __shared__ float sx[8][32], sy[8][32];
  const int c = blockIdx.x * 32 + threadIdx.x, y = threadIdx.y;
  float ax = 0.f, ay = 0.f;
  if (c < C) {
    const int64_t b0 = m_blocks * y / 8, b1 = m_blocks * (y + 1) / 8;
    for (int64_t b = b0; b < b1; ++b) {
      const float2 v = col_part[b * C + c];
      ax += v.x;
      ay += v.y;
    }
  }
  sx[y][threadIdx.x] = ax;
  sy[y][threadIdx.x] = ay;
  __syncthreads();
  if (y == 0 && c < C) {
    float tx = 0.f, ty = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      tx += sx[k][threadIdx.x];
      ty += sy[k][threadIdx.x];
    }
    if (grad_gamma != nullptr) grad_gamma[c] = Elem<T>::from_f(tx);
    if (grad_beta != nullptr) grad_beta[c] = Elem<T>::from_f(ty);
  }
}

// argument checks shared by every entry point (no CUDA call)
const char* shape_problem(const pcv_ln_linear_bwd_params& p) {
  if (p.C < 8 || (p.C % 8)) return "input channels must be a multiple of 8 (16-byte TMA strides)";
  if (p.n_k < 0 || p.n_v < 0 || p.n_k + p.n_v < 1) return "no output columns";
  if ((p.n_k % 64) != 0) return "K width must be a multiple of 64";
  if ((p.n_v % 8) != 0) return "V width must be a multiple of 8";
  if (p.rows < 1 || p.rows > (int64_t)0x7fffff00) return "row count out of range";
  return nullptr;
}

const char* args_problem(const pcv_ln_linear_bwd_params& p) {
  if (p.dtype != PCV_BF16 && p.dtype != PCV_F16) return "dtype must be bf16 or fp16";
  if (const char* w = shape_problem(p)) return w;
  if (p.x == nullptr || p.row_stats == nullptr || p.w == nullptr) return "x, row_stats and w must not be NULL";
  if ((p.n_k && p.grad_k == nullptr) || (p.n_v && p.grad_v == nullptr)) return "grad_k / grad_v is NULL for a non-zero width";
  if (!p.grad_x && !p.grad_w && !p.grad_b && !p.grad_gamma && !p.grad_beta) return "no gradient requested";
  if (!al16(p.x) || !al16(p.w) || (p.n_k && !al16(p.grad_k)) || (p.n_v && !al16(p.grad_v)) || !al16(p.grad_x) ||
      !al16(p.gamma))
    return "x / w / grad_k / grad_v / grad_x / gamma must be 16-byte aligned";
  if ((p.x_stride_row % 8) || p.x_stride_row < p.C || (p.n_k && ((p.gk_stride_row % 8) || p.gk_stride_row < p.n_k)) ||
      (p.n_v && ((p.gv_stride_row % 8) || p.gv_stride_row < p.n_v)))
    return "row strides must be multiples of 8 elements covering the row";
  return nullptr;
}

template <bool BF16>
int launch_t(const pcv_ln_linear_bwd_params& p, const Plan& pl, cudaStream_t stream) {
  using T = typename std::conditional<BF16, __nv_bfloat16, __half>::type;
  uint8_t* ws = reinterpret_cast<uint8_t*>(p.workspace);
  float2* row_part = reinterpret_cast<float2*>(ws);
  float2* col_part = reinterpret_cast<float2*>(ws + pl.off_col);
  float* p_part = reinterpret_cast<float*>(ws + pl.off_p);
  float* db_part = reinterpret_cast<float*>(ws + pl.off_db);
  const float2* stats = reinterpret_cast<const float2*>(p.row_stats);
  const int rows = (int)p.rows;
  int rc = attach_wait_diag(&g_wait_diag);
  if (rc != PCV_OK) return rc;

  const bool want_col = p.grad_gamma != nullptr || p.grad_beta != nullptr;
  if (p.grad_x != nullptr || want_col) {
    CUtensorMap tgk, tgv, tw;
    if (p.n_k && (rc = make_tmap_2d(&tgk, p.grad_k, p.dtype, p.n_k, rows, p.gk_stride_row, kBM)) != PCV_OK) return rc;
    if (p.n_v && (rc = make_tmap_2d(&tgv, p.grad_v, p.dtype, p.n_v, rows, p.gv_stride_row, kBM)) != PCV_OK) return rc;
    if (!p.n_k) tgk = tgv;
    if (!p.n_v) tgv = tgk;
    if ((rc = make_tmap_2d(&tw, p.w, p.dtype, p.C, pl.n_total, p.C, kBK)) != PCV_OK) return rc;
    DxParams dp{};
    dp.x = p.x;
    dp.stats = stats;
    dp.gamma = p.gamma;
    dp.grad_x = p.grad_x;
    dp.row_part = row_part;
    dp.col_part = want_col ? col_part : nullptr;
    dp.x_stride = p.x_stride_row;
    dp.rows = p.rows;
    dp.C = p.C;
    dp.kb_k = p.n_k / kBK;
    dp.num_kb = (pl.n_total + kBK - 1) / kBK;
    dp.tiles_c = pl.tiles_c;
    prof_mark_begin(stream);
    rc = launch_kernel(lnlin_dx_kernel<BF16>, dim3((unsigned)(pl.m_blocks * pl.tiles_c)), kThreads, kSmemBytes, 0,
                       stream, tgk, tgv, tw, dp);
    prof_mark_end(stream);
    if (rc != PCV_OK) return rc;
    if (p.grad_x != nullptr) {
      const int blocks = (int)std::min<int64_t>((p.rows + 7) / 8, kWorkers * 8);
      lnlin_dx_fixup_kernel<T><<<blocks, 256, 0, stream>>>(reinterpret_cast<const T*>(p.x), p.x_stride_row, stats,
                                                            row_part, pl.tiles_c, reinterpret_cast<T*>(p.grad_x),
                                                            p.rows, p.C);
      PCV_CHECK_CUDA(cudaGetLastError());
      count_launch();
    }
    if (want_col) {
      lnlin_colsum_kernel<T><<<(p.C + 31) / 32, dim3(32, 8), 0, stream>>>(
          col_part, pl.m_blocks, p.C, reinterpret_cast<T*>(p.grad_gamma), reinterpret_cast<T*>(p.grad_beta));
      PCV_CHECK_CUDA(cudaGetLastError());
      count_launch();
    }
  }

  if (p.grad_w == nullptr && p.grad_b != nullptr) {
    lnlin_db_kernel<T><<<dim3((pl.n_total + 255) / 256, pl.splits), 256, 0, stream>>>(
        reinterpret_cast<const T*>(p.grad_k), p.gk_stride_row, reinterpret_cast<const T*>(p.grad_v), p.gv_stride_row,
        p.n_k, pl.n_total, p.rows, pl.kb_rows, pl.splits, db_part);
    PCV_CHECK_CUDA(cudaGetLastError());
    count_launch();
  } else if (p.grad_w != nullptr) {
    CUtensorMap tx, tgk, tgv;
    if ((rc = make_tmap_2d(&tx, p.x, p.dtype, p.C, rows, p.x_stride_row, kBK)) != PCV_OK) return rc;
    if (p.n_k && (rc = make_tmap_2d(&tgk, p.grad_k, p.dtype, p.n_k, rows, p.gk_stride_row, kBK)) != PCV_OK) return rc;
    if (p.n_v && (rc = make_tmap_2d(&tgv, p.grad_v, p.dtype, p.n_v, rows, p.gv_stride_row, kBK)) != PCV_OK) return rc;
    if (!p.n_k) tgk = tgv;
    if (!p.n_v) tgv = tgk;
    DwParams wp{};
    wp.stats = stats;
    wp.p_part = p_part;
    wp.db_part = db_part;
    wp.rows = p.rows;
    wp.kb_rows = pl.kb_rows;
    wp.C = p.C;
    wp.n_k = p.n_k;
    wp.n_v = p.n_v;
    wp.n_total = pl.n_total;
    wp.tiles_c = pl.tiles_c;
    wp.tiles_n = pl.tiles_n;
    wp.splits = pl.splits;
    prof_mark_begin(stream);
    rc = launch_kernel(lnlin_dw_kernel<BF16>, dim3((unsigned)(pl.splits * pl.tiles_c * pl.tiles_n)), kThreads,
                       kSmemBytes, 0, stream, tx, tgk, tgv, wp);
    prof_mark_end(stream);
    if (rc != PCV_OK) return rc;
  }
  if (p.grad_w != nullptr || p.grad_b != nullptr) {
    const int64_t total = (int64_t)pl.n_total * (p.grad_w != nullptr ? p.C : 1);
    const int blocks = (int)std::min<int64_t>((total + 255) / 256, kWorkers * 16);
    lnlin_dw_finish_kernel<T><<<blocks, 256, 0, stream>>>(p_part, db_part, reinterpret_cast<const T*>(p.gamma),
                                                          reinterpret_cast<const T*>(p.beta),
                                                          reinterpret_cast<T*>(p.grad_w), reinterpret_cast<T*>(p.grad_b),
                                                          pl.splits, pl.n_total, p.C);
    PCV_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  return PCV_OK;
}

}  // namespace

bool ln_linear_bwd_supported(const pcv_ln_linear_bwd_params& p, const char** why) {
  if (const char* w = args_problem(p)) {
    *why = w;
    return false;
  }
  if (const char* w = device_problem()) {
    *why = w;
    return false;
  }
  return true;
}

int ln_linear_bwd_workspace_bytes(const pcv_ln_linear_bwd_params& p, size_t* bytes) {
  PCV_REQUIRE(bytes != nullptr, PCV_ERR_INVALID, "ln_linear_bwd_workspace_bytes: bytes is NULL");
  const char* w = shape_problem(p);
  PCV_REQUIRE(w == nullptr, PCV_ERR_UNSUPPORTED, "ln_linear_bwd_workspace_bytes: %s", w);
  *bytes = make_plan(p.rows, p.C, p.n_k, p.n_v).bytes;
  return PCV_OK;
}

int launch_ln_linear_bwd(const pcv_ln_linear_bwd_params& p, cudaStream_t stream) {
  const char* w = args_problem(p);
  PCV_REQUIRE(w == nullptr, PCV_ERR_UNSUPPORTED, "ln_linear_bwd: %s", w);
  const Plan pl = make_plan(p.rows, p.C, p.n_k, p.n_v);
  PCV_REQUIRE(p.workspace != nullptr && (reinterpret_cast<uintptr_t>(p.workspace) & 255) == 0 &&
                  p.workspace_bytes >= pl.bytes,
              PCV_ERR_WORKSPACE, "ln_linear_bwd: workspace must be 256-byte aligned and hold %zu bytes", pl.bytes);
  w = device_problem();
  PCV_REQUIRE(w == nullptr, PCV_ERR_UNSUPPORTED, "ln_linear_bwd: %s", w);
  return p.dtype == PCV_BF16 ? launch_t<true>(p, pl, stream) : launch_t<false>(p, pl, stream);
}

}  // namespace pcv
