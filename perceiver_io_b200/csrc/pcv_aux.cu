// pcv_aux.cu — the small HBM-bound kernels around the attention core (sm_90a):
//   combine   : exact merge of partial softmax states (split-M inside a GPU, M-shards across GPUs)
//   rotary    : RotaryPositionEmbedding.rotate           (reference position.py:30-50)
//   kv_append : KV-cache concat                          (reference modules.py:117-121)
//   pack_pad  : pad-mask bytes -> bit words read by the tensor-core attention kernels
// All are pure streaming kernels: coalesced 16-byte (or widest legal) accesses, grid sized
// from the problem, no shared memory.
#include "pcv_common.cuh"

#include <algorithm>
#include <type_traits>

namespace pcv {
namespace {

// ---------------------------------------------------------------------------------------------
// combine: one warp per (b,h,n) row; lanes stride over dv.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
combine_kernel(const float* __restrict__ po, const float* __restrict__ pm, const float* __restrict__ pl,
               int nparts, int B, int H, int N, int dv, T* __restrict__ out, int64_t osb, int64_t osn,
               int64_t osh, float* __restrict__ mo, float* __restrict__ mm, float* __restrict__ ml) {
  const int64_t R = (int64_t)B * H * N;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= R) return;

  float m = -INFINITY;
  for (int g = 0; g < nparts; ++g) m = fmaxf(m, pm[(int64_t)g * R + r]);
  float l = 0.f;
  for (int g = 0; g < nparts; ++g) {
    const float mg = pm[(int64_t)g * R + r];
    const float w = (mg == -INFINITY) ? 0.f : exp2f(mg - m);
    l += pl[(int64_t)g * R + r] * w;
  }
  const int n = (int)(r % N);
  const int h = (int)((r / N) % H);
  const int b = (int)(r / ((int64_t)N * H));
  const float inv = (out != nullptr) ? 1.f / l : 1.f;
  for (int c = lane; c < dv; c += 32) {
    float acc = 0.f;
    for (int g = 0; g < nparts; ++g) {
      const float mg = pm[(int64_t)g * R + r];
      const float w = (mg == -INFINITY) ? 0.f : exp2f(mg - m);
      acc = fmaf(po[((int64_t)g * R + r) * dv + c], w, acc);
    }
    if (out != nullptr) {
      out[(int64_t)b * osb + (int64_t)n * osn + (int64_t)h * osh + c] = Elem<T>::from_f(acc * inv);
    } else {
      mo[r * dv + c] = acc;
    }
  }
  if (out == nullptr && lane == 0) {
    mm[r] = m;
    ml[r] = l;
  }
}

template <typename T>
int combine_t(const float* po, const float* pm, const float* pl, int nparts, int B, int H, int N, int dv,
              void* out, int64_t osb, int64_t osn, int64_t osh, float* mo, float* mm, float* ml,
              cudaStream_t stream) {
  const int64_t R = (int64_t)B * H * N;
  const int warps = 8;
  const int64_t blocks = (R + warps - 1) / warps;
  combine_kernel<T><<<(unsigned)blocks, warps * 32, 0, stream>>>(po, pm, pl, nparts, B, H, N, dv,
                                                                 reinterpret_cast<T*>(out), osb, osn, osh, mo,
                                                                 mm, ml);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

// ---------------------------------------------------------------------------------------------
// combine over peers: one warp per owned row; every lane keeps num_peers 16-byte loads in flight (the
// remote ones cross NVLink), then pushes the normalised row to every rank's output buffer.  `fast` is
// peers_fast_path(p), the same for the whole grid.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) combine_peers_kernel(const pcv_peer_combine_params p, const bool fast) {
  const int64_t r = p.row_begin + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= p.row_end) return;
  const int G = p.num_peers;
  const int n = (int)(r % p.N);
  const int h = (int)((r / p.N) % p.H);
  const int b = (int)(r / ((int64_t)p.N * p.H));
  const int64_t o_off = (int64_t)b * p.o_stride_b + (int64_t)n * p.o_stride_n + (int64_t)h * p.o_stride_h;

  if (fast) {
    // fast path (dv <= 128): every remote load of the row — row max, denominator and this lane's 16 bytes of the
    // numerator from every peer — is issued BEFORE anything is consumed, so the warp pays one NVLink round trip
    float mg[PCV_MAX_PEERS], lg[PCV_MAX_PEERS];
    float4 x[PCV_MAX_PEERS];
    const int c = lane * 4;
    const bool active = c < p.dv;
#pragma unroll
    for (int g = 0; g < PCV_MAX_PEERS; ++g) {
      if (g < G) {
        // L2-only loads (no read-only / L1 path): the rows were written by OTHER GPUs into peer-mapped memory
        mg[g] = __ldcg(p.part_m[g] + r);
        lg[g] = __ldcg(p.part_l[g] + r);
        x[g] = active ? __ldcg(reinterpret_cast<const float4*>(p.part_o[g] + r * p.dv + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
      } else {
        mg[g] = -INFINITY;
        lg[g] = 0.f;
        x[g] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    float m = -INFINITY;
#pragma unroll
    for (int g = 0; g < PCV_MAX_PEERS; ++g) m = fmaxf(m, mg[g]);
    float l = 0.f;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int g = 0; g < PCV_MAX_PEERS; ++g) {
      const float w = (mg[g] != -INFINITY) ? exp2f(mg[g] - m) : 0.f;
      l = fmaf(lg[g], w, l);
      acc.x = fmaf(x[g].x, w, acc.x);
      acc.y = fmaf(x[g].y, w, acc.y);
      acc.z = fmaf(x[g].z, w, acc.z);
      acc.w = fmaf(x[g].w, w, acc.w);
    }
    if (active) {
      const float inv = 1.f / l;
      T v0 = Elem<T>::from_f(acc.x * inv), v1 = Elem<T>::from_f(acc.y * inv);
      T v2 = Elem<T>::from_f(acc.z * inv), v3 = Elem<T>::from_f(acc.w * inv);
      uint2 packed;
      packed.x = (uint32_t)(*reinterpret_cast<unsigned short*>(&v0)) | ((uint32_t)(*reinterpret_cast<unsigned short*>(&v1)) << 16);
      packed.y = (uint32_t)(*reinterpret_cast<unsigned short*>(&v2)) | ((uint32_t)(*reinterpret_cast<unsigned short*>(&v3)) << 16);
#pragma unroll
      for (int g = 0; g < PCV_MAX_PEERS; ++g)
        if (g < G) *reinterpret_cast<uint2*>(reinterpret_cast<T*>(p.out[g]) + o_off + c) = packed;
    }
    return;
  }

  // general path
  float w[PCV_MAX_PEERS];
  float m = -INFINITY;
  for (int g = 0; g < G; ++g) {
    w[g] = p.part_m[g][r];
    m = fmaxf(m, w[g]);
  }
  float l = 0.f;
  for (int g = 0; g < G; ++g) {
    w[g] = (w[g] != -INFINITY) ? exp2f(w[g] - m) : 0.f;
    l += p.part_l[g][r] * w[g];
  }
  const float inv = 1.f / l;
  for (int c = lane; c < p.dv; c += 32) {
    float acc = 0.f;
    for (int g = 0; g < G; ++g) acc = fmaf(p.part_o[g][r * p.dv + c], w[g], acc);
    for (int g = 0; g < G; ++g) reinterpret_cast<T*>(p.out[g])[o_off + c] = Elem<T>::from_f(acc * inv);
  }
}

// ---------------------------------------------------------------------------------------------
// rescale: one warp per row, float4 where the row length and part_o's alignment allow (`vec`, the same for the
// whole grid: with dv % 4 == 0 every row of a 16-byte aligned part_o is 16-byte aligned).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rescale_kernel(const pcv_rescale_params p, const bool vec) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= p.rows) return;
  const float mo = p.part_m[r], mn = p.new_m[r];
  const float w = (mo == -INFINITY) ? 0.f : exp2f(mo - mn);
  float* row = p.part_o + r * p.dv;
  if (vec) {
    float4* row4 = reinterpret_cast<float4*>(row);
    for (int c = lane; c < (p.dv >> 2); c += 32) {
      float4 x = row4[c];
      x.x *= w; x.y *= w; x.z *= w; x.w *= w;
      row4[c] = x;
    }
  } else {
    for (int c = lane; c < p.dv; c += 32) row[c] *= w;
  }
  __syncwarp();
  if (lane == 0) {
    p.part_l[r] *= w;
    p.part_m[r] = mn;
  }
}

// ---------------------------------------------------------------------------------------------
// rotary: one thread per channel pair.
// AT (pcv_rotary_apply_at): with row b's bounds w = at.bounds + b * at.bounds_stride_b, the angle row of input row i
// is w[0] + i, and so is its output row when w[1] != 0; rows whose angle row lies outside [0, at.capacity) are skipped.
// ---------------------------------------------------------------------------------------------
template <bool AT>
__device__ __forceinline__ bool at_rows(const pcv_rotary_params& p, const pcv_dev_rows& at, int b, int i, int* arow,
                                        int* yrow) {
  if constexpr (AT) {
    const int32_t* w = at.bounds + (int64_t)b * at.bounds_stride_b;
    *arow = w[0] + i;
    *yrow = w[1] ? *arow : i;
    return *arow >= 0 && *arow < at.capacity;
  } else {
    *arow = p.angle_row0 + i;
    *yrow = i;
    return true;
  }
}

template <typename T, bool AT>
__global__ void __launch_bounds__(256) rotary_kernel(const pcv_rotary_params p, const pcv_dev_rows at) {
  const int d2 = (p.d + 1) >> 1;
  const int64_t total = (int64_t)p.B * p.n * p.H * d2;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int pr = (int)(idx % d2);
    int64_t rest = idx / d2;
    const int h = (int)(rest % p.H);
    rest /= p.H;
    const int i = (int)(rest % p.n);
    const int b = (int)(rest / p.n);
    const int c = 2 * pr;
    int arow, yrow;
    if (!at_rows<AT>(p, at, b, i, &arow, &yrow)) continue;
    const T* x = reinterpret_cast<const T*>(p.x) + (int64_t)b * p.x_stride_b + (int64_t)i * p.x_stride_n +
                 (int64_t)h * p.x_stride_h;
    T* y = reinterpret_cast<T*>(p.y) + (int64_t)b * p.y_stride_b + (int64_t)yrow * p.y_stride_n +
           (int64_t)h * p.y_stride_h;
    const float x0 = Elem<T>::to_f(x[c]);
    const float x1 = (c + 1 < p.d) ? Elem<T>::to_f(x[c + 1]) : 0.f;
    if (c + 1 < p.rotate_dim) {
      const float* a = p.angles + (p.a_stride_b ? (int64_t)b * p.a_stride_b : 0) + (int64_t)arow * p.a_stride_n;
      float s0, c0, s1, c1;
      sincosf(a[c], &s0, &c0);
      sincosf(a[c + 1], &s1, &c1);
      y[c] = Elem<T>::from_f(x0 * c0 - x1 * s0);
      y[c + 1] = Elem<T>::from_f(x1 * c1 + x0 * s1);
    } else {
      y[c] = Elem<T>::from_f(x0);
      if (c + 1 < p.d) y[c + 1] = Elem<T>::from_f(x1);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// kv_append: rows of C elements copied with 16-byte vectors when alignment allows.
// blockIdx.y selects the segment: 0 = K cache, 1 = K fresh, 2 = V cache, 3 = V fresh.
// ---------------------------------------------------------------------------------------------
struct CopySeg {
  const char* src;
  char* dst;
  int64_t s_sb, s_sl, d_sb, d_sl;  // byte strides
  int rows;                         // rows per batch
  int row_bytes;
  int dst_row0;
};
struct CopyArgs {
  CopySeg seg[4];
  int B;
};

// AT (pcv_kv_append_at): the first destination row of batch row b is at.bounds[b * at.bounds_stride_b]; rows outside
// [0, at.capacity) are skipped
template <bool AT>
__device__ __forceinline__ bool dst_row(const CopySeg& s, const pcv_dev_rows& at, int b, int row, int* r) {
  if constexpr (AT) {
    *r = at.bounds[(int64_t)b * at.bounds_stride_b] + row;
    return *r >= 0 && *r < at.capacity;
  } else {
    *r = s.dst_row0 + row;
    return true;
  }
}

template <bool AT>
__global__ void __launch_bounds__(256) kv_append_kernel(const CopyArgs a, const pcv_dev_rows at) {
  const CopySeg s = a.seg[blockIdx.y];
  if (s.rows == 0 || s.src == nullptr) return;
  const bool vec = ((reinterpret_cast<uintptr_t>(s.src) | reinterpret_cast<uintptr_t>(s.dst) | (uintptr_t)s.s_sb |
                     (uintptr_t)s.s_sl | (uintptr_t)s.d_sb | (uintptr_t)s.d_sl | (uintptr_t)s.row_bytes) & 15) == 0;
  if (vec) {
    const int vpr = s.row_bytes >> 4;
    const int64_t total = (int64_t)a.B * s.rows * vpr;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
      const int w = (int)(idx % vpr);
      const int64_t rr = idx / vpr;
      const int row = (int)(rr % s.rows);
      const int b = (int)(rr / s.rows);
      int drow;
      if (!dst_row<AT>(s, at, b, row, &drow)) continue;
      const int4 val = *reinterpret_cast<const int4*>(s.src + b * s.s_sb + row * s.s_sl + ((int64_t)w << 4));
      *reinterpret_cast<int4*>(s.dst + b * s.d_sb + (int64_t)drow * s.d_sl + ((int64_t)w << 4)) = val;
    }
  } else {
    const int epr = s.row_bytes >> 1;
    const int64_t total = (int64_t)a.B * s.rows * epr;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
      const int w = (int)(idx % epr);
      const int64_t rr = idx / epr;
      const int row = (int)(rr % s.rows);
      const int b = (int)(rr / s.rows);
      int drow;
      if (!dst_row<AT>(s, at, b, row, &drow)) continue;
      const unsigned short val =
          *reinterpret_cast<const unsigned short*>(s.src + b * s.s_sb + row * s.s_sl + ((int64_t)w << 1));
      *reinterpret_cast<unsigned short*>(s.dst + b * s.d_sb + (int64_t)drow * s.d_sl + ((int64_t)w << 1)) = val;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// kv_append_fp8: kv_append onto e4m3 caches.  blockIdx.y as in kv_append; every thread moves 16 channels: segments 0 / 2
// copy 16 bytes of old e4m3 rows, segments 1 / 3 read 16 bf16 / fp16 channels of a new row, multiply them by the
// channels' inverse scales and round them to e4m3 (row_bytes = channels = e4m3 bytes of a row in every segment).
// ---------------------------------------------------------------------------------------------
struct QuantArgs {
  CopySeg seg[4];        // byte strides; the new rows' source strides are those of their 16-bit elements
  const float* inv[4];   // [1] / [3]: per-channel inverse scales of the new K / V rows
  int B;
};

template <typename T, bool AT>
__global__ void __launch_bounds__(256) kv_append_fp8_kernel(const QuantArgs a, const pcv_dev_rows at) {
  const CopySeg s = a.seg[blockIdx.y];
  if (s.rows == 0 || s.src == nullptr) return;
  const bool quant = blockIdx.y & 1;
  const float* inv = a.inv[blockIdx.y];
  const int vpr = s.row_bytes >> 4;
  const int64_t total = (int64_t)a.B * s.rows * vpr;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int w = (int)(idx % vpr);
    const int64_t rr = idx / vpr;
    const int row = (int)(rr % s.rows);
    const int b = (int)(rr / s.rows);
    int drow;
    if (!dst_row<AT>(s, at, b, row, &drow)) continue;
    const char* src = s.src + b * s.s_sb + row * s.s_sl;
    int4* dst = reinterpret_cast<int4*>(s.dst + b * s.d_sb + (int64_t)drow * s.d_sl + ((int64_t)w << 4));
    if (!quant) {
      *dst = *reinterpret_cast<const int4*>(src + ((int64_t)w << 4));
      continue;
    }
    const uint4* x = reinterpret_cast<const uint4*>(src + ((int64_t)w << 5));
    const uint4 u[2] = {x[0], x[1]};
    const float4* iv = reinterpret_cast<const float4*>(inv + 16 * w);
    uint32_t packed[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // channels 4k .. 4k + 3
      const typename Elem<T>::T2* h = reinterpret_cast<const typename Elem<T>::T2*>(&u[k >> 1]) + 2 * (k & 1);
      const float2 lo = Elem<T>::to_f2(h[0]), hi = Elem<T>::to_f2(h[1]);
      const float4 sc = iv[k];
      packed[k] = cvt_e4m3x2(lo.x * sc.x, lo.y * sc.y) | (cvt_e4m3x2(hi.x * sc.z, hi.y * sc.w) << 16);
    }
    *dst = make_int4((int)packed[0], (int)packed[1], (int)packed[2], (int)packed[3]);
  }
}

// ---------------------------------------------------------------------------------------------
// rotary_fp8: rotary with e4m3 output, one thread per channel pair (one 16-bit store).  T is the input: bf16 / fp16,
// or uint8_t for e4m3 codes dequantised with x_descale[h].  The pair is rotated in fp32 and rounded once.
// ---------------------------------------------------------------------------------------------
template <typename T, bool AT>
__global__ void __launch_bounds__(256)
    rotary_fp8_kernel(const pcv_rotary_params p, const pcv_rotary_fp8 f, const pcv_dev_rows at) {
  const int d2 = p.d >> 1;
  const int64_t total = (int64_t)p.B * p.n * p.H * d2;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int pr = (int)(idx % d2);
    int64_t rest = idx / d2;
    const int h = (int)(rest % p.H);
    rest /= p.H;
    const int i = (int)(rest % p.n);
    const int b = (int)(rest / p.n);
    const int c = 2 * pr;
    int arow, yrow;
    if (!at_rows<AT>(p, at, b, i, &arow, &yrow)) continue;
    const T* x = reinterpret_cast<const T*>(p.x) + (int64_t)b * p.x_stride_b + (int64_t)i * p.x_stride_n +
                 (int64_t)h * p.x_stride_h;
    uint8_t* y = reinterpret_cast<uint8_t*>(p.y) + (int64_t)b * p.y_stride_b + (int64_t)yrow * p.y_stride_n +
                 (int64_t)h * p.y_stride_h;
    float x0, x1;
    if constexpr (std::is_same<T, uint8_t>::value) {
      const float2 v = e4m3x2_to_f2(*reinterpret_cast<const uint16_t*>(x + c));
      const float ds = f.x_descale[h];
      x0 = v.x * ds;
      x1 = v.y * ds;
    } else {
      x0 = Elem<T>::to_f(x[c]);
      x1 = Elem<T>::to_f(x[c + 1]);
    }
    float y0 = x0, y1 = x1;
    if (c + 1 < p.rotate_dim) {
      const float* a = p.angles + (p.a_stride_b ? (int64_t)b * p.a_stride_b : 0) + (int64_t)arow * p.a_stride_n;
      float s0, c0, s1, c1;
      sincosf(a[c], &s0, &c0);
      sincosf(a[c + 1], &s1, &c1);
      y0 = x0 * c0 - x1 * s0;
      y1 = x1 * c1 + x0 * s1;
    }
    const float inv = f.y_inv_scale[h];
    *reinterpret_cast<uint16_t*>(y + c) = (uint16_t)cvt_e4m3x2(y0 * inv, y1 * inv);
  }
}

// pad_mask bytes (B, M) -> bit words (B, wpr), wpr = pad_words_per_row(M); bit set = padding key
__global__ void __launch_bounds__(256) pack_pad_kernel(const uint8_t* __restrict__ pad, int64_t stride_b, int B, int M,
                                                       int wpr, uint32_t* __restrict__ bits) {
  const int64_t total = (int64_t)B * wpr;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(idx / wpr), w = (int)(idx % wpr);
    uint32_t word = 0;
    const int j0 = w * 32;
    for (int i = 0; i < 32; ++i) {
      const int j = j0 + i;
      if (j < M && pad[(int64_t)b * stride_b + j] != 0) word |= (1u << i);
    }
    bits[idx] = word;
  }
}

}  // namespace

int launch_pack_pad(const uint8_t* pad, int64_t stride_b, int B, int M, uint32_t* bits, cudaStream_t stream) {
  const int wpr = pad_words_per_row(M);
  const int64_t total = (int64_t)B * wpr;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, 1024);
  pack_pad_kernel<<<blocks, 256, 0, stream>>>(pad, stride_b, B, M, wpr, bits);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

int launch_combine_ex(const float* po, const float* pm, const float* pl, int nparts, const pcv_attn_params& p,
                      cudaStream_t stream) {
  void* out = p.write_partial ? nullptr : p.out;
  if (p.dtype == PCV_BF16)
    return combine_t<__nv_bfloat16>(po, pm, pl, nparts, p.B, p.H, p.N, p.dv, out, p.o_stride_b, p.o_stride_n,
                                    p.o_stride_h, p.part_o, p.part_m, p.part_l, stream);
  return combine_t<__half>(po, pm, pl, nparts, p.B, p.H, p.N, p.dv, out, p.o_stride_b, p.o_stride_n,
                           p.o_stride_h, p.part_o, p.part_m, p.part_l, stream);
}

int launch_combine(const pcv_combine_params& p, cudaStream_t stream) {
  PCV_REQUIRE(p.part_o && p.part_m && p.part_l && p.out, PCV_ERR_INVALID, "combine: null pointer argument");
  PCV_REQUIRE(p.num_parts >= 1 && p.B >= 1 && p.H >= 1 && p.N >= 1 && p.dv >= 1, PCV_ERR_INVALID,
              "combine: non-positive dimension");
  PCV_REQUIRE(p.dtype == PCV_BF16 || p.dtype == PCV_F16, PCV_ERR_INVALID, "combine: unknown dtype %d", p.dtype);
  if (p.dtype == PCV_BF16)
    return combine_t<__nv_bfloat16>(p.part_o, p.part_m, p.part_l, p.num_parts, p.B, p.H, p.N, p.dv, p.out,
                                    p.o_stride_b, p.o_stride_n, p.o_stride_h, nullptr, nullptr, nullptr, stream);
  return combine_t<__half>(p.part_o, p.part_m, p.part_l, p.num_parts, p.B, p.H, p.N, p.dv, p.out, p.o_stride_b,
                           p.o_stride_n, p.o_stride_h, nullptr, nullptr, nullptr, stream);
}

int launch_merge_partials(const pcv_merge_params& p, cudaStream_t stream) {
  PCV_REQUIRE(p.part_o && p.part_m && p.part_l && p.out_o && p.out_m && p.out_l, PCV_ERR_INVALID, "merge_partials: null pointer");
  PCV_REQUIRE(p.num_parts >= 1 && p.rows >= 1 && p.rows < (int64_t)1 << 31 && p.dv >= 1, PCV_ERR_INVALID,
              "merge_partials: bad dimension");
  // rows are independent: present them to the row-per-warp merge kernel as (B=1, H=1, N=rows)
  return combine_t<__nv_bfloat16>(p.part_o, p.part_m, p.part_l, p.num_parts, 1, 1, (int)p.rows, p.dv, nullptr, 0, 0, 0,
                                  p.out_o, p.out_m, p.out_l, stream);
}

// the rule stated beside pcv_peer_combine_params: 16-byte loads of every part_o row and 8-byte stores of every
// output row (c = 4 * lane, so every element offset a lane touches is a multiple of 4)
static bool peers_fast_path(const pcv_peer_combine_params& p) {
  if ((p.dv & 3) != 0 || p.dv > 128 || ((p.o_stride_b | p.o_stride_n | p.o_stride_h) & 3) != 0) return false;
  for (int g = 0; g < p.num_peers; ++g)
    if (!al16(p.part_o[g]) || (reinterpret_cast<uintptr_t>(p.out[g]) & 7u) != 0) return false;
  return true;
}

int launch_combine_peers(const pcv_peer_combine_params& p, cudaStream_t stream) {
  PCV_REQUIRE(p.num_peers >= 1 && p.num_peers <= PCV_MAX_PEERS, PCV_ERR_INVALID, "combine_peers: num_peers=%d", p.num_peers);
  PCV_REQUIRE(p.rank >= 0 && p.rank < p.num_peers, PCV_ERR_INVALID, "combine_peers: bad rank %d", p.rank);
  PCV_REQUIRE(p.B >= 1 && p.H >= 1 && p.N >= 1 && p.dv >= 1, PCV_ERR_INVALID, "combine_peers: bad dimension");
  PCV_REQUIRE(p.dtype == PCV_BF16 || p.dtype == PCV_F16, PCV_ERR_INVALID, "combine_peers: unknown dtype %d", p.dtype);
  const int64_t R = (int64_t)p.B * p.H * p.N;
  PCV_REQUIRE(p.row_begin >= 0 && p.row_begin <= p.row_end && p.row_end <= R, PCV_ERR_INVALID, "combine_peers: bad row range");
  for (int g = 0; g < p.num_peers; ++g)
    PCV_REQUIRE(p.part_o[g] && p.part_m[g] && p.part_l[g] && p.out[g], PCV_ERR_INVALID, "combine_peers: null pointer for peer %d", g);
  const int64_t rows = p.row_end - p.row_begin;
  if (rows == 0) return PCV_OK;
  const int warps = 8;
  const unsigned blocks = (unsigned)((rows + warps - 1) / warps);
  const bool fast = peers_fast_path(p);
  if (p.dtype == PCV_BF16)
    combine_peers_kernel<__nv_bfloat16><<<blocks, warps * 32, 0, stream>>>(p, fast);
  else
    combine_peers_kernel<__half><<<blocks, warps * 32, 0, stream>>>(p, fast);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

int launch_rescale(const pcv_rescale_params& p, cudaStream_t stream) {
  PCV_REQUIRE(p.part_o && p.part_m && p.part_l && p.new_m, PCV_ERR_INVALID, "rescale: null pointer argument");
  PCV_REQUIRE(p.rows >= 1 && p.dv >= 1, PCV_ERR_INVALID, "rescale: bad dimension");
  const int warps = 8;
  const bool vec = (p.dv & 3) == 0 && al16(p.part_o);
  rescale_kernel<<<(unsigned)((p.rows + warps - 1) / warps), warps * 32, 0, stream>>>(p, vec);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

// the device rows of the *_at entry points
static bool dev_rows_ok(const pcv_dev_rows* at) { return at == nullptr || (at->bounds != nullptr && at->capacity >= 1); }
static bool dev_stride_ok(const pcv_dev_rows* at) { return at == nullptr || at->bounds_stride_b >= 0; }

bool rotary_fp8_supported(const pcv_rotary_params& p, const pcv_rotary_fp8& f, const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (!p.x || !p.y || !p.angles) return fail("null pointer argument");
  if (f.y_inv_scale == nullptr) return fail("y_inv_scale is NULL");
  if (p.dtype != PCV_BF16 && p.dtype != PCV_F16 && p.dtype != PCV_E4M3) return fail("x must be bf16, fp16 or e4m3");
  if (p.dtype == PCV_E4M3 && f.x_descale == nullptr) return fail("e4m3 input needs x_descale");
  if (p.B < 1 || p.n < 0 || p.H < 1 || p.d < 2) return fail("bad dimension");
  if (p.d % 2) return fail("d must be even");
  if (p.rotate_dim < 0 || p.rotate_dim > p.d || (p.rotate_dim % 2)) return fail("rotate_dim must be even and <= d");
  if (p.angle_row0 < 0) return fail("negative angle_row0");
  if ((p.x_stride_b | p.x_stride_n | p.x_stride_h | p.y_stride_b | p.y_stride_n | p.y_stride_h) & 1)
    return fail("strides must be even");
  if ((reinterpret_cast<uintptr_t>(p.y) & 1) || (p.dtype == PCV_E4M3 && (reinterpret_cast<uintptr_t>(p.x) & 1)))
    return fail("e4m3 pointers must be 2-byte aligned");
  return true;
}

template <typename T>
static void rotary_t(const pcv_rotary_params& p, const pcv_rotary_fp8* f, const pcv_dev_rows* at, unsigned blocks,
                     cudaStream_t stream) {
  const pcv_dev_rows r = at != nullptr ? *at : pcv_dev_rows{};
  if (f != nullptr) {
    auto* kernel = at != nullptr ? rotary_fp8_kernel<T, true> : rotary_fp8_kernel<T, false>;
    kernel<<<blocks, 256, 0, stream>>>(p, *f, r);
  } else if constexpr (!std::is_same<T, uint8_t>::value) {  // e4m3 input: e4m3 output only (rotary_fp8_supported)
    auto* kernel = at != nullptr ? rotary_kernel<T, true> : rotary_kernel<T, false>;
    kernel<<<blocks, 256, 0, stream>>>(p, r);
  }
}

int launch_rotary(const pcv_rotary_params& p, const pcv_rotary_fp8* f, const pcv_dev_rows* at, cudaStream_t stream) {
  if (f != nullptr) {
    const char* why = "";
    PCV_REQUIRE(rotary_fp8_supported(p, *f, &why), PCV_ERR_INVALID, "rotary_fp8: %s", why);
  } else {
    PCV_REQUIRE(p.x && p.y && p.angles, PCV_ERR_INVALID, "rotary: null pointer argument");
    PCV_REQUIRE(p.B >= 1 && p.n >= 0 && p.H >= 1 && p.d >= 1, PCV_ERR_INVALID, "rotary: bad dimension");
    PCV_REQUIRE(p.rotate_dim >= 0 && p.rotate_dim <= p.d && (p.rotate_dim % 2) == 0, PCV_ERR_INVALID,
                "rotary: rotate_dim=%d must be even and <= d=%d", p.rotate_dim, p.d);
    PCV_REQUIRE(p.angle_row0 >= 0, PCV_ERR_INVALID, "rotary: negative angle_row0");
    PCV_REQUIRE(p.dtype == PCV_BF16 || p.dtype == PCV_F16, PCV_ERR_INVALID, "rotary: unknown dtype %d", p.dtype);
  }
  PCV_REQUIRE(dev_rows_ok(at), PCV_ERR_INVALID, "%s: rows->bounds NULL or capacity < 1",
              f != nullptr ? "rotary_at_fp8" : "rotary_at");
  PCV_REQUIRE(dev_stride_ok(at), PCV_ERR_INVALID, "%s: rows->bounds_stride_b must be >= 0",
              f != nullptr ? "rotary_at_fp8" : "rotary_at");
  if (p.n == 0) return PCV_OK;
  const int64_t total = (int64_t)p.B * p.n * p.H * ((p.d + 1) / 2);  // one thread per channel pair
  const unsigned blocks = (unsigned)std::min<int64_t>((total + 255) / 256, 132 * 16);
  if (p.dtype == PCV_BF16)
    rotary_t<__nv_bfloat16>(p, f, at, blocks, stream);
  else if (p.dtype == PCV_F16)
    rotary_t<__half>(p, f, at, blocks, stream);
  else
    rotary_t<uint8_t>(p, f, at, blocks, stream);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

bool kv_append_fp8_supported(const pcv_kv_append_params& p, const pcv_kv_fp8_scales& f, const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (!p.k_dst || !p.v_dst || (p.n > 0 && (!p.k_new || !p.v_new))) return fail("null pointer argument");
  if (f.k_inv_scale == nullptr || f.v_inv_scale == nullptr) return fail("k_inv_scale / v_inv_scale are NULL");
  if (p.B < 1 || p.L_old < 0 || p.n < 0 || p.Ck < 1 || p.Cv < 1) return fail("bad dimension");
  if (p.L_old > 0 && (!p.k_cache || !p.v_cache)) return fail("cache pointers required");
  if (p.dtype != PCV_BF16 && p.dtype != PCV_F16) return fail("the new rows must be bf16 or fp16");
  if ((p.Ck % 16) || (p.Cv % 16)) return fail("Ck and Cv must be multiples of 16");
  const void* ptrs[] = {p.k_cache, p.v_cache, p.k_new, p.v_new, p.k_dst, p.v_dst, f.k_inv_scale, f.v_inv_scale};
  for (const void* ptr : ptrs)
    if (!al16(ptr)) return fail("pointers must be 16-byte aligned");
  if ((p.kc_stride_b | p.kc_stride_l | p.vc_stride_b | p.vc_stride_l | p.kd_stride_b | p.kd_stride_l | p.vd_stride_b |
       p.vd_stride_l) & 15)
    return fail("e4m3 strides must be multiples of 16 bytes");
  if ((p.kn_stride_b | p.kn_stride_l | p.vn_stride_b | p.vn_stride_l) & 7)
    return fail("new-row strides must be multiples of 8 elements");
  return true;
}

int launch_kv_append(const pcv_kv_append_params& p, const pcv_kv_fp8_scales* f, const pcv_dev_rows* at,
                     cudaStream_t stream) {
  if (f != nullptr) {
    const char* why = "";
    PCV_REQUIRE(kv_append_fp8_supported(p, *f, &why), PCV_ERR_INVALID, "kv_append_fp8: %s", why);
  } else {
    PCV_REQUIRE(p.k_new && p.v_new && p.k_dst && p.v_dst, PCV_ERR_INVALID, "kv_append: null pointer argument");
    PCV_REQUIRE(p.B >= 1 && p.L_old >= 0 && p.n >= 0 && p.Ck >= 1 && p.Cv >= 1, PCV_ERR_INVALID,
                "kv_append: bad dimension");
    PCV_REQUIRE(p.L_old == 0 || (p.k_cache && p.v_cache), PCV_ERR_INVALID, "kv_append: cache pointers required");
    PCV_REQUIRE(p.dtype >= PCV_BF16 && p.dtype <= PCV_F32, PCV_ERR_INVALID, "kv_append: unknown dtype %d", p.dtype);
  }
  if (at != nullptr) {
    const char* what = f != nullptr ? "kv_append_at_fp8" : "kv_append_at";
    PCV_REQUIRE(dev_rows_ok(at), PCV_ERR_INVALID, "%s: rows->bounds NULL or capacity < 1", what);
    PCV_REQUIRE(dev_stride_ok(at), PCV_ERR_INVALID, "%s: rows->bounds_stride_b must be >= 0", what);
    PCV_REQUIRE(p.L_old == 0 && p.k_cache == nullptr && p.v_cache == nullptr, PCV_ERR_INVALID,
                "%s: an append at device rows takes no cache (k_cache = v_cache = NULL, L_old = 0)", what);
  }
  // element sizes: es of the new rows; ds of the cache and destination rows (1 for e4m3 caches, else es)
  const int es = p.dtype == PCV_F32 ? 4 : 2, ds = f != nullptr ? 1 : es;
  auto seg = [&](const void* src, void* dst, int64_t ssb, int64_t ssl, int64_t dsb, int64_t dsl, int rows, int C,
                 int row0, int src_es) {
    CopySeg s;
    s.src = reinterpret_cast<const char*>(src);
    s.dst = reinterpret_cast<char*>(dst);
    s.s_sb = ssb * src_es; s.s_sl = ssl * src_es; s.d_sb = dsb * ds; s.d_sl = dsl * ds;
    s.rows = rows; s.row_bytes = C * ds; s.dst_row0 = row0;
    if (src == dst && row0 == 0) s.rows = 0;  // in-place arena: the old rows are already there
    return s;
  };
  const CopySeg segs[4] = {
      seg(p.k_cache, p.k_dst, p.kc_stride_b, p.kc_stride_l, p.kd_stride_b, p.kd_stride_l, p.L_old, p.Ck, 0, ds),
      seg(p.k_new, p.k_dst, p.kn_stride_b, p.kn_stride_l, p.kd_stride_b, p.kd_stride_l, p.n, p.Ck, p.L_old, es),
      seg(p.v_cache, p.v_dst, p.vc_stride_b, p.vc_stride_l, p.vd_stride_b, p.vd_stride_l, p.L_old, p.Cv, 0, ds),
      seg(p.v_new, p.v_dst, p.vn_stride_b, p.vn_stride_l, p.vd_stride_b, p.vd_stride_l, p.n, p.Cv, p.L_old, es)};
  int64_t maxwork = 1;
  for (const CopySeg& s : segs) maxwork = std::max<int64_t>(maxwork, (int64_t)p.B * s.rows * (s.row_bytes >> 4));
  const dim3 grid((unsigned)std::min<int64_t>((maxwork + 255) / 256, 132 * 8), 4, 1);
  const pcv_dev_rows r = at != nullptr ? *at : pcv_dev_rows{};
  if (f == nullptr) {
    CopyArgs a;
    std::copy(segs, segs + 4, a.seg);
    a.B = p.B;
    auto* kernel = at != nullptr ? kv_append_kernel<true> : kv_append_kernel<false>;
    kernel<<<grid, 256, 0, stream>>>(a, r);
  } else {
    QuantArgs a;
    std::copy(segs, segs + 4, a.seg);
    a.inv[0] = a.inv[2] = nullptr;
    a.inv[1] = f->k_inv_scale;
    a.inv[3] = f->v_inv_scale;
    a.B = p.B;
    auto* kernel = p.dtype == PCV_BF16 ? (at != nullptr ? kv_append_fp8_kernel<__nv_bfloat16, true>
                                                        : kv_append_fp8_kernel<__nv_bfloat16, false>)
                                       : (at != nullptr ? kv_append_fp8_kernel<__half, true>
                                                        : kv_append_fp8_kernel<__half, false>);
    kernel<<<grid, 256, 0, stream>>>(a, r);
  }
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

}  // namespace pcv
