// pcv_attn_simt.cu — shape-generic fused attention forward on the CUDA cores (sm_90a).
//
// This is the coverage kernel of the library: any head dim (odd ones included), any strides,
// fp32 math.  It implements exactly the semantics documented in include/pcv_attn.h
// (reference: perceiver/model/core/modules.py:146-164) with an online softmax, so the
// (B,H,N,M) score tensor is never materialised.  The tcgen05 kernel (pcv_attn_tc.cu) takes over
// whenever the shape fits it; this one also serves as the on-device cross-check for it.
//
// Work decomposition: one CTA = 32 query rows of one (b,h) x one contiguous key range
// ("split"); 8 warps x 4 rows.  Keys stream through shared memory 32 at a time: lane j owns
// key j of the tile for the QK^T dot products (row max / row sum via warp shuffles), then lanes
// own output channels for the PV update (probabilities broadcast with shuffles).
#include "pcv_common.cuh"

namespace pcv {
namespace {

constexpr int kRowsPerWarp = 4;
constexpr int kWarps = 8;
constexpr int kRowsPerCta = kRowsPerWarp * kWarps;  // 32
constexpr int kKeysPerTile = 32;

template <typename T>
__device__ __forceinline__ uint32_t load_pair(const T* base, int64_t off0, bool ok0, bool ok1) {
  // two consecutive channels packed into one 32-bit word (low = even channel); zero outside
  unsigned short lo = 0, hi = 0;
  if (ok0) lo = *reinterpret_cast<const unsigned short*>(base + off0);
  if (ok1) hi = *reinterpret_cast<const unsigned short*>(base + off0 + 1);
  return (uint32_t)lo | ((uint32_t)hi << 16);
}

template <typename T>
__device__ __forceinline__ float2 unpack_pair(uint32_t w) {
  typename Elem<T>::T2 v = *reinterpret_cast<typename Elem<T>::T2*>(&w);
  return Elem<T>::to_f2(v);
}

template <typename T, int DVW>
__global__ void __launch_bounds__(kWarps * 32)
attn_simt_kernel(const pcv_attn_params p, int nsplit, int keys_per_split, float* __restrict__ wo,
                 float* __restrict__ wm, float* __restrict__ wl) {
  extern __shared__ uint32_t smem[];
  const int dq2 = (p.dqk + 1) >> 1;
  const int qs = dq2 | 1;  // odd word stride: lane j reading row j is bank-conflict free
  const int dv2 = (p.dv + 1) >> 1;
  uint32_t* Qs = smem;
  uint32_t* Ks = Qs + kRowsPerCta * qs;
  uint32_t* Vs = Ks + kKeysPerTile * qs;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // blockIdx.x = bh * tiles + query tile: B*H is not bounded by gridDim.y's 65535
  const int tiles = (p.N + kRowsPerCta - 1) / kRowsPerCta;
  const int bh = (int)(blockIdx.x / (unsigned)tiles);
  const int b = bh / p.H, h = bh % p.H;
  const int n0 = (int)(blockIdx.x - (unsigned)bh * tiles) * kRowsPerCta;
  const int split = blockIdx.z;
  const int kb = split * keys_per_split;
  const int ke = min(p.M, kb + keys_per_split);

  const T* q = reinterpret_cast<const T*>(p.q) + (p.q_stride_b ? (int64_t)b * p.q_stride_b : 0) +
               (int64_t)h * p.q_stride_h;
  const T* k = reinterpret_cast<const T*>(p.k) + (int64_t)b * p.k_stride_b + (int64_t)h * p.k_stride_h;
  const T* v = reinterpret_cast<const T*>(p.v) + (int64_t)b * p.v_stride_b + (int64_t)h * p.v_stride_h;

  for (int idx = tid; idx < kRowsPerCta * dq2; idx += blockDim.x) {
    const int r = idx / dq2, w = idx - r * dq2, c = 2 * w, n = n0 + r;
    const bool rok = n < p.N;
    Qs[r * qs + w] = load_pair(q, (int64_t)n * p.q_stride_n + c, rok && c < p.dqk, rok && c + 1 < p.dqk);
  }

  const float scale_log2 = p.scale * kLog2e;
  const int causal_shift = p.m_total - p.N;

  float m[kRowsPerWarp], l[kRowsPerWarp], o[kRowsPerWarp][DVW][2];
#pragma unroll
  for (int i = 0; i < kRowsPerWarp; ++i) {
    m[i] = -INFINITY;
    l[i] = 0.f;
#pragma unroll
    for (int ci = 0; ci < DVW; ++ci) o[i][ci][0] = o[i][ci][1] = 0.f;
  }

  for (int j0 = kb; j0 < ke; j0 += kKeysPerTile) {
    __syncthreads();
    for (int idx = tid; idx < kKeysPerTile * dq2; idx += blockDim.x) {
      const int r = idx / dq2, w = idx - r * dq2, c = 2 * w, j = j0 + r;
      const bool rok = j < ke;
      Ks[r * qs + w] = load_pair(k, (int64_t)j * p.k_stride_m + c, rok && c < p.dqk, rok && c + 1 < p.dqk);
    }
    for (int idx = tid; idx < kKeysPerTile * dv2; idx += blockDim.x) {
      const int r = idx / dv2, w = idx - r * dv2, c = 2 * w, j = j0 + r;
      const bool rok = j < ke;
      Vs[r * dv2 + w] = load_pair(v, (int64_t)j * p.v_stride_m + c, rok && c < p.dv, rok && c + 1 < p.dv);
    }
    __syncthreads();

    float s[kRowsPerWarp];
#pragma unroll
    for (int i = 0; i < kRowsPerWarp; ++i) s[i] = 0.f;
    for (int w = 0; w < dq2; ++w) {
      const float2 kk = unpack_pair<T>(Ks[lane * qs + w]);
#pragma unroll
      for (int i = 0; i < kRowsPerWarp; ++i) {
        const float2 qq = unpack_pair<T>(Qs[(warp * kRowsPerWarp + i) * qs + w]);
        s[i] = fmaf(qq.x, kk.x, s[i]);
        s[i] = fmaf(qq.y, kk.y, s[i]);
      }
    }

    const int j = j0 + lane;
    const bool valid = j < ke;
    const bool padded = valid && p.pad_mask != nullptr && p.pad_mask[(int64_t)b * p.pad_stride_b + j] != 0;
    const int jg = p.m_offset + j;

#pragma unroll
    for (int i = 0; i < kRowsPerWarp; ++i) {
      const int n = n0 + warp * kRowsPerWarp + i;
      float t = s[i] * scale_log2;
      if (padded || (p.causal && jg > n + causal_shift)) t = kMaskedScore;
      if (!valid) t = -INFINITY;
      const float m_new = fmaxf(m[i], warp_max(t));
      const float alpha = exp2f(m[i] - m_new);
      const float pe = exp2f(t - m_new);
      l[i] = l[i] * alpha + warp_sum(pe);
      m[i] = m_new;
#pragma unroll
      for (int ci = 0; ci < DVW; ++ci) {
        o[i][ci][0] *= alpha;
        o[i][ci][1] *= alpha;
      }
      s[i] = pe;
    }

    for (int jj = 0; jj < kKeysPerTile; ++jj) {
      float pj[kRowsPerWarp];
#pragma unroll
      for (int i = 0; i < kRowsPerWarp; ++i) pj[i] = __shfl_sync(0xffffffffu, s[i], jj);
#pragma unroll
      for (int ci = 0; ci < DVW; ++ci) {
        const int w = lane + 32 * ci;
        if (w < dv2) {
          const float2 vv = unpack_pair<T>(Vs[jj * dv2 + w]);
#pragma unroll
          for (int i = 0; i < kRowsPerWarp; ++i) {
            o[i][ci][0] = fmaf(pj[i], vv.x, o[i][ci][0]);
            o[i][ci][1] = fmaf(pj[i], vv.y, o[i][ci][1]);
          }
        }
      }
    }
  }

  const bool direct = (nsplit == 1) && !p.write_partial;
#pragma unroll
  for (int i = 0; i < kRowsPerWarp; ++i) {
    const int n = n0 + warp * kRowsPerWarp + i;
    if (n >= p.N) continue;
    if (direct) {
      const float inv = 1.f / l[i];
      T* out = reinterpret_cast<T*>(p.out) + (int64_t)b * p.o_stride_b + (int64_t)n * p.o_stride_n +
               (int64_t)h * p.o_stride_h;
#pragma unroll
      for (int ci = 0; ci < DVW; ++ci) {
        const int c = 2 * (lane + 32 * ci);
        if (c < p.dv) out[c] = Elem<T>::from_f(o[i][ci][0] * inv);
        if (c + 1 < p.dv) out[c + 1] = Elem<T>::from_f(o[i][ci][1] * inv);
      }
    } else {
      const int64_t R = (int64_t)p.B * p.H * p.N;
      const int64_t r = ((int64_t)b * p.H + h) * p.N + n;
      float* po = wo + ((int64_t)split * R + r) * p.dv;
#pragma unroll
      for (int ci = 0; ci < DVW; ++ci) {
        const int c = 2 * (lane + 32 * ci);
        if (c < p.dv) po[c] = o[i][ci][0];
        if (c + 1 < p.dv) po[c + 1] = o[i][ci][1];
      }
      if (lane == 0) {
        wm[(int64_t)split * R + r] = m[i];
        wl[(int64_t)split * R + r] = l[i];
      }
    }
  }
}

struct SimtPlan {
  int nsplit;
  int keys_per_split;
  size_t smem_bytes;
};

SimtPlan make_plan(const pcv_attn_params& p) {
  SimtPlan pl;
  const int64_t ctas = (int64_t)((p.N + kRowsPerCta - 1) / kRowsPerCta) * p.B * p.H;
  const int64_t want = 132 * 4;  // ~2 waves at 2 CTAs/SM
  int nsplit = (int)((want + ctas - 1) / ctas);
  const int max_split = (p.M + 255) / 256;
  if (nsplit > max_split) nsplit = max_split;
  if (nsplit < 1) nsplit = 1;
  int kps = (p.M + nsplit - 1) / nsplit;
  kps = (kps + kKeysPerTile - 1) / kKeysPerTile * kKeysPerTile;
  nsplit = (p.M + kps - 1) / kps;
  pl.nsplit = nsplit;
  pl.keys_per_split = kps;
  const int dq2 = (p.dqk + 1) / 2, qs = dq2 | 1, dv2 = (p.dv + 1) / 2;
  pl.smem_bytes = sizeof(uint32_t) * ((size_t)(kRowsPerCta + kKeysPerTile) * qs + (size_t)kKeysPerTile * dv2);
  return pl;
}

template <typename T, int DVW>
int launch_t(const pcv_attn_params& p, const SimtPlan& pl, cudaStream_t stream) {
  auto kern = attn_simt_kernel<T, DVW>;
  if (pl.smem_bytes > 48 * 1024) {
    PCV_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  const int64_t R = (int64_t)p.B * p.H * p.N;
  float *wo = nullptr, *wm = nullptr, *wl = nullptr;
  const bool direct = pl.nsplit == 1 && !p.write_partial;
  if (!direct) {
    if (pl.nsplit == 1) {
      wo = p.part_o; wm = p.part_m; wl = p.part_l;  // single split: emit the caller's partial directly
    } else {
      wo = reinterpret_cast<float*>(p.workspace);
      wm = wo + (size_t)pl.nsplit * R * p.dv;
      wl = wm + (size_t)pl.nsplit * R;
    }
  }
  dim3 grid((unsigned)((int64_t)(p.N + kRowsPerCta - 1) / kRowsPerCta * p.B * p.H), 1, pl.nsplit);
  prof_mark_begin(stream);
  kern<<<grid, kWarps * 32, pl.smem_bytes, stream>>>(p, pl.nsplit, pl.keys_per_split, wo, wm, wl);
  prof_mark_end(stream);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

template <typename T>
int launch_dv(const pcv_attn_params& p, const SimtPlan& pl, cudaStream_t stream) {
  const int dvw = ((p.dv + 1) / 2 + 31) / 32;
  if (dvw <= 1) return launch_t<T, 1>(p, pl, stream);
  if (dvw <= 2) return launch_t<T, 2>(p, pl, stream);
  if (dvw <= 4) return launch_t<T, 4>(p, pl, stream);
  if (dvw <= 8) return launch_t<T, 8>(p, pl, stream);
  set_error("simt attention: dv=%d exceeds the supported maximum of 512", p.dv);
  return PCV_ERR_UNSUPPORTED;
}

}  // namespace

int attn_simt_workspace_bytes(const pcv_attn_params& p, size_t* bytes) {
  const SimtPlan pl = make_plan(p);
  const size_t R = (size_t)p.B * p.H * p.N;
  *bytes = pl.nsplit > 1 ? sizeof(float) * pl.nsplit * R * ((size_t)p.dv + 2) : 0;
  return PCV_OK;
}

int launch_attn_simt(const pcv_attn_params& p, cudaStream_t stream) {
  const SimtPlan pl = make_plan(p);
  PCV_REQUIRE(p.dqk <= 1024, PCV_ERR_UNSUPPORTED, "simt attention: dqk=%d exceeds 1024", p.dqk);
  PCV_REQUIRE(pl.smem_bytes <= 200 * 1024, PCV_ERR_UNSUPPORTED, "simt attention: tile does not fit shared memory");
  PCV_REQUIRE((int64_t)(p.N + kRowsPerCta - 1) / kRowsPerCta * p.B * p.H <= INT32_MAX, PCV_ERR_UNSUPPORTED,
              "simt attention: B*H*ceil(N/32) exceeds the grid");
  size_t need = 0;
  attn_simt_workspace_bytes(p, &need);
  PCV_REQUIRE(need == 0 || (p.workspace != nullptr && p.workspace_bytes >= need), PCV_ERR_WORKSPACE,
              "simt attention: workspace of %zu bytes required, %zu given", need, p.workspace_bytes);
  int rc = (p.dtype == PCV_BF16) ? launch_dv<__nv_bfloat16>(p, pl, stream) : launch_dv<__half>(p, pl, stream);
  if (rc != PCV_OK) return rc;
  if (pl.nsplit > 1) {
    const int64_t R = (int64_t)p.B * p.H * p.N;
    const float* wo = reinterpret_cast<const float*>(p.workspace);
    const float* wm = wo + (size_t)pl.nsplit * R * p.dv;
    const float* wl = wm + (size_t)pl.nsplit * R;
    // merge the splits; either into the final output or into the caller's partial state
    return launch_combine_ex(wo, wm, wl, pl.nsplit, p, stream);
  }
  return PCV_OK;
}

}  // namespace pcv
