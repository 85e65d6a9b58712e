// pcv_vocab.cuh — what the kernels that scan one row of logits per 512-thread CTA share: sample_kernel and
// spec_verify_kernel (pcv_sample.cu), beam_rows_kernel (pcv_beam.cu) and cs_candidates_kernel (pcv_contrastive.cu).
// Each stages its row's fp32 values in V floats of dynamic shared memory, V <= PCV_SAMPLE_MAX_VOCAB.
#pragma once

#include "pcv_common.cuh"

namespace pcv {

namespace sm90 {
int set_smem_limit(const void* kernel, int smem);  // pcv_sm90_host.cu
}

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;

// order-preserving key of a float: a < b <=> key(a) < key(b); -0 and +0 share a key
__device__ __forceinline__ uint32_t order_key(float x) {
  uint32_t u = __float_as_uint(x);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// hist[bin] += 1 for every lane with bin < 256: one shared atomic per distinct bin of the warp.  Called by all 32 lanes.
__device__ __forceinline__ void hist_count(uint32_t* hist, uint32_t bin) {
  if (!__ballot_sync(0xffffffffu, bin < 256u)) return;
  const unsigned group = __match_any_sync(0xffffffffu, bin);
  if (bin < 256u && (threadIdx.x & 31) == (unsigned)(__ffs(group) - 1)) atomicAdd(hist + bin, (uint32_t)__popc(group));
}

template <typename T>
__device__ __forceinline__ float load_f(const T* p) {
  return Elem<T>::to_f(*p);
}

// The calling warp's contiguous segment [s0, s1) of the vocabulary: ceil(V / kThreads) * 32 indices per warp, so the
// segments of the later warps may be empty.
struct WarpSegment {
  int s0, s1;
};
__device__ __forceinline__ WarpSegment warp_segment(int V) {
  const int seg = ((V + kWarps * 32 - 1) / (kWarps * 32)) * 32;
  const int s0 = (threadIdx.x >> 5) * seg;
  return WarpSegment{s0, min(V, s0 + seg)};
}

// The k-th largest order key of xs[0 .. V), 1 <= k <= V: a radix select of four passes, each a 256-bin count histogram
// of the next 8 bits of the keys that share the prefix chosen so far.  Called by all threads; every thread returns the
// result.  Every thread reads the radix state before the histogram barrier of a pass and warp 0 writes it only after
// that barrier, so the function's shared state may be reused, by a later call, as soon as it returns.
__device__ __forceinline__ uint32_t select_key(const float* xs, int V, uint32_t k) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sel[2];   // radix state: key prefix, count still needed
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t prefix = 0, need = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += kThreads) hist[i] = 0;
    __syncthreads();
    if (shift != 24) prefix = sel[0], need = sel[1];
    const uint32_t hi_mask = shift == 24 ? 0u : ~0u << (shift + 8);
    for (int base = 0; base < V; base += kThreads) {
      const int i = base + tid;
      uint32_t bin = 256u;
      if (i < V) {
        const uint32_t key = order_key(xs[i]);
        if ((key & hi_mask) == prefix) bin = (key >> shift) & 255u;
      }
      hist_count(hist, bin);
    }
    __syncthreads();
    if (warp == 0) {   // lane l owns bins 8l .. 8l+7; find d with above(d) < need <= above(d) + h[d], from the top
      uint32_t h[8], own = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) h[j] = hist[8 * lane + j], own += h[j];
      uint32_t incl = own;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      uint32_t above = __shfl_sync(0xffffffffu, incl, 31) - incl;   // the counts of the lanes above this one
#pragma unroll
      for (int j = 7; j >= 0; --j) {
        if (above < need && above + h[j] >= need) {
          sel[0] = prefix | ((uint32_t)(8 * lane + j) << shift);
          sel[1] = need - above;
        }
        above += h[j];
      }
    }
    __syncthreads();
  }
  return sel[0];
}

// Stages src[0 .. V) as fp32 in xs and returns, to every thread, its max m and S = Σ exp((double)x_i - (double)m) in
// fp64 (per-thread strided sums, a warp butterfly, then the warps in order: a fixed order).  Called by all threads.
struct RowStats {
  float m;
  double S;
};
template <typename T>
__device__ __forceinline__ RowStats stage_max_sum(const T* src, int V, float* xs) {
  __shared__ float redf[kWarps];
  __shared__ double redd[kWarps];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float m = -INFINITY;
  for (int i = tid; i < V; i += kThreads) {
    const float x = load_f(src + i);
    xs[i] = x;
    m = fmaxf(m, x);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) redf[warp] = m;
  __syncthreads();
  m = redf[0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w) m = fmaxf(m, redf[w]);
  double s = 0.0;
  for (int i = tid; i < V; i += kThreads) s += exp((double)xs[i] - (double)m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) redd[warp] = s;
  __syncthreads();
  double S = 0.0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) S += redd[w];
  return RowStats{m, S};
}

// The nsel largest order keys of xs[0 .. V), given thr = select_key(xs, V, nsel): every key above thr, then the keys
// equal to it in index order, unranked, into ckey / cidx[0 .. nsel).  Warp w collects its own warp_segment.  Called by
// all threads; ends with a barrier, after which ckey / cidx are complete.
__device__ __forceinline__ void collect_top(const float* xs, int V, uint32_t nsel, uint32_t thr, uint32_t* ckey,
                                            int32_t* cidx) {
  __shared__ uint32_t wgt[kWarps], weq[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const auto [s0, s1] = warp_segment(V);
  uint32_t ngt = 0, neq = 0;
  for (int base = s0; base < s1; base += 32) {
    const int i = base + lane;
    const uint32_t key = i < s1 ? order_key(xs[i]) : 0u;
    ngt += __popc(__ballot_sync(0xffffffffu, i < s1 && key > thr));
    neq += __popc(__ballot_sync(0xffffffffu, i < s1 && key == thr));
  }
  if (lane == 0) wgt[warp] = ngt, weq[warp] = neq;
  __syncthreads();
  uint32_t gt_before = 0, eq_before = 0, gt_total = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    gt_before += w < warp ? wgt[w] : 0u;
    eq_before += w < warp ? weq[w] : 0u;
    gt_total += wgt[w];
  }
  const uint32_t need_eq = nsel - gt_total;
  for (int base = s0; base < s1; base += 32) {
    const int i = base + lane;
    const uint32_t key = i < s1 ? order_key(xs[i]) : 0u;
    const unsigned below = (1u << lane) - 1u;
    const unsigned bg = __ballot_sync(0xffffffffu, i < s1 && key > thr);
    const unsigned be = __ballot_sync(0xffffffffu, i < s1 && key == thr);
    if ((bg >> lane) & 1u) {
      const uint32_t slot = gt_before + __popc(bg & below);
      ckey[slot] = key, cidx[slot] = i;
    } else if ((be >> lane) & 1u) {
      const uint32_t r = eq_before + __popc(be & below);
      if (r < need_eq) ckey[gt_total + r] = key, cidx[gt_total + r] = i;
    }
    gt_before += __popc(bg);
    eq_before += __popc(be);
  }
  __syncthreads();
}

// The rank of candidate c among ckey / cidx[0 .. n): key descending, then index ascending.
__device__ __forceinline__ int top_rank(const uint32_t* ckey, const int32_t* cidx, int n, int c) {
  const uint32_t key = ckey[c];
  const int idx = cidx[c];
  int rank = 0;
  for (int j = 0; j < n; ++j) rank += (ckey[j] > key || (ckey[j] == key && cidx[j] < idx)) ? 1 : 0;
  return rank;
}

// Launches the row kernel kern[dtype] (the bf16, fp16 and fp32 instantiations, in pcv_dtype order; the callers' checks
// refuse any other dtype) on `grid` CTAs of kThreads with V floats of dynamic shared memory.
template <typename P>
int launch_row_kernel(void (*const (&kern)[3])(P), int dtype, int V, int grid, const P& p, cudaStream_t stream) {
  static_assert(PCV_BF16 == 0 && PCV_F16 == 1 && PCV_F32 == 2, "kern[] is indexed by dtype");
  const int smem = V * (int)sizeof(float);
  // once per kernel and device, for the largest row: whatever V, since the kernels' static shared memory adds to the
  // dynamic V floats and can take a V below 48 KB of floats over the default limit
  const int rc = sm90::set_smem_limit(reinterpret_cast<const void*>(kern[dtype]),
                                      PCV_SAMPLE_MAX_VOCAB * (int)sizeof(float));
  if (rc != PCV_OK) return rc;
  kern[dtype]<<<grid, kThreads, smem, stream>>>(p);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

}  // namespace pcv
