// pcv_attn_decode.cu — attention for a handful of query rows against a long key/value cache (sm_90a):
// the Perceiver AR decode step (reference modules.py:146-164 with i = 1 query, j = n cached keys; SURVEY.md
// §8(f)3).  With N <= 4 queries the two contractions are matrix-vector products: every K and V byte is used once,
// the tensor cores have nothing to amortise (the 128-row tcgen05 tile would waste 127/128 of its MMA rows) and the
// roofline is HBM: algorithmic bytes = B*M*(Dqk + Dv)*2 per call.  So this is a pure streaming kernel:
//
//   grid = B * splits * H CTAs with the head index fastest (CTAs that run together cover all heads of the same key
//   rows, so DRAM pages are consumed whole); CTA = 4 warps, one (b, h) and a contiguous key range;
//   a key's row is split over LPK lanes x 16 bytes (LPK = max head dim / 8 rounded up to a power of two, <= 32), so a
//   warp covers 32/LPK keys per step with fully coalesced 16-byte loads; kUnroll steps are in flight per warp
//   (all K and V loads of a block are issued before the first is consumed);
//   scores are reduced inside the lane group with shuffles; online softmax per lane group in the log2 domain with
//   one rescale per block of kUnroll keys; probabilities stay fp32 (no bf16 rounding of P: closer to the fp64
//   reference than the tensor-core path);
//   lane groups -> warps -> CTA are merged through shared memory, the split states go to the workspace and the LAST
//   CTA of every (b, h) (atomic ticket) merges them and writes the normalised output or the partial state: one
//   launch, no follow-up merge kernel (CUDA-graph friendly).
// Masks follow include/pcv_attn.h: finite fill for padding / causal keys (a fully masked row is the uniform average).
// The e4m3 variant (FP8, pcv_attn_decode_fp8) reads an FP8 KV cache through the same body: a 16-byte
// load carries 16 channels, so it moves half the bytes per key.
#include "pcv_common.cuh"

#include <algorithm>
#include <type_traits>

namespace pcv {
namespace {

constexpr int kDecWarps = 4;
constexpr int kDecThreads = kDecWarps * 32;
constexpr int kMaxQ = 4;

struct DecParams {
  pcv_attn_params a;
  int nsplit;
  union {
    int keys_per_split;  // without WIN
    int win_stride_b;    // WIN: int32s between the windows of batch rows b and b + 1 (0: one shared window)
  };
  float* ws_o;        // [B*H][nsplit][NQ][dv]
  float* ws_m;        // [B*H][nsplit][NQ]
  float* ws_l;        // [B*H][nsplit][NQ]
  unsigned int* tickets;  // [B*H], zero on entry; the last CTA of a (b,h) resets its ticket
};

template <int NQ>
struct Unroll {
  static constexpr int value = 4;  // warp steps per register buffer; two buffers: 16 independent 16-byte loads per lane
};

template <typename T>
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const typename Elem<T>::T2* h = reinterpret_cast<const typename Elem<T>::T2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 x = Elem<T>::to_f2(h[i]);
    f[2 * i] = x.x;
    f[2 * i + 1] = x.y;
  }
}

// One 16-byte chunk of a K / V row -> floats: 8 bf16 / fp16 channels, or 16 e4m3 channels (FP8)
template <typename T, bool FP8>
__device__ __forceinline__ void unpack_chunk(const uint4& u, float (&f)[FP8 ? 16 : 8]) {
  if constexpr (FP8)
    unpack16_e4m3(u, f);
  else
    unpack8<T>(u, f);
}

// LPK lanes share one key; NQ query rows.  FP8 (pcv_attn_decode_fp8): K / V are e4m3 rows (a 16-byte chunk carries 16
// channels), k_descale[h] is folded into the scaled q and v_descale[h, c] multiplies the accumulator once, before the
// merge; everything else is shared.  WIN (pcv_attn_decode_window): the keys are batch row b's window [w[0], w[1]),
// w = win + b * p.win_stride_b, of an arena of a.M rows, read from device memory: every split takes an equal share of
// the window, the causal mask is right-aligned to its end, and an empty window writes zeros.  f8 and win are unused
// without FP8 / WIN.
template <typename T, int LPK, int NQ, bool FP8, bool WIN>
__global__ void __launch_bounds__(kDecThreads)
    attn_decode_kernel(const DecParams p, const pcv_decode_fp8 f8, const int32_t* win) {
  constexpr int CH = FP8 ? 16 : 8;        // channels per 16-byte chunk of a K / V row
  using KV = typename std::conditional<FP8, uint8_t, T>::type;
  // e4m3 rows hold twice the channels per register: four query rows take half the unroll to stay out of local memory
  constexpr int kUnroll = (FP8 && NQ > 1) ? 2 : Unroll<NQ>::value;
  constexpr int KPW = 32 / LPK;           // keys per warp step
  constexpr int KPB = KPW * kUnroll;      // keys per warp block
  const pcv_attn_params& a = p.a;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sub = lane % LPK;             // 16-byte chunk of the row this lane owns
  const int grp = lane / LPK;             // key of the warp step this lane works on
  // blockIdx.x = (b * nsplit + split) * H + h
  const int h = blockIdx.x % a.H;
  const int split = (blockIdx.x / a.H) % p.nsplit;
  const int b = blockIdx.x / (a.H * p.nsplit);
  const int bh = b * a.H + h;
  int kb, ke, wend = 0;
  if constexpr (WIN) {
    const int32_t* w = win + (int64_t)b * p.win_stride_b;
    const int w0 = max(w[0], 0);
    wend = min(w[1], a.M);
    const int kps = (max(wend - w0, 0) + p.nsplit - 1) / p.nsplit;
    kb = w0 + split * kps;
    ke = min(wend, kb + kps);
  } else {
    kb = split * p.keys_per_split;
    ke = min(a.M, kb + p.keys_per_split);
  }
  const int c0 = sub * CH;
  const bool kq_live = c0 < a.dqk, v_live = c0 < a.dv;

  const T* qp = reinterpret_cast<const T*>(a.q) + (a.q_stride_b ? (int64_t)b * a.q_stride_b : 0) + (int64_t)h * a.q_stride_h + c0;
  const KV* kp = reinterpret_cast<const KV*>(a.k) + (int64_t)b * a.k_stride_b + (int64_t)h * a.k_stride_h + c0;
  const KV* vp = reinterpret_cast<const KV*>(a.v) + (int64_t)b * a.v_stride_b + (int64_t)h * a.v_stride_h + c0;
  const uint8_t* pad = a.pad_mask ? a.pad_mask + (int64_t)b * a.pad_stride_b : nullptr;

  const float scale_log2 = a.scale * kLog2e;
  float q[NQ][CH];
#pragma unroll
  for (int i = 0; i < NQ; ++i) {
    if constexpr (FP8) {
      const float qs = scale_log2 * f8.k_descale[h];  // scores of the dequantised keys, in the log2 domain
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        uint4 u = make_uint4(0, 0, 0, 0);
        if (kq_live && i < a.N) u = *reinterpret_cast<const uint4*>(qp + (int64_t)i * a.q_stride_n + 8 * half);
        float x[8];
        unpack8<T>(u, x);
#pragma unroll
        for (int c = 0; c < 8; ++c) q[i][8 * half + c] = x[c] * qs;
      }
    } else {
      uint4 u = make_uint4(0, 0, 0, 0);
      if (kq_live && i < a.N) u = *reinterpret_cast<const uint4*>(qp + (int64_t)i * a.q_stride_n);
      unpack8<T>(u, q[i]);
#pragma unroll
      for (int c = 0; c < 8; ++c) q[i][c] *= scale_log2;   // scores come out in the log2 domain
    }
  }
  // key jg masked for query n iff jg > n + causal_shift (a window: right-aligned to its end)
  const int causal_shift = (WIN ? wend : a.m_total) - a.N;

  float m[NQ], l[NQ], acc[NQ][CH];
#pragma unroll
  for (int i = 0; i < NQ; ++i) {
    m[i] = -INFINITY;
    l[i] = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[i][c] = 0.f;
  }

  // keys of this CTA are dealt to the warps in blocks of KPB keys: warp w takes blocks w, w + kDecWarps, ...
  // Register double buffering: the loads of block i+1 are issued BEFORE block i is consumed, so every lane always
  // has kUnroll K rows + kUnroll V rows (16 bytes each) in flight while it computes.
  uint4 ku[2][kUnroll], vu[2][kUnroll];
  bool masked[2][kUnroll];
  auto load_block = [&](int buf, int j0) {
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int j = j0 + u * KPW + grp;
      ku[buf][u] = make_uint4(0, 0, 0, 0);
      vu[buf][u] = make_uint4(0, 0, 0, 0);
      masked[buf][u] = false;
      if (j < ke) {
        if (kq_live) ku[buf][u] = __ldcs(reinterpret_cast<const uint4*>(kp + (int64_t)j * a.k_stride_m));
        if (v_live) vu[buf][u] = __ldcs(reinterpret_cast<const uint4*>(vp + (int64_t)j * a.v_stride_m));
        masked[buf][u] = pad != nullptr && pad[j] != 0;
      }
    }
  };
  auto consume_block = [&](int buf, int j0) {
    float s[NQ][kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      float kf[CH];
      unpack_chunk<T, FP8>(ku[buf][u], kf);
      const int j = j0 + u * KPW + grp;
#pragma unroll
      for (int i = 0; i < NQ; ++i) {
        float d = 0.f;
#pragma unroll
        for (int c = 0; c < CH; ++c) d = fmaf(q[i][c], kf[c], d);
#pragma unroll
        for (int o = LPK / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (masked[buf][u] || (a.causal && a.m_offset + j > i + causal_shift)) d = kMaskedScore;
        if (j >= ke) d = -INFINITY;
        s[i][u] = d;
      }
    }
#pragma unroll
    for (int i = 0; i < NQ; ++i) {
      float mb = s[i][0];
#pragma unroll
      for (int u = 1; u < kUnroll; ++u) mb = fmaxf(mb, s[i][u]);
      const float m_new = fmaxf(m[i], mb);
      if (m_new == -INFINITY) continue;  // no live key in this block for this lane group
      const float alpha = exp2f(m[i] - m_new);
      m[i] = m_new;
      l[i] *= alpha;
#pragma unroll
      for (int c = 0; c < CH; ++c) acc[i][c] *= alpha;
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const float pe = exp2f(s[i][u] - m_new);
        l[i] += pe;
        float vf[CH];
        unpack_chunk<T, FP8>(vu[buf][u], vf);
#pragma unroll
        for (int c = 0; c < CH; ++c) acc[i][c] = fmaf(pe, vf[c], acc[i][c]);
      }
    }
  };
  {
    constexpr int kStride = kDecWarps * KPB;
    int j0 = kb + warp * KPB;
    if (j0 < ke) load_block(0, j0);
    while (j0 < ke) {
      if (j0 + kStride < ke) load_block(1, j0 + kStride);
      consume_block(0, j0);
      j0 += kStride;
      if (j0 >= ke) break;
      if (j0 + kStride < ke) load_block(0, j0 + kStride);
      consume_block(1, j0);
      j0 += kStride;
    }
  }
  if constexpr (FP8) {  // the V dequantisation factors of this lane's channels
    if (v_live) {
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const float vd = f8.v_descale[(int64_t)h * a.dv + c0 + c];
#pragma unroll
        for (int i = 0; i < NQ; ++i) acc[i][c] *= vd;
      }
    }
  }

  // ---- merge: lane groups of a warp -> warps of the CTA (shared memory) -----------------------------------
  __shared__ float sm_m[kDecWarps][NQ], sm_l[kDecWarps][NQ];
  __shared__ float sm_o[kDecWarps][NQ][LPK * CH];
#pragma unroll
  for (int i = 0; i < NQ; ++i) {
    // groups: lanes with equal `sub` hold the same channels for different keys
#pragma unroll
    for (int o = LPK; o < 32; o <<= 1) {
      const float m_o = __shfl_xor_sync(0xffffffffu, m[i], o);
      const float l_o = __shfl_xor_sync(0xffffffffu, l[i], o);
      const float m_new = fmaxf(m[i], m_o);
      const float wa = (m[i] == -INFINITY) ? 0.f : exp2f(m[i] - m_new);
      const float wb = (m_o == -INFINITY) ? 0.f : exp2f(m_o - m_new);
      l[i] = l[i] * wa + l_o * wb;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const float a_o = __shfl_xor_sync(0xffffffffu, acc[i][c], o);
        acc[i][c] = acc[i][c] * wa + a_o * wb;
      }
      m[i] = m_new;
    }
    if (grp == 0) {
      if (sub == 0) {
        sm_m[warp][i] = m[i];
        sm_l[warp][i] = l[i];
      }
#pragma unroll
      for (int c = 0; c < CH; ++c) sm_o[warp][i][c0 + c] = acc[i][c];
    }
  }
  __syncthreads();

  const int dvp = LPK * CH;
  // CTA state -> workspace: thread t handles (query i, channel c)
  const int64_t wbase = ((int64_t)bh * p.nsplit + split) * NQ;
  for (int idx = threadIdx.x; idx < NQ * dvp; idx += kDecThreads) {
    const int i = idx / dvp, c = idx - i * dvp;
    float mm = -INFINITY;
#pragma unroll
    for (int w = 0; w < kDecWarps; ++w) mm = fmaxf(mm, sm_m[w][i]);
    float o = 0.f, ll = 0.f;
#pragma unroll
    for (int w = 0; w < kDecWarps; ++w) {
      const float wt = (sm_m[w][i] == -INFINITY) ? 0.f : exp2f(sm_m[w][i] - mm);
      o = fmaf(sm_o[w][i][c], wt, o);
      ll = fmaf(sm_l[w][i], wt, ll);
    }
    if (c < a.dv) p.ws_o[(wbase + i) * a.dv + c] = o;
    if (c == 0) {
      p.ws_m[wbase + i] = mm;
      p.ws_l[wbase + i] = ll;
    }
  }

  // ---- the last CTA of this (b, h) merges the splits ---------------------------------------------------------
  __shared__ unsigned int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(p.tickets + bh, 1u);
    s_last = (t == (unsigned int)p.nsplit - 1) ? 1u : 0u;
    if (s_last) p.tickets[bh] = 0u;  // ready for the next launch on this workspace
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int idx = threadIdx.x; idx < NQ * a.dv; idx += kDecThreads) {
    const int i = idx / a.dv, c = idx - i * a.dv;
    if (i >= a.N) continue;
    const int64_t sb = (int64_t)bh * p.nsplit * NQ + i;
    float mm = -INFINITY;
    for (int sp = 0; sp < p.nsplit; ++sp) mm = fmaxf(mm, __ldcg(p.ws_m + sb + (int64_t)sp * NQ));
    float o = 0.f, ll = 0.f;
    for (int sp = 0; sp < p.nsplit; ++sp) {
      const float ms = __ldcg(p.ws_m + sb + (int64_t)sp * NQ);
      const float wt = (ms == -INFINITY) ? 0.f : exp2f(ms - mm);
      o = fmaf(__ldcg(p.ws_o + (sb + (int64_t)sp * NQ) * a.dv + c), wt, o);
      ll = fmaf(__ldcg(p.ws_l + sb + (int64_t)sp * NQ), wt, ll);
    }
    if constexpr (WIN) {  // an empty window (ll == 0) writes zeros
      T* out = reinterpret_cast<T*>(a.out) + (int64_t)b * a.o_stride_b + (int64_t)i * a.o_stride_n + (int64_t)h * a.o_stride_h;
      out[c] = Elem<T>::from_f(ll > 0.f ? o / ll : 0.f);
    } else if (!a.write_partial) {
      T* out = reinterpret_cast<T*>(a.out) + (int64_t)b * a.o_stride_b + (int64_t)i * a.o_stride_n + (int64_t)h * a.o_stride_h;
      out[c] = Elem<T>::from_f(o / ll);
    } else {
      const int64_t r = ((int64_t)b * a.H + h) * a.N + i;
      a.part_o[r * a.dv + c] = o;
      if (c == 0) {
        a.part_m[r] = mm;
        a.part_l[r] = ll;
      }
    }
  }
}

int choose_split(const pcv_attn_params& a, int* nsplit, int* keys_per_split) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t bh = (int64_t)a.B * a.H;
  // ~12 CTAs (of 4 warps) per SM overall — several waves, so the tail wave is short — at least 256 keys per CTA,
  // splits on 128-key boundaries
  int64_t want = std::max<int64_t>(1, (12LL * sms + bh - 1) / bh);
  const int64_t max_by_keys = std::max<int64_t>(1, a.M / 256);
  want = std::min<int64_t>(std::min<int64_t>(want, max_by_keys), 256);
  int64_t kps = (a.M + want - 1) / want;
  kps = (kps + 127) / 128 * 128;
  *keys_per_split = (int)kps;
  *nsplit = (int)((a.M + kps - 1) / kps);
  return PCV_OK;
}

size_t align256(size_t x) { return (x + 255) / 256 * 256; }

// rows of up to 4 chunks use the 4-lane instantiation with idle lanes; e4m3 rows of up to 256 channels take 16 chunks
template <typename T, bool FP8, bool WIN>
int launch_decode(const DecParams& p, const pcv_decode_fp8& f, const int32_t* win, int lpk, cudaStream_t stream) {
  const dim3 grid((unsigned)((int64_t)p.nsplit * p.a.B * p.a.H));
  auto run = [&](auto lanes) {
    constexpr int LPK = decltype(lanes)::value;
    if (p.a.N == 1)
      attn_decode_kernel<T, LPK, 1, FP8, WIN><<<grid, kDecThreads, 0, stream>>>(p, f, win);
    else  // 2-4 query rows share the four-row instantiation (rows beyond N are zero queries whose results are dropped)
      attn_decode_kernel<T, LPK, 4, FP8, WIN><<<grid, kDecThreads, 0, stream>>>(p, f, win);
  };
  if (lpk <= 4)
    run(std::integral_constant<int, 4>{});
  else if (lpk == 8)
    run(std::integral_constant<int, 8>{});
  else if (FP8 || lpk == 16)
    run(std::integral_constant<int, 16>{});
  else if constexpr (!FP8)
    run(std::integral_constant<int, 32>{});
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

// lanes per key: 16-byte chunks of the longer head row (8 bf16 / fp16 or 16 e4m3 channels each), a power of two
int lanes_per_key(const pcv_attn_params& a, bool fp8) {
  const int ch = fp8 ? 16 : 8;
  const int chunks = (std::max(a.dqk, a.dv) + ch - 1) / ch;
  int lpk = 1;
  while (lpk < chunks) lpk <<= 1;
  return lpk;
}

}  // namespace

bool attn_decode_supported(const pcv_attn_params& a, const pcv_decode_fp8* f, const pcv_dev_rows* rows,
                           const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (rows != nullptr) {
    if (rows->bounds == nullptr) return fail("rows->bounds is NULL");
    if (rows->capacity != a.M) return fail("M must equal rows->capacity (k / v / pad_mask point at arena row 0)");
    if (rows->bounds_stride_b < 0) return fail("rows->bounds_stride_b must be >= 0");
  }
  if (a.dtype != PCV_BF16 && a.dtype != PCV_F16) return fail("dtype (of q and out) must be bf16 or fp16");
  if (a.impl != PCV_IMPL_AUTO && a.impl != PCV_IMPL_DECODE) return fail("impl must be AUTO or DECODE");
  if (rows != nullptr) {
    if (a.write_partial) return fail("the window decode writes the normalised output only (no write_partial)");
    if (a.m_total != a.M || a.m_offset != 0) return fail("the window decode takes no key shard (m_total != M or m_offset != 0)");
  }
  if (a.N > kMaxQ) return fail("more than 4 query rows");
  if (a.dqk > 256 || a.dv > 256) return fail("head dim > 256");
  const int64_t kv = f != nullptr ? 16 : 8;  // K / V elements per 16-byte chunk
  if ((a.dqk % kv) || (a.dv % kv))
    return fail(f != nullptr ? "head dims must be multiples of 16" : "head dims must be multiples of 8");
  if (f != nullptr) {
    if (a.write_partial) return fail("the e4m3 decode writes the normalised output only (no write_partial)");
    if (a.m_total != a.M || a.m_offset != 0) return fail("the e4m3 decode takes no key shard (m_total != M or m_offset != 0)");
    if (f->k_descale == nullptr || f->v_descale == nullptr) return fail("k_descale / v_descale are NULL");
  }
  if (!al16(a.q) || !al16(a.k) || !al16(a.v)) return fail("q/k/v must be 16-byte aligned");
  if ((a.q_stride_n % 8) || (a.q_stride_h % 8) || (a.q_stride_b % 8))
    return fail("q strides must be multiples of 8 elements");
  if ((a.k_stride_m % kv) || (a.v_stride_m % kv) || (a.k_stride_h % kv) || (a.v_stride_h % kv) || (a.k_stride_b % kv) ||
      (a.v_stride_b % kv))
    return fail(f != nullptr ? "e4m3 k/v strides must be multiples of 16 elements"
                             : "k/v strides must be multiples of 8 elements");
  return true;
}

int attn_decode_workspace_bytes(const pcv_attn_params& a, size_t* bytes) {
  int nsplit = 1, kps = a.M;
  choose_split(a, &nsplit, &kps);
  const int nq = a.N <= 1 ? 1 : 4;
  const size_t rows = (size_t)a.B * a.H * nsplit * nq;
  *bytes = align256(rows * a.dv * 4) + 2 * align256(rows * 4) + align256((size_t)a.B * a.H * 4);
  return PCV_OK;
}

// Checks the workspace, fills the kernel params and zeroes the tickets.
static int decode_setup(const pcv_attn_params& a, DecParams* p, cudaStream_t stream) {
  size_t need = 0;
  attn_decode_workspace_bytes(a, &need);
  PCV_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= need, PCV_ERR_WORKSPACE,
              "decode attention: workspace of %zu bytes required, %zu given", need, a.workspace_bytes);
  *p = DecParams{};
  p->a = a;
  choose_split(a, &p->nsplit, &p->keys_per_split);
  const int nq = a.N <= 1 ? 1 : 4;
  const size_t rows = (size_t)a.B * a.H * p->nsplit * nq;
  char* ws = reinterpret_cast<char*>(a.workspace);
  p->ws_o = reinterpret_cast<float*>(ws);
  ws += align256(rows * a.dv * 4);
  p->ws_m = reinterpret_cast<float*>(ws);
  ws += align256(rows * 4);
  p->ws_l = reinterpret_cast<float*>(ws);
  ws += align256(rows * 4);
  p->tickets = reinterpret_cast<unsigned int*>(ws);
  // the workspace is caller memory with arbitrary contents: the tickets must start at zero
  PCV_CHECK_CUDA(cudaMemsetAsync(p->tickets, 0, (size_t)a.B * a.H * 4, stream));
  return PCV_OK;
}

int launch_attn_decode(const pcv_attn_params& a, const pcv_decode_fp8* f, const pcv_dev_rows* rows,
                       cudaStream_t stream) {
  DecParams p;
  const int rc0 = decode_setup(a, &p, stream);  // with rows: planned on the whole arena, fixed for a graph
  if (rc0 != PCV_OK) return rc0;
  const int lpk = lanes_per_key(a, f != nullptr);
  const pcv_decode_fp8 f8 = f != nullptr ? *f : pcv_decode_fp8{};
  const int32_t* win = rows != nullptr ? rows->bounds : nullptr;
  if (rows != nullptr) p.win_stride_b = rows->bounds_stride_b;  // the window kernel splits the window, not M
  auto launch = [&](auto t) {
    using T = decltype(t);
    if (f != nullptr)
      return win != nullptr ? launch_decode<T, true, true>(p, f8, win, lpk, stream)
                            : launch_decode<T, true, false>(p, f8, win, lpk, stream);
    return win != nullptr ? launch_decode<T, false, true>(p, f8, win, lpk, stream)
                          : launch_decode<T, false, false>(p, f8, win, lpk, stream);
  };
  prof_mark_begin(stream);
  const int rc = a.dtype == PCV_BF16 ? launch(__nv_bfloat16{}) : launch(__half{});
  prof_mark_end(stream);
  return rc;
}

}  // namespace pcv
