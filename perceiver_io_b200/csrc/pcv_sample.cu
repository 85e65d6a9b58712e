// pcv_sample.cu — token sampling on the device (pcv_sample, pcv_sample_uniforms): one token per logits row under
// temperature, top-k and top-p, with 🤗's TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper semantics and
// inverse-CDF sampling.  oracle/sample_oracle.py restates every step in numpy.
//
// One CTA of 512 threads per row ρ (batch row b = ρ / rows_per_batch); the row's fp32 x is staged in shared memory.
//   1. x_i = float(logit_i) / temperature, a true fp32 division.  temperature == 0: the argmax of the logits, the lowest
//      index on ties (torch.argmax); nothing random is drawn and the log-probability written is 0.  A row whose largest
//      x is +-inf has no finite mass and is greedy too: the lowest index of the largest x.
//   2. top-k: keep every token with x_i >= the k-th largest x (tokens tied with it stay).  A radix select over
//      order-preserving uint32 keys (-0 folded onto +0), four passes of 256-bin count histograms.
//   3. masses: w_i = round(2^40 · exp(x_i - max x)) in uint64 fixed point (exp in fp64, round half to even), Z = Σ w_i
//      over the kept tokens; V <= 32768 keeps Z below 2^56.  Every sum from here on is an integer sum.
//   4. top-p: with W≤(v) = Σ_{kept, x_j <= v} w_j and cut = floor((1 - (double)top_p) · (double)Z) (fp64 ops), token i
//      is removed iff W≤(x_i) <= cut — 🤗's `cumulative_probs <= 1 - top_p` applied to whole tie groups (a group that
//      straddles the cut stays whole).  The top tie group always stays.  A radix select over the same keys with
//      mass-weighted uint64 histograms.
//   5. draw: 64 bits u = sample_bits(seeds[b], b, positions[ρ]), t = hi64(u · Z_kept); the token is the first index, in
//      vocabulary order, whose kept prefix mass exceeds t (softmax + multinomial on the filtered scores, drawn in index
//      order).  The log-probability written is log(w_token) - log(Z_kept) in fp64, rounded to fp32.
// No floating-point atomics anywhere: the histograms are integer atomics, the scans are fixed-order warp shuffles.
//
// Determinism: a row's token is a pure function of the row's logit bits, temperature, top_k, top_p, its seed, b and its
// position.  It does not depend on R, on the other rows, on the launch or on graph capture; two launches are
// bit-identical.  The logits must be free of NaN and +inf.
//
// Speculative sampling (pcv_spec_verify, pcv_spec_uniforms): the rejection rule of Leviathan et al. / Chen et al. on the
// same integer masses, steps 1-4 shared with sample_kernel (stage_row, kept_threshold); the rule is stated at
// spec_verify_kernel and in include/pcv_attn.h, and oracle/spec_oracle.py restates it with Python integers.
#include "pcv_hash.cuh"
#include "pcv_vocab.cuh"

namespace pcv {

namespace {

constexpr double kMassScale = 1099511627776.0;  // 2^40
using u64 = unsigned long long;

// The 64 random bits of (seed, b, position): two evaluations of three hash_round rounds with distinct keys, the two
// multipliers in swapped order so the halves' rounds collide independently.  The seed's low word enters before the first
// round and its high word before the second, so seeds that differ in either word (adjacent seeds included) pass through
// at least two rounds.
__device__ __forceinline__ uint32_t sample_half(uint32_t word, uint32_t seed_lo, uint32_t seed_hi, uint32_t ca,
                                                uint32_t cb, uint32_t k0, uint32_t k1, uint32_t k2) {
  uint32_t x = hash_round(word ^ seed_lo, ca, k0);
  x = hash_round(x ^ seed_hi, cb, k1);
  return hash_round(x, ca, k2);
}

__device__ __forceinline__ u64 sample_bits(u64 seed, uint32_t b, uint32_t pos) {
  const uint32_t word = (b * 0x9E3779B1u + pos) * 0x85EBCA6Bu;
  const uint32_t lo = (uint32_t)seed, hi = (uint32_t)(seed >> 32);
  const uint32_t h0 = sample_half(word, lo, hi, 0xD2511F53u, 0xCD9E8D57u, 0x3C6EF372u, 0xA54FF53Au, 0x510E527Fu);
  const uint32_t h1 = sample_half(word, lo, hi, 0xCD9E8D57u, 0xD2511F53u, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u);
  return ((u64)h1 << 32) | h0;
}

// w = round(2^40 exp(x - m)); 0 below x - m = -29, where 2^40 exp(x - m) < 0.28
__device__ __forceinline__ u64 token_mass(float x, float m) {
  const double d = (double)x - (double)m;  // exact: both are floats within 2^6 of each other where it matters
  return d < -29.0 ? 0ull : __double2ull_rn(exp(d) * kMassScale);
}

__device__ __forceinline__ u64 warp_sum_u64(u64 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ u64 warp_max_u64(u64 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, (u64)__shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// every thread gets the block's maximum
__device__ __forceinline__ u64 block_max_u64(u64 v, u64* red) {
  v = warp_max_u64(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[threadIdx.x & (kWarps - 1)];
  v = warp_max_u64(v);
  __syncthreads();
  return v;
}

// hist[bin] += v for every lane with bin < 256; lanes with one bin are summed in registers first, so a warp issues one
// shared atomic per distinct bin.  Called by all 32 lanes.
__device__ __forceinline__ void hist_mass(u64* hist, uint32_t bin, u64 v) {
  if (!__ballot_sync(0xffffffffu, bin < 256u)) return;
  const unsigned group = __match_any_sync(0xffffffffu, bin);
  u64 sum = 0;
  if (group == 0xffffffffu) {
    sum = warp_sum_u64(v);
  } else {
#pragma unroll 1
    for (int j = 0; j < 32; ++j) {
      const u64 o = __shfl_sync(0xffffffffu, v, j);
      if ((group >> j) & 1u) sum += o;
    }
  }
  if (bin < 256u && (threadIdx.x & 31) == (unsigned)(__ffs(group) - 1)) atomicAdd(hist + bin, sum);
}

// Step 1 of the sampler on the row src[0 .. V): stages x in xs (x / temperature unless greedy) and returns the
// largest order key in the high word and the complement of the lowest index holding it in the low word.  Called by all
// threads.
template <typename T>
__device__ __forceinline__ u64 stage_row(const T* src, int V, float temperature, float* xs, u64* red) {
  const bool greedy = temperature == 0.f;
  u64 best = 0;
  for (int i = threadIdx.x; i < V; i += kThreads) {
    float x = load_f(src + i);
    if (!greedy) x = x / temperature;
    xs[i] = x;
    best = max(best, ((u64)order_key(x) << 32) | (uint32_t)~(uint32_t)i);
  }
  return block_max_u64(best, red);   // the largest key, and of its ties the lowest index
}

// Steps 2-4 of the sampler (temperature > 0) on the staged row xs whose largest key is top: the least kept key lo under
// v.top_k and v.top_p.  Called by all threads.
template <typename Values>
__device__ __forceinline__ uint32_t kept_threshold(int V, const Values& v, uint32_t top, const float* xs) {
  __shared__ u64 mhist[256];       // top-p masses
  __shared__ u64 sel[2];           // radix state: [0] key prefix, [1] mass below
  __shared__ u64 cut_s;            // the top-p cut
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float m = key_value(top);

  // ---- top-k: the k-th largest key, kept iff key >= lo ----
  uint32_t lo = 0;
  if (v.top_k > 0 && v.top_k < V) lo = select_key(xs, V, (uint32_t)v.top_k);

  // ---- top-p: the least kept key whose W≤ exceeds the cut ----
  if (v.top_p < 1.f) {
    if (tid == 0) sel[0] = 0, sel[1] = 0;
    bool done = false;
    for (int shift = 24; shift >= 0 && !done; shift -= 8) {
      for (int i = tid; i < 256; i += kThreads) mhist[i] = 0;
      __syncthreads();
      const uint32_t prefix = (uint32_t)sel[0], hi_mask = shift == 24 ? 0u : ~0u << (shift + 8);
      const u64 below0 = sel[1];
      for (int base = 0; base < V; base += kThreads) {
        const int i = base + tid;
        uint32_t bin = 256u;
        u64 w = 0;
        if (i < V) {
          const float x = xs[i];
          const uint32_t k = order_key(x);
          if (k >= lo && (k & hi_mask) == prefix) {
            w = token_mass(x, m);
            if (w) bin = (k >> shift) & 255u;
          }
        }
        hist_mass(mhist, bin, w);
      }
      __syncthreads();
      if (warp == 0) {   // lane l owns bins 8l .. 8l+7; the first bin, ascending, whose cumulative mass exceeds the cut
        u64 h[8], own = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = mhist[8 * lane + j], own += h[j];
        u64 incl = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const u64 t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        if (shift == 24) {   // the first pass sees every kept token: Z and the cut
          const u64 Z = __shfl_sync(0xffffffffu, incl, 31);
          const double c = floor((1.0 - (double)v.top_p) * (double)Z);
          if (lane == 0) cut_s = (u64)c;
          __syncwarp();
          if (cut_s >= Z) {   // nothing would stay: the top tie group does
            if (lane == 0) sel[0] = top, sel[1] = ~0ull;
          }
        }
        __syncwarp();
        if (sel[1] != ~0ull) {
          const u64 cut = cut_s;
          u64 below = below0 + incl - own;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (below <= cut && below + h[j] > cut) {
              sel[0] = prefix | ((uint32_t)(8 * lane + j) << shift);
              sel[1] = below;
            }
            below += h[j];
          }
        }
      }
      __syncthreads();
      done = sel[1] == ~0ull;
    }
    lo = max(lo, (uint32_t)sel[0]);
  }
  return lo;
}

// Without the minimum of one CTA per SM in its launch bounds, ptxas fits this kernel in 40 registers (three 512-thread
// CTAs per SM) by spilling to local memory.
template <typename T>
__global__ void __launch_bounds__(kThreads, 1) sample_kernel(const pcv_sample_params p) {
  extern __shared__ __align__(16) float xs[];   // the row's x (V floats)
  __shared__ u64 red[kWarps];
  const int V = p.V, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t row = blockIdx.x;
  const T* src = static_cast<const T*>(p.logits) + row * p.stride_row;
  const u64 best = stage_row(src, V, p.temperature, xs, red);
  const uint32_t top = (uint32_t)(best >> 32);
  const float m = key_value(top);
  if (p.temperature == 0.f || !isfinite(m)) {   // a non-finite max leaves no finite mass: the row is greedy
    if (tid == 0) {
      p.tokens[row] = (int64_t)(uint32_t)~(uint32_t)best;
      if (p.logprobs) p.logprobs[row] = 0.f;
    }
    return;
  }
  const uint32_t lo = kept_threshold(V, p, top, xs);

  // ---- draw: warp w owns a contiguous segment of the vocabulary ----
  const auto [s0, s1] = warp_segment(V);
  u64 part = 0;
  for (int i = s0 + lane; i < s1; i += 32) {
    const float x = xs[i];
    if (order_key(x) >= lo) part += token_mass(x, m);
  }
  part = warp_sum_u64(part);
  __syncthreads();   // red[] was last read by block_max_u64
  if (lane == 0) red[warp] = part;
  __syncthreads();
  u64 before = 0, Zk = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    const u64 v = red[w];
    before += w < warp ? v : 0ull;
    Zk += v;
  }
  const int64_t b = row / p.rows_per_batch;
  const u64 bits = sample_bits(p.seeds[b], (uint32_t)b, (uint32_t)p.positions[row]);
  const u64 t = __umul64hi(bits, Zk);
  if (t < before || t >= before + part) return;   // exactly one warp holds the draw (its part is > 0)
  u64 acc = before;
  for (int base = s0; base < s1; base += 32) {
    const int i = base + lane;
    u64 w = 0;
    if (i < s1) {
      const float x = xs[i];
      if (order_key(x) >= lo) w = token_mass(x, m);
    }
    u64 incl = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u64 v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, acc + incl > t);
    if (hit) {
      if (lane == __ffs(hit) - 1) {
        p.tokens[row] = i;
        if (p.logprobs) p.logprobs[row] = (float)(log((double)w) - log((double)Zk));
      }
      return;
    }
    acc += __shfl_sync(0xffffffffu, incl, 31);
  }
}

__global__ void sample_uniforms_kernel(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int R, int rpb) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int b = r / rpb;
  out[r] = sample_bits(seeds[b], (uint32_t)b, (uint32_t)positions[r]);
}


// ---- speculative sampling (pcv_spec_verify) ----------------------------------------------------------------------------
using u128 = unsigned __int128;
constexpr u64 kMassOne = 1ull << 40;   // the mass of a greedy row's one token
constexpr int kAcceptStream = 0, kResidualStream = 1;

// The accept (stream 0) and residual (stream 1) bits of (seed, b, position): sample_bits' construction with round keys
// of their own, so the three streams are independent at equal counters and every existing draw keeps its bits.
__device__ __forceinline__ u64 spec_bits(u64 seed, uint32_t b, uint32_t pos, int stream) {
  const uint32_t word = (b * 0x9E3779B1u + pos) * 0x85EBCA6Bu;
  const uint32_t lo = (uint32_t)seed, hi = (uint32_t)(seed >> 32);
  const bool acc = stream == kAcceptStream;
  const uint32_t h0 = sample_half(word, lo, hi, 0xD2511F53u, 0xCD9E8D57u, acc ? 0x428A2F98u : 0x923F82A4u,
                                  acc ? 0x71374491u : 0xAB1C5ED5u, acc ? 0xB5C0FBCFu : 0xD807AA98u);
  const uint32_t h1 = sample_half(word, lo, hi, 0xCD9E8D57u, 0xD2511F53u, acc ? 0xE9B5DBA5u : 0x12835B01u,
                                  acc ? 0x3956C25Bu : 0x243185BEu, acc ? 0x59F111F1u : 0x550C7DC3u);
  return ((u64)h1 << 32) | h0;
}

// filter values in the field names kept_threshold reads
struct FilterValues {
  float temperature;
  int32_t top_k;
  float top_p;
};

// A filtered row.  greedy: the one kept token is `arg`.  Otherwise the kept tokens are those with order_key(x) >= lo,
// each of mass token_mass(x, m), with x the row's scaled value in xs.
struct RowFilter {
  bool greedy;
  int arg;
  float m;
  uint32_t lo;
};

template <typename T>
__device__ __forceinline__ RowFilter filter_row(const T* src, int V, const FilterValues& v, float* xs, u64* red) {
  const u64 best = stage_row(src, V, v.temperature, xs, red);
  const uint32_t top = (uint32_t)(best >> 32);
  if (v.temperature == 0.f || !isfinite(key_value(top))) return RowFilter{true, (int)(uint32_t)~(uint32_t)best, 0.f, 0u};
  return RowFilter{false, 0, key_value(top), kept_threshold(V, v, top, xs)};
}

// the kept mass of token i of a filtered row whose scaled value is x
__device__ __forceinline__ u64 kept_mass(const RowFilter& f, float x, int i) {
  return f.greedy ? (i == f.arg ? kMassOne : 0ull) : (order_key(x) >= f.lo ? token_mass(x, f.m) : 0ull);
}

// floor(u * z / 2^64), exact for z < 2^128 with u * floor(z / 2^64) < 2^128 (here z < 2^111)
__device__ __forceinline__ u128 mul_hi64(u64 u, u128 z) {
  return (u128)u * (u64)(z >> 64) + __umul64hi(u, (u64)z);
}

__device__ __forceinline__ u128 shfl_u128(u128 v, int src) {
  const u64 lo = __shfl_sync(0xffffffffu, (u64)v, src), hi = __shfl_sync(0xffffffffu, (u64)(v >> 64), src);
  return ((u128)hi << 64) | lo;
}
__device__ __forceinline__ u128 shfl_up_u128(u128 v, int o) {
  const u64 lo = __shfl_up_sync(0xffffffffu, (u64)v, o), hi = __shfl_up_sync(0xffffffffu, (u64)(v >> 64), o);
  return ((u128)hi << 64) | lo;
}
__device__ __forceinline__ u128 shfl_xor_u128(u128 v, int o) {
  const u64 lo = __shfl_xor_sync(0xffffffffu, (u64)v, o), hi = __shfl_xor_sync(0xffffffffu, (u64)(v >> 64), o);
  return ((u128)hi << 64) | lo;
}

// every thread gets the block's sum
__device__ __forceinline__ u64 block_sum_u64(u64 v, u64* red) {
  v = warp_sum_u64(v);
  __syncthreads();   // red[] may still be read
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  u64 s = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) s += red[w];
  return s;
}

// Warp w's contiguous segment [s0, s1) of the vocabulary, its weight sum and the sums before it and over the block.
struct Segment {
  int s0, s1;
  u128 before, part, total;
};

template <typename W>
__device__ __forceinline__ Segment segment_sums(int V, W weight, u128* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const WarpSegment ws = warp_segment(V);
  Segment s;
  s.s0 = ws.s0;
  s.s1 = ws.s1;
  u128 part = 0;
  for (int y = s.s0 + lane; y < s.s1; y += 32) part += weight(y);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += shfl_xor_u128(part, o);
  __syncthreads();   // red[] of an earlier call has been read
  if (lane == 0) red[warp] = part;
  __syncthreads();
  s.part = part;
  s.before = 0;
  s.total = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    const u128 v = red[w];
    s.before += w < warp ? v : (u128)0;
    s.total += v;
  }
  return s;
}

// *out = the first index, in vocabulary order, whose prefix weight exceeds t (t < s.total): written by the one warp
// whose segment holds it.
template <typename W>
__device__ __forceinline__ void segment_find(W weight, const Segment& s, u128 t, int64_t* out) {
  const int lane = threadIdx.x & 31;
  if (t < s.before || t >= s.before + s.part) return;
  u128 acc = s.before;
  for (int base = s.s0; base < s.s1; base += 32) {
    const int y = base + lane;
    u128 incl = y < s.s1 ? weight(y) : (u128)0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u128 v = shfl_up_u128(incl, o);
      if (lane >= o) incl += v;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, acc + incl > t);
    if (hit) {
      if (lane == __ffs(hit) - 1) *out = y;
      return;
    }
    acc += shfl_u128(incl, 31);
  }
}

// One CTA per (batch row b, target row i), i = 0 .. G.  With P / Zp the kept masses and their sum of target row i and
// Q / Zq those of draft row i under the draft's filter values (i < G), x = tokens[b, i + 1]:
//   accept x iff hi64(u_a * Q(x) * Zp) < P(x) * Zq  (u_a: the accept stream at (seeds[b], b, positions[b, i]));
//   accepted: out[b, i] = -1.  Rejected: out[b, i] = the residual draw: the first index whose prefix sum of
//   R(y) = max(0, P(y) Zq - Q(y) Zp) exceeds hi64(u_r * ΣR) (u_r: the residual stream at the same counter), or, when
//   ΣR = 0, the draw from P.  i = G: out[b, G] = the draw from P with u_r (the bonus token).
// The draft row is filtered first and only its filter (m, lo, Zq, Q(x)) is kept: the target row then takes the same
// shared buffer, and the residual pass recomputes Q(y) from the draft logits in global memory.
template <typename T>
__global__ void __launch_bounds__(kThreads) spec_verify_kernel(const pcv_spec_verify_params p) {
  extern __shared__ __align__(16) float xs[];   // the row's x (V floats): the draft row's, then the target row's
  __shared__ u64 red[kWarps];
  __shared__ u128 red128[kWarps];
  const int V = p.V, G = p.G, tid = threadIdx.x;
  const int b = blockIdx.x / (G + 1), i = blockIdx.x % (G + 1);
  const int64_t cell = (int64_t)b * (G + 1) + i;
  const bool has_draft = i < G;
  const T* tsrc = static_cast<const T*>(p.target) + b * p.t_stride_b + i * p.t_stride_row;
  const T* dsrc = static_cast<const T*>(p.draft) + b * p.d_stride_b + (has_draft ? i : 0) * p.d_stride_row;
  const int64_t x = has_draft ? p.tokens[cell + 1] : -1;
  const bool x_in = x >= 0 && x < V;   // a token outside the vocabulary has P = Q = 0: it is rejected

  RowFilter fq{true, -1, 0.f, 0u};
  u64 Zq = 0, Qx = 0;
  if (has_draft) {
    fq = filter_row(dsrc, V, FilterValues{p.draft_temperature, p.draft_top_k, p.draft_top_p}, xs, red);
    u64 part = 0;
    for (int y = tid; y < V; y += kThreads) part += kept_mass(fq, xs[y], y);
    Zq = block_sum_u64(part, red);
    if (x_in) Qx = kept_mass(fq, xs[x], (int)x);
    __syncthreads();   // every thread has read xs before the target row replaces it
  }
  const RowFilter fp = filter_row(tsrc, V, FilterValues{p.temperature, p.top_k, p.top_p}, xs, red);
  u64 part = 0;
  for (int y = tid; y < V; y += kThreads) part += kept_mass(fp, xs[y], y);
  const u64 Zp = block_sum_u64(part, red);

  const u64 seed = p.seeds[b];
  const uint32_t pos = (uint32_t)p.positions[cell];
  if (has_draft) {
    const u64 Px = x_in ? kept_mass(fp, xs[x], (int)x) : 0ull;
    const u64 ua = spec_bits(seed, (uint32_t)b, pos, kAcceptStream);
    if (mul_hi64(ua, (u128)Qx * Zp) < (u128)Px * Zq) {
      if (tid == 0) p.out_tokens[cell] = -1;
      return;
    }
  }
  const u64 ur = spec_bits(seed, (uint32_t)b, pos, kResidualStream);
  const float tq = p.draft_temperature;
  auto target_mass = [&](int y) -> u128 { return kept_mass(fp, xs[y], y); };
  auto residual = [&](int y) -> u128 {
    const u128 a = (u128)kept_mass(fp, xs[y], y) * Zq;
    const u128 c = (u128)kept_mass(fq, fq.greedy ? 0.f : load_f(dsrc + y) / tq, y) * Zp;
    return a > c ? a - c : (u128)0;
  };
  bool from_residual = has_draft;
  Segment s;
  if (from_residual) {
    s = segment_sums(V, residual, red128);
    from_residual = s.total != 0;   // ΣR = 0 only for a draft Q and P both give no mass: draw from P
  }
  if (!from_residual) s = segment_sums(V, target_mass, red128);
  const u128 t = mul_hi64(ur, s.total);
  if (from_residual) segment_find(residual, s, t, p.out_tokens + cell);
  else segment_find(target_mass, s, t, p.out_tokens + cell);
}

// One thread per batch row: n = the first rejected draft (its cell holds the correction) or G (the bonus), then the
// row's output in place: the n accepted drafts, the correction or bonus token, -1 after it.
__global__ void spec_resolve_kernel(const pcv_spec_verify_params p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  const int G = p.G;
  int64_t* out = p.out_tokens + (int64_t)b * (G + 1);
  const int64_t* fed = p.tokens + (int64_t)b * (G + 1);
  int n = 0;
  while (n < G && out[n] < 0) ++n;
  for (int j = 0; j < n; ++j) out[j] = fed[j + 1];
  for (int j = n + 1; j <= G; ++j) out[j] = -1;
  p.accepted[b] = n;
}

__global__ void spec_uniforms_kernel(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int R, int rpb,
                                     int stream) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int b = r / rpb;
  out[r] = spec_bits(seeds[b], (uint32_t)b, (uint32_t)positions[r], stream);
}

}  // namespace

int sample_check(const pcv_sample_params* p) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "sample: params is NULL");
  PCV_REQUIRE(p->logits && p->seeds && p->positions && p->tokens, PCV_ERR_INVALID,
              "sample: logits / seeds / positions / tokens pointer is NULL");
  PCV_REQUIRE(p->dtype == PCV_BF16 || p->dtype == PCV_F16 || p->dtype == PCV_F32, PCV_ERR_INVALID,
              "sample: unknown dtype %d (bf16, fp16 or fp32 logits)", p->dtype);
  PCV_REQUIRE(p->V >= 1 && p->V <= PCV_SAMPLE_MAX_VOCAB, PCV_ERR_UNSUPPORTED, "sample: V=%d must be in [1, %d]", p->V,
              PCV_SAMPLE_MAX_VOCAB);
  PCV_REQUIRE(p->R >= 1, PCV_ERR_INVALID, "sample: R=%d must be >= 1", p->R);
  PCV_REQUIRE(p->stride_row >= p->V, PCV_ERR_INVALID, "sample: stride_row=%lld is below V=%d",
              (long long)p->stride_row, p->V);
  PCV_REQUIRE(p->rows_per_batch >= 1 && p->R % p->rows_per_batch == 0, PCV_ERR_INVALID,
              "sample: R=%d is not a multiple of rows_per_batch=%d", p->R, p->rows_per_batch);
  PCV_REQUIRE(p->temperature >= 0.f, PCV_ERR_INVALID, "sample: temperature must be >= 0 (0: greedy), got %g",
              (double)p->temperature);
  PCV_REQUIRE(p->top_k >= 0, PCV_ERR_INVALID, "sample: top_k must be >= 0 (0: off), got %d", p->top_k);
  PCV_REQUIRE(p->top_p > 0.f && p->top_p <= 1.f, PCV_ERR_INVALID, "sample: top_p must be in (0, 1] (1: off), got %g",
              (double)p->top_p);
  return PCV_OK;
}

int launch_sample(const pcv_sample_params& p, cudaStream_t stream) {
  void (*const kern[3])(pcv_sample_params) = {sample_kernel<__nv_bfloat16>, sample_kernel<__half>, sample_kernel<float>};
  return launch_row_kernel(kern, p.dtype, p.V, p.R, p, stream);
}

int launch_sample_uniforms(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int R, int rows_per_batch,
                           cudaStream_t stream) {
  PCV_REQUIRE(out && seeds && positions, PCV_ERR_INVALID, "sample_uniforms: out / seeds / positions pointer is NULL");
  PCV_REQUIRE(R >= 1 && rows_per_batch >= 1 && R % rows_per_batch == 0, PCV_ERR_INVALID,
              "sample_uniforms: R=%d must be >= 1 and a multiple of rows_per_batch=%d", R, rows_per_batch);
  sample_uniforms_kernel<<<(R + 255) / 256, 256, 0, stream>>>(out, seeds, positions, R, rows_per_batch);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

static bool sampling_values_ok(const char* who, float temperature, int32_t top_k, float top_p) {
  PCV_REQUIRE(temperature >= 0.f, false, "spec_verify: %s temperature must be >= 0 (0: greedy), got %g", who,
              (double)temperature);
  PCV_REQUIRE(top_k >= 0, false, "spec_verify: %s top_k must be >= 0 (0: off), got %d", who, top_k);
  PCV_REQUIRE(top_p > 0.f && top_p <= 1.f, false, "spec_verify: %s top_p must be in (0, 1] (1: off), got %g", who,
              (double)top_p);
  return true;
}

int spec_verify_check(const pcv_spec_verify_params* p) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "spec_verify: params is NULL");
  PCV_REQUIRE(p->target && p->draft && p->tokens && p->seeds && p->positions && p->out_tokens && p->accepted,
              PCV_ERR_INVALID, "spec_verify: target / draft / tokens / seeds / positions / out_tokens / accepted pointer "
              "is NULL");
  PCV_REQUIRE(p->dtype == PCV_BF16 || p->dtype == PCV_F16 || p->dtype == PCV_F32, PCV_ERR_INVALID,
              "spec_verify: unknown dtype %d (bf16, fp16 or fp32 logits)", p->dtype);
  PCV_REQUIRE(p->draft_dtype == p->dtype, PCV_ERR_INVALID,
              "spec_verify: the draft logits' dtype %d differs from the target logits' dtype %d", p->draft_dtype,
              p->dtype);
  PCV_REQUIRE(p->V >= 1 && p->V <= PCV_SAMPLE_MAX_VOCAB, PCV_ERR_UNSUPPORTED, "spec_verify: V=%d must be in [1, %d]",
              p->V, PCV_SAMPLE_MAX_VOCAB);
  PCV_REQUIRE(p->G >= 1 && p->G <= PCV_SPEC_MAX_DRAFTS, PCV_ERR_UNSUPPORTED, "spec_verify: G=%d must be in [1, %d]",
              p->G, PCV_SPEC_MAX_DRAFTS);
  PCV_REQUIRE(p->B >= 1, PCV_ERR_INVALID, "spec_verify: B=%d must be >= 1", p->B);
  PCV_REQUIRE(p->t_stride_b >= p->V && p->t_stride_row >= p->V && p->d_stride_b >= p->V && p->d_stride_row >= p->V,
              PCV_ERR_INVALID, "spec_verify: a stride (target %lld / %lld, draft %lld / %lld) is below V=%d",
              (long long)p->t_stride_b, (long long)p->t_stride_row, (long long)p->d_stride_b,
              (long long)p->d_stride_row, p->V);
  const int64_t cells = (int64_t)p->B * (p->G + 1);
  PCV_REQUIRE(p->out_tokens + cells <= p->tokens || p->tokens + cells <= p->out_tokens, PCV_ERR_INVALID,
              "spec_verify: out_tokens overlaps tokens");
  if (!sampling_values_ok("target", p->temperature, p->top_k, p->top_p)) return PCV_ERR_INVALID;
  if (!sampling_values_ok("draft", p->draft_temperature, p->draft_top_k, p->draft_top_p)) return PCV_ERR_INVALID;
  return PCV_OK;
}

int launch_spec_verify(const pcv_spec_verify_params& p, cudaStream_t stream) {
  void (*const kern[3])(pcv_spec_verify_params) = {
      spec_verify_kernel<__nv_bfloat16>, spec_verify_kernel<__half>, spec_verify_kernel<float>};
  const int rc = launch_row_kernel(kern, p.dtype, p.V, p.B * (p.G + 1), p, stream);
  if (rc != PCV_OK) return rc;
  spec_resolve_kernel<<<(p.B + 127) / 128, 128, 0, stream>>>(p);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

int launch_spec_uniforms(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int R, int rows_per_batch,
                         int stream_id, cudaStream_t stream) {
  PCV_REQUIRE(out && seeds && positions, PCV_ERR_INVALID, "spec_uniforms: out / seeds / positions pointer is NULL");
  PCV_REQUIRE(R >= 1 && rows_per_batch >= 1 && R % rows_per_batch == 0, PCV_ERR_INVALID,
              "spec_uniforms: R=%d must be >= 1 and a multiple of rows_per_batch=%d", R, rows_per_batch);
  PCV_REQUIRE(stream_id == 0 || stream_id == 1, PCV_ERR_INVALID,
              "spec_uniforms: stream_id=%d must be 0 (accept) or 1 (residual)", stream_id);
  spec_uniforms_kernel<<<(R + 255) / 256, 256, 0, stream>>>(out, seeds, positions, R, rows_per_batch, stream_id);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

}  // namespace pcv
