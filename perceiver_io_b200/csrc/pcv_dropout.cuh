// pcv_dropout.cuh — the attention-probability dropout mask (modules.py:161: nn.Dropout on the softmax output), shared
// by the dropout forward (attn_fwd_drop_kernel, pcv_attn_tc.cu), the backward kernels (pcv_attn_bwd.cu) and the mask
// export (pcv_attn_dropout_mask / pcv_attn_dropout_mask_range).
// oracle/dropout_oracle.py restates it in numpy.
//
// Counter-based: the keep decision of element (b, h, query q, key k) is a pure function of (seed, b*H+h, q, k), so every
// kernel regenerates the same mask without storing it.  One 32-bit hash per 2 x 2 block (query pair q>>1, key pair k>>1)
// yields four random bytes, byte (q&1)*2 + (k&1) belongs to (q, k); an element is dropped iff its byte < thresh, i.e.
// with probability thresh/256 (the requested p rounded to 1/256; the survivors are scaled by exactly 256/(256 - thresh)).
// A thread that walks keys (query fixed) or queries (key fixed) needs one hash per two columns either way, and its own
// side of the input is a per-thread constant.
// Hash: x = qside ^ kside, then two Philox-style rounds x <- hi(x*C) ^ lo(x*C) ^ K (one IMAD.WIDE + one LOP3 each).
// Checked on 8M-element masks: keep rate, row / column rates, autocorrelation at lags up to 64 in both directions, across
// heads and across adjacent seeds all at the sampling-noise floor (one round is NOT enough: seeds correlate at 3 %).
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>

#include "pcv_hash.cuh"

namespace pcv {

__device__ __forceinline__ uint32_t drop_qword(uint32_t bh, uint32_t q) { return bh * 0x9E3779B1u + (q >> 1); }
__device__ __forceinline__ uint32_t drop_qside(uint32_t seed_lo, uint32_t qword) { return qword * 0x9E3779B1u ^ seed_lo; }
__device__ __forceinline__ uint32_t drop_kside(uint32_t seed_hi, uint32_t k) { return (k >> 1) * 0x85EBCA6Bu ^ seed_hi; }
__device__ __forceinline__ uint32_t drop_finish(uint32_t qside, uint32_t kside) {
  uint32_t x = qside ^ kside;
  x = hash_round(x, 0xD2511F53u, 0x9E3779B9u);
  return hash_round(x, 0xCD9E8D57u, 0xBB67AE85u);
}
__device__ __forceinline__ uint32_t drop_bits(uint32_t seed_lo, uint32_t seed_hi, uint32_t bh, uint32_t q, uint32_t k) {
  return drop_finish(drop_qside(seed_lo, drop_qword(bh, q)), drop_kside(seed_hi, k));
}
__device__ __forceinline__ bool drop_keep(uint32_t bits, uint32_t q, uint32_t k, uint32_t thresh) {
  return ((bits >> (((q & 1u) * 2u + (k & 1u)) * 8u)) & 0xffu) >= thresh;
}

// The kernels' view of a dropout probability: p rounded to 1/256, at least 1/256 when p > 0 (thresh = 0: keep all).
struct DropoutRule {
  uint32_t thresh;
  uint32_t seed_lo, seed_hi;
  float scale;  // survivors are multiplied by 256 / (256 - thresh) = 1 / (1 - thresh/256)
};

inline DropoutRule dropout_rule(float dropout_p, uint64_t seed) {
  DropoutRule r{0u, (uint32_t)(seed & 0xffffffffu), (uint32_t)(seed >> 32), 1.f};
  if (dropout_p > 0.f) {
    const long t = std::min(255L, std::max(1L, std::lround((double)dropout_p * 256.0)));
    r.thresh = (uint32_t)t;
    r.scale = (float)(256.0 / (256.0 - (double)t));
  }
  return r;
}

}  // namespace pcv
