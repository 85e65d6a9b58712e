// pcv_hash.cuh — the round function of the library's counter-based hashes: the attention-dropout mask
// (pcv_dropout.cuh) and the sampler's random bits (pcv_sample.cu).
#pragma once

#include <cstdint>

namespace pcv {

// One Philox-style round: x <- hi(x*c) ^ lo(x*c) ^ k (one IMAD.WIDE + one LOP3).
__device__ __forceinline__ uint32_t hash_round(uint32_t x, uint32_t c, uint32_t k) {
  const uint64_t pr = (uint64_t)x * c;
  return (uint32_t)(pr >> 32) ^ (uint32_t)pr ^ k;
}

}  // namespace pcv
