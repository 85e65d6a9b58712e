// pcv_cached_tile.cuh — the shared-memory tile helpers of the tensor-core attention kernels over a KV cache
// (attn_cached_fp8_kernel in pcv_attn_cached.cu, attn_window_kernel in pcv_attn_window.cu): exact e4m3 -> 16-bit
// conversion and the SWIZZLE_128B layout their wgmma descriptors read.
#pragma once

#include "pcv_sm90.cuh"

namespace pcv {
namespace cached_tile {

// 16 e4m3 codes -> 16 16-bit values (two 16-byte chunks, lowest channel first), exact
template <bool BF16>
__device__ __forceinline__ void convert16(const uint4& u, uint4& lo, uint4& hi) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
  uint32_t h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint16_t pair = (uint16_t)(w[i >> 1] >> (16 * (i & 1)));
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h[i]) : "h"(pair));
    if constexpr (BF16) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h[i]));
      h[i] = sm90::pack2(f.x, f.y, true);
    }
  }
  lo = make_uint4(h[0], h[1], h[2], h[3]);
  hi = make_uint4(h[4], h[5], h[6], h[7]);
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// byte offset of 16-byte chunk `ch` (8 16-bit channels) of row r in a SWIZZLE_128B box
__device__ __forceinline__ uint32_t swz(int r, int ch) { return (uint32_t)(r * 128 + ((ch ^ (r & 7)) << 4)); }

}  // namespace cached_tile
}  // namespace pcv
