// pcv_common.cuh — shared host/device helpers for libpcv_attn.so (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cfloat>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/pcv_attn.h"

namespace pcv {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// bracket the dominant kernel with events while profiling is enabled (no-ops otherwise)
void prof_mark_begin(cudaStream_t stream);
void prof_mark_end(cudaStream_t stream);

#define PCV_CHECK_CUDA(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::pcv::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                       __LINE__);                                                         \
      return PCV_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

#define PCV_REQUIRE(cond, code, ...)  \
  do {                                \
    if (!(cond)) {                    \
      ::pcv::set_error(__VA_ARGS__);  \
      return (code);                  \
    }                                 \
  } while (0)

// ---- numeric conventions shared by every kernel ---------------------------------------------
// Scores live in the log2 domain: t = s * scale * log2(e).  Masked keys (padding / causal) take
// the reference's finite fill, keys beyond the end of the tensor are excluded with -inf.
constexpr float kMaskedScore = -FLT_MAX;
constexpr float kLog2e = 1.4426950408889634f;

// ---- element traits --------------------------------------------------------------------------
template <typename T> struct Elem;
template <> struct Elem<__nv_bfloat16> {
  using T2 = __nv_bfloat162;
  static __device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float x) { return __float2bfloat16_rn(x); }
  static __device__ __forceinline__ float2 to_f2(__nv_bfloat162 x) { return __bfloat1622float2(x); }
};
template <> struct Elem<__half> {
  using T2 = __half2;
  static __device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
  static __device__ __forceinline__ __half from_f(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ float2 to_f2(__half2 x) { return __half22float2(x); }
};
template <> struct Elem<float> {  // fp32 outputs (a key shard's grad_q contribution)
  static __device__ __forceinline__ float to_f(float x) { return x; }
  static __device__ __forceinline__ float from_f(float x) { return x; }
};

// ---- e4m3 ------------------------------------------------------------------------------------
// two floats -> two e4m3 bytes (round to nearest even, saturating at +-448), `lo` in the low byte
__device__ __forceinline__ uint32_t cvt_e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// two e4m3 bytes (low byte first) -> two floats; exact (every e4m3 value is an f16 value)
__device__ __forceinline__ float2 e4m3x2_to_f2(uint16_t x) {
  uint32_t h;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(x));
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}
// 16 e4m3 bytes -> 16 floats
__device__ __forceinline__ void unpack16_e4m3(const uint4& u, float (&f)[16]) {
  const uint16_t* b = reinterpret_cast<const uint16_t*>(&u);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float2 x = e4m3x2_to_f2(b[i]);
    f[2 * i] = x.x;
    f[2 * i + 1] = x.y;
  }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

inline bool al16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0; }

// ---- launchers implemented in the individual .cu files ---------------------------------------
// pad_mask bytes (B, M) -> bit words (B, pad_words_per_row(M)), bit set = padding key; one row covers whole 128-key tiles
inline int pad_words_per_row(int M) { return 4 * ((M + 127) / 128); }
int launch_pack_pad(const uint8_t* pad, int64_t stride_b, int B, int M, uint32_t* bits, cudaStream_t stream);

int launch_attn_simt(const pcv_attn_params& p, cudaStream_t stream);
int attn_simt_workspace_bytes(const pcv_attn_params& p, size_t* bytes);

struct DropoutRule;  // pcv_dropout.cuh
bool attn_tc_supported(const pcv_attn_params& p, const char** why);
// drop != nullptr: the one-pass dropout forward (attn_fwd_drop_kernel; partial state, no fuse, no pair; the mask takes
// global key indices, so a key shard must start at an even m_offset)
int launch_attn_tc(const pcv_attn_params& p, cudaStream_t stream, const pcv_shard_fuse* fuse = nullptr,
                   const DropoutRule* drop = nullptr);
bool attn_tc_fuse_supported(const pcv_attn_params& p, const char** why);
int attn_tc_workspace_bytes(const pcv_attn_params& p, size_t* bytes);
// the FP8 forward (attn_fwd_fp8_kernel): e4m3 q / k / V^T; workspace as attn_tc_workspace_bytes
bool attn_tc_fp8_supported(const pcv_attn_params& p, const pcv_fp8_attn& f, const char** why);
int launch_attn_tc_fp8(const pcv_attn_params& p, const pcv_fp8_attn& f, cudaStream_t stream);
int debug_read(uint32_t* out, int n);  // the watchdog record of the wgmma kernels (16 words)
int debug_plan(int B, int H, int N, int M, int workers, int rows_per_unit, int rows_per_tile, int32_t* segs,
               int max_segs, int32_t* counts);  // host-only dump of the tcgen05 work plan
int debug_pair_workers(int32_t* workers, int32_t* clusters_fit);  // the current device's CTA-pair plan width

// the streaming decode kernel: f != nullptr for e4m3 K / V rows (pcv_attn_decode_fp8), rows != nullptr for the key
// window read from device memory (pcv_attn_decode_window (_fp8), M = the arena's capacity)
bool attn_decode_supported(const pcv_attn_params& p, const pcv_decode_fp8* f, const pcv_dev_rows* rows, const char** why);
int launch_attn_decode(const pcv_attn_params& p, const pcv_decode_fp8* f, const pcv_dev_rows* rows, cudaStream_t stream);
int attn_decode_workspace_bytes(const pcv_attn_params& p, size_t* bytes);
// the tensor-core attention of 1 to 64 query rows (pcv_attn_cached.cu): rows == nullptr for the whole e4m3 cache
// (pcv_attn_cached_fp8; f required, band 0), else the window read from device memory of a bf16 / fp16 or e4m3 (f)
// arena with a causal band (pcv_attn_cached_window (_fp8), M = the arena's capacity)
bool attn_cached_supported(const pcv_attn_params& p, const pcv_decode_fp8* f, const pcv_dev_rows* rows, int band,
                           const char** why);
int attn_cached_workspace_bytes(const pcv_attn_params& p, size_t* bytes);
int launch_attn_cached(const pcv_attn_params& p, const pcv_decode_fp8* f, const pcv_dev_rows* rows, int band,
                       cudaStream_t stream);

int launch_combine(const pcv_combine_params& p, cudaStream_t stream);
// Merge `nparts` partial states laid out [part][B][H][N]([dv]) either into p.out (normalised) or,
// when p.write_partial is set, into p.part_o / p.part_m / p.part_l (still un-normalised).
int launch_combine_ex(const float* po, const float* pm, const float* pl, int nparts,
                      const pcv_attn_params& p, cudaStream_t stream);
int launch_combine_peers(const pcv_peer_combine_params& p, cudaStream_t stream);
int launch_merge_partials(const pcv_merge_params& p, cudaStream_t stream);
int launch_rescale(const pcv_rescale_params& p, cudaStream_t stream);
// f != nullptr: the *_fp8 entry points (e4m3 caches / output); at != nullptr: the *_at entry points (rows read from
// device memory, pcv_dev_rows)
int launch_rotary(const pcv_rotary_params& p, const pcv_rotary_fp8* f, const pcv_dev_rows* at, cudaStream_t stream);
int launch_kv_append(const pcv_kv_append_params& p, const pcv_kv_fp8_scales* f, const pcv_dev_rows* at,
                     cudaStream_t stream);
bool kv_append_fp8_supported(const pcv_kv_append_params& p, const pcv_kv_fp8_scales& f, const char** why);
bool rotary_fp8_supported(const pcv_rotary_params& p, const pcv_rotary_fp8& f, const char** why);
int launch_ln_stats(const pcv_ln_stats_params& p, cudaStream_t stream);
bool kv_project_supported(const pcv_kvproj_params& p, const char** why);
int launch_kv_project(const pcv_kvproj_params& p, cudaStream_t stream);
bool kv_project_fp8_supported(const pcv_kvproj_params& p, const pcv_kvproj_fp8& f, const char** why);
int launch_kv_project_fp8(const pcv_kvproj_params& p, const pcv_kvproj_fp8& f, cudaStream_t stream);
bool ln_linear_bwd_supported(const pcv_ln_linear_bwd_params& p, const char** why);
int ln_linear_bwd_workspace_bytes(const pcv_ln_linear_bwd_params& p, size_t* bytes);
int launch_ln_linear_bwd(const pcv_ln_linear_bwd_params& p, cudaStream_t stream);
// shard == nullptr: the backward over all keys (pcv_attn_bwd); else one key shard's (pcv_attn_bwd_shard)
bool attn_bwd_supported(const pcv_attn_bwd_params& p, const pcv_key_shard* shard, const char** why);
int attn_bwd_workspace_bytes(const pcv_attn_bwd_params& p, const pcv_key_shard* shard, size_t* bytes);
int launch_attn_bwd(const pcv_attn_bwd_params& p, const pcv_key_shard* shard, cudaStream_t stream);
int launch_dropout_mask(uint8_t* keep, int B, int H, int N, int key_begin, int key_end, float dropout_p, uint64_t seed,
                        cudaStream_t stream);
// token sampling (pcv_sample.cu)
int sample_check(const pcv_sample_params* p);
int launch_sample(const pcv_sample_params& p, cudaStream_t stream);
int launch_sample_uniforms(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int R, int rows_per_batch,
                           cudaStream_t stream);
int spec_verify_check(const pcv_spec_verify_params* p);
int launch_spec_verify(const pcv_spec_verify_params& p, cudaStream_t stream);
int launch_spec_uniforms(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int R, int rows_per_batch,
                         int stream_id, cudaStream_t stream);
// beam search (pcv_beam.cu)
int beam_step_check(const pcv_beam_step_params* p, bool logprobs = false);
int launch_beam_step(const pcv_beam_step_params& p, bool logprobs, cudaStream_t stream);
int kv_gather_check(const pcv_kv_gather_params* p, const pcv_dev_rows* rows);
int launch_kv_gather(const pcv_kv_gather_params& p, const pcv_dev_rows& rows, cudaStream_t stream);
// contrastive search (pcv_contrastive.cu)
int contrastive_candidates_check(const pcv_contrastive_candidates_params* p);
int launch_contrastive_candidates(const pcv_contrastive_candidates_params& p, cudaStream_t stream);
int contrastive_rank_check(const pcv_contrastive_rank_params* p);
int launch_contrastive_rank(const pcv_contrastive_rank_params& p, cudaStream_t stream);
// logits processors (pcv_process.cu)
int logits_process_check(const pcv_logits_process_params* p);
int launch_logits_process(const pcv_logits_process_params& p, cudaStream_t stream);
// prompt-lookup drafts (pcv_lookup.cu)
int prompt_lookup_check(const pcv_prompt_lookup_params* p);
int launch_prompt_lookup(const pcv_prompt_lookup_params& p, cudaStream_t stream);

}  // namespace pcv
