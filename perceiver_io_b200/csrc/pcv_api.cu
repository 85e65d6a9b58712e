// pcv_api.cu — the extern "C" surface of libpcv_attn.so (see include/pcv_attn.h).
// Argument validation, kernel-family dispatch and error reporting live here; kernels live in
// pcv_attn_tc.cu (tcgen05), pcv_attn_simt.cu (CUDA cores) and pcv_aux.cu.
#include "pcv_common.cuh"
#include "pcv_dropout.cuh"

#include <atomic>
#include <cstring>
#include <mutex>
#include <utility>
#include <vector>

namespace pcv {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

static std::mutex g_prof_mu;
static bool g_prof_on = false;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_events;

void prof_mark_begin(cudaStream_t stream) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (!g_prof_on) return;
  cudaEvent_t a, b;
  if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) return;
  cudaEventRecord(a, stream);
  g_prof_events.emplace_back(a, b);
}
void prof_mark_end(cudaStream_t stream) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (!g_prof_on || g_prof_events.empty()) return;
  cudaEventRecord(g_prof_events.back().second, stream);
}

// fp8: the params of pcv_attn_fwd_fp8 (e4m3 operands) or of the workspace query, which serves both forwards
static int validate_attn(const pcv_attn_params* p, bool fp8 = false) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "attn: params is NULL");
  PCV_REQUIRE(p->q && p->k && p->v, PCV_ERR_INVALID, "attn: q/k/v pointer is NULL");
  PCV_REQUIRE(p->B >= 1 && p->H >= 1 && p->N >= 1 && p->M >= 1, PCV_ERR_INVALID,
              "attn: B=%d H=%d N=%d M=%d must all be >= 1", p->B, p->H, p->N, p->M);
  PCV_REQUIRE(p->dqk >= 1 && p->dv >= 1, PCV_ERR_INVALID, "attn: dqk=%d dv=%d must be >= 1", p->dqk, p->dv);
  PCV_REQUIRE(fp8 || p->dtype != PCV_E4M3, PCV_ERR_UNSUPPORTED,
              "attn: e4m3 operands run on pcv_attn_fwd_fp8 only (no CTA pair, fused merge, dropout or decode kernel)");
  PCV_REQUIRE(p->dtype == PCV_BF16 || p->dtype == PCV_F16 || p->dtype == PCV_E4M3, PCV_ERR_INVALID,
              "attn: unknown dtype %d", p->dtype);
  PCV_REQUIRE(p->m_total >= p->M && p->m_offset >= 0 && p->m_offset + p->M <= p->m_total, PCV_ERR_INVALID,
              "attn: shard [%d,%d) outside m_total=%d", p->m_offset, p->m_offset + p->M, p->m_total);
  PCV_REQUIRE(!p->causal || p->m_total >= p->N, PCV_ERR_INVALID,
              "attn: causal attention needs m_total (%d) >= N (%d)", p->m_total, p->N);
  if (p->write_partial) {
    PCV_REQUIRE(p->part_o && p->part_m && p->part_l, PCV_ERR_INVALID, "attn: write_partial set but part_* NULL");
  } else {
    PCV_REQUIRE(p->out != nullptr, PCV_ERR_INVALID, "attn: out pointer is NULL");
  }
  PCV_REQUIRE(p->impl >= PCV_IMPL_AUTO && p->impl <= PCV_IMPL_DECODE, PCV_ERR_INVALID, "attn: unknown impl %d", p->impl);
  return PCV_OK;
}

// few query rows against a long cache: the streaming kernel (HBM-bound) beats a 128-row tensor-core tile
static bool use_decode(const pcv_attn_params& p, const char** why) {
  if (p.impl != PCV_IMPL_AUTO && p.impl != PCV_IMPL_DECODE) {
    *why = "another kernel was requested";
    return false;
  }
  if (!attn_decode_supported(p, nullptr, nullptr, why)) return false;
  if (p.M < 1024) *why = "short key axis (the general kernels are as fast)";
  return p.M >= 1024;
}

// The one-pass dropout forward: the tensor-core kernel's partial state, over all keys of an unsharded call or (shard)
// over a key shard starting at an even global key.
static bool partial_dropout_supported(const pcv_attn_params& p, float dropout_p, bool shard, const char** why) {
  auto no = [&](const char* w) {
    *why = w;
    return false;
  };
  if (!(dropout_p > 0.f && dropout_p < 1.f)) return no("dropout_p must be in (0, 1)");
  if (!p.write_partial) return no("the call must write the partial state (write_partial = 1)");
  if (!shard && (p.m_total != p.M || p.m_offset != 0))
    return no("key sharding takes no dropout here (pcv_attn_fwd_partial_dropout_shard)");
  if (p.m_offset % 2) return no("m_offset must be even (the dropout mask hashes key pairs)");
  if (p.impl != PCV_IMPL_AUTO && p.impl != PCV_IMPL_TCGEN05) return no("only the single-CTA tensor-core kernel takes dropout");
  return attn_tc_supported(p, why);
}

static bool use_tc(const pcv_attn_params& p, const char** why) {
  if (p.impl == PCV_IMPL_SIMT || p.impl == PCV_IMPL_DECODE) {
    *why = "another kernel was requested";
    return false;
  }
  return attn_tc_supported(p, why);
}

}  // namespace pcv

using namespace pcv;

extern "C" {

int pcv_abi_version(void) { return PCV_ABI_VERSION; }

const char* pcv_last_error(void) { return g_err; }

int pcv_profile_begin(void) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_on = true;
  return PCV_OK;
}

int pcv_profile_end(double* main_kernel_ms_total, int32_t* main_kernel_launches) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_on = false;
  double total = 0.0;
  int n = 0;
  for (auto& ev : g_prof_events) {
    float ms = 0.f;
    if (cudaEventSynchronize(ev.second) == cudaSuccess && cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) {
      total += ms;
      ++n;
    }
    cudaEventDestroy(ev.first);
    cudaEventDestroy(ev.second);
  }
  g_prof_events.clear();
  if (main_kernel_ms_total) *main_kernel_ms_total = total;
  if (main_kernel_launches) *main_kernel_launches = n;
  return PCV_OK;
}

int pcv_debug_read(uint32_t* out, int32_t n) {
  PCV_REQUIRE(out != nullptr && n >= 0, PCV_ERR_INVALID, "debug_read: bad argument");
  return debug_read(out, n);
}

int pcv_debug_trace_read(uint64_t*, int32_t) {
  set_error("debug_trace_read: the kernels record no clock trace");
  return PCV_ERR_UNSUPPORTED;
}

int pcv_debug_plan(int32_t B, int32_t H, int32_t N, int32_t M, int32_t workers, int32_t rows_per_unit,
                   int32_t rows_per_tile, int32_t* segs, int32_t max_segs, int32_t* counts) {
  PCV_REQUIRE(B > 0 && H > 0 && N > 0 && M > 0 && workers > 0, PCV_ERR_INVALID, "debug_plan: sizes must be positive");
  PCV_REQUIRE(rows_per_tile == 128 && (rows_per_unit == 128 || rows_per_unit == 256 || rows_per_unit == 512),
              PCV_ERR_INVALID, "debug_plan: rows_per_tile must be 128 and rows_per_unit 128, 256 or 512");
  PCV_REQUIRE(counts != nullptr && (segs != nullptr || max_segs == 0), PCV_ERR_INVALID, "debug_plan: NULL argument");
  return debug_plan(B, H, N, M, workers, rows_per_unit, rows_per_tile, segs, max_segs, counts);
}

int pcv_debug_pair_workers(int32_t* workers, int32_t* clusters_fit) {
  PCV_REQUIRE(workers != nullptr && clusters_fit != nullptr, PCV_ERR_INVALID, "debug_pair_workers: NULL argument");
  return debug_pair_workers(workers, clusters_fit);
}

uint64_t pcv_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int pcv_get_device_info(pcv_device_info* info) {
  PCV_REQUIRE(info != nullptr, PCV_ERR_INVALID, "device_info: NULL argument");
  int dev = 0;
  PCV_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  PCV_CHECK_CUDA(cudaGetDeviceProperties(&prop, dev));
  info->device = dev;
  info->sm_major = prop.major;
  info->sm_minor = prop.minor;
  info->num_sms = prop.multiProcessorCount;
  info->smem_optin_bytes = (int)prop.sharedMemPerBlockOptin;
  info->tcgen05_ok = (prop.major == 9) ? 1 : 0;
  return PCV_OK;
}

int pcv_attn_supported_tcgen05(const pcv_attn_params* p) {
  if (validate_attn(p) != PCV_OK) return 0;
  const char* why = "";
  const bool ok = attn_tc_supported(*p, &why);
  if (!ok) set_error("tcgen05 path not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_attn_workspace_bytes(const pcv_attn_params* p, size_t* bytes) {
  int rc = validate_attn(p, true);
  if (rc != PCV_OK) return rc;
  PCV_REQUIRE(bytes != nullptr, PCV_ERR_INVALID, "attn: bytes is NULL");
  if (p->dtype == PCV_E4M3) return attn_tc_workspace_bytes(*p, bytes);  // pcv_attn_fwd_fp8: the tensor-core kernel
  const char* why = "";
  if (use_decode(*p, &why)) return attn_decode_workspace_bytes(*p, bytes);
  PCV_REQUIRE(p->impl != PCV_IMPL_DECODE, PCV_ERR_UNSUPPORTED, "attn: decode kernel requested but %s", why);
  if (use_tc(*p, &why)) return attn_tc_workspace_bytes(*p, bytes);
  PCV_REQUIRE(p->impl != PCV_IMPL_TCGEN05 && p->impl != PCV_IMPL_TCGEN05_PAIR, PCV_ERR_UNSUPPORTED,
              "attn: tcgen05 kernel requested but %s", why);
  return attn_simt_workspace_bytes(*p, bytes);
}

int pcv_attn_fwd(const pcv_attn_params* p, void* stream) {
  int rc = validate_attn(p);
  if (rc != PCV_OK) return rc;
  const char* why = "";
  if (use_decode(*p, &why)) return launch_attn_decode(*p, nullptr, nullptr, reinterpret_cast<cudaStream_t>(stream));
  PCV_REQUIRE(p->impl != PCV_IMPL_DECODE, PCV_ERR_UNSUPPORTED, "attn: decode kernel requested but %s", why);
  if (use_tc(*p, &why)) return launch_attn_tc(*p, reinterpret_cast<cudaStream_t>(stream));
  PCV_REQUIRE(p->impl != PCV_IMPL_TCGEN05 && p->impl != PCV_IMPL_TCGEN05_PAIR, PCV_ERR_UNSUPPORTED,
              "attn: tcgen05 kernel requested but %s", why);
  return launch_attn_simt(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_fwd_sharded_supported(const pcv_attn_params* p) {
  if (validate_attn(p) != PCV_OK) return 0;
  const char* why = "";
  const bool ok = p->impl != PCV_IMPL_SIMT && attn_tc_fuse_supported(*p, &why);
  if (!ok) set_error("fused M-shard merge not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_attn_fwd_sharded(const pcv_attn_params* p, const pcv_shard_fuse* f, void* stream) {
  PCV_REQUIRE(p != nullptr && f != nullptr, PCV_ERR_INVALID, "attn_fwd_sharded: NULL argument");
  PCV_REQUIRE(f->num_peers >= 1 && f->num_peers <= PCV_MAX_PEERS && f->rank >= 0 && f->rank < f->num_peers, PCV_ERR_INVALID,
              "attn_fwd_sharded: rank %d of %d", f->rank, f->num_peers);
  PCV_REQUIRE(f->epoch >= 1, PCV_ERR_INVALID, "attn_fwd_sharded: epoch must start at 1");
  for (int g = 0; g < f->num_peers; ++g)
    PCV_REQUIRE(f->part[g] && f->out[g] && f->flags[g], PCV_ERR_INVALID, "attn_fwd_sharded: NULL buffer of rank %d", g);
  // the tail loads 16 bytes of every part[g] row, stores 8 bytes (4 channels) of every out[g] row at o_off + 4 * lane
  // and spins on 32-bit flag words: refuse what those accesses cannot address instead of faulting on the device
  for (int g = 0; g < f->num_peers; ++g) {
    PCV_REQUIRE(al16(f->part[g]), PCV_ERR_INVALID, "attn_fwd_sharded: part[%d] must be 16-byte aligned", g);
    PCV_REQUIRE((reinterpret_cast<uintptr_t>(f->out[g]) & 7u) == 0, PCV_ERR_INVALID,
                "attn_fwd_sharded: out[%d] must be 8-byte aligned", g);
    PCV_REQUIRE((reinterpret_cast<uintptr_t>(f->flags[g]) & 3u) == 0, PCV_ERR_INVALID,
                "attn_fwd_sharded: flags[%d] must be 4-byte aligned", g);
  }
  PCV_REQUIRE(((f->o_stride_b | f->o_stride_n | f->o_stride_h) & 3) == 0, PCV_ERR_INVALID,
              "attn_fwd_sharded: output strides (%lld, %lld, %lld) must be multiples of 4 elements",
              (long long)f->o_stride_b, (long long)f->o_stride_n, (long long)f->o_stride_h);
  pcv_attn_params q = *p;
  q.write_partial = 1;
  // validate_attn wants part_* for a partial launch; they are replaced by part[rank] inside the launcher
  q.part_o = reinterpret_cast<float*>(f->part[f->rank]);
  q.part_m = q.part_o;
  q.part_l = q.part_o;
  int rc = validate_attn(&q);
  if (rc != PCV_OK) return rc;
  return launch_attn_tc(q, reinterpret_cast<cudaStream_t>(stream), f);
}

int pcv_attn_combine(const pcv_combine_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "combine: params is NULL");
  return launch_combine(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_combine_peers(const pcv_peer_combine_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "combine_peers: params is NULL");
  return launch_combine_peers(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_merge_partials(const pcv_merge_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "merge_partials: params is NULL");
  return launch_merge_partials(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_partial_rescale(const pcv_rescale_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "rescale: params is NULL");
  return launch_rescale(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_rotary_apply(const pcv_rotary_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "rotary: params is NULL");
  return launch_rotary(*p, nullptr, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_kv_append(const pcv_kv_append_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "kv_append: params is NULL");
  return launch_kv_append(*p, nullptr, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_kv_project_supported(const pcv_kvproj_params* p) {
  if (p == nullptr) return 0;
  const char* why = "";
  const bool ok = kv_project_supported(*p, &why);
  if (!ok) set_error("kv_project not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_ln_stats(const pcv_ln_stats_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "ln_stats: params is NULL");
  return launch_ln_stats(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_kv_project(const pcv_kvproj_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "kv_project: params is NULL");
  return launch_kv_project(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_ln_linear_bwd_supported(const pcv_ln_linear_bwd_params* p) {
  if (p == nullptr) {
    set_error("ln_linear_bwd: params is NULL");
    return 0;
  }
  const char* why = "";
  const bool ok = ln_linear_bwd_supported(*p, &why);
  if (!ok) set_error("ln_linear_bwd not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_ln_linear_bwd_workspace_bytes(const pcv_ln_linear_bwd_params* p, size_t* bytes) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "ln_linear_bwd_workspace_bytes: params is NULL");
  return ln_linear_bwd_workspace_bytes(*p, bytes);
}

int pcv_ln_linear_bwd(const pcv_ln_linear_bwd_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "ln_linear_bwd: params is NULL");
  return launch_ln_linear_bwd(*p, reinterpret_cast<cudaStream_t>(stream));
}

// s == nullptr: the unsharded backward
static int bwd_check(const pcv_attn_bwd_params* p, const pcv_key_shard* s) {
  if (p == nullptr) return 0;
  const char* why = "";
  const bool ok = attn_bwd_supported(*p, s, &why);
  if (!ok) set_error("attn_bwd not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_attn_bwd_supported(const pcv_attn_bwd_params* p) { return bwd_check(p, nullptr); }

int pcv_attn_bwd_workspace_bytes(const pcv_attn_bwd_params* p, size_t* bytes) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "attn_bwd_workspace_bytes: params is NULL");
  return attn_bwd_workspace_bytes(*p, nullptr, bytes);
}

int pcv_attn_bwd(const pcv_attn_bwd_params* p, void* stream) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "attn_bwd: params is NULL");
  return launch_attn_bwd(*p, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_bwd_shard_supported(const pcv_attn_bwd_params* p, const pcv_key_shard* s) {
  if (s == nullptr) {
    set_error("attn_bwd_shard: shard is NULL");
    return 0;
  }
  return bwd_check(p, s);
}

int pcv_attn_bwd_shard_workspace_bytes(const pcv_attn_bwd_params* p, const pcv_key_shard* s, size_t* bytes) {
  PCV_REQUIRE(p != nullptr && s != nullptr, PCV_ERR_INVALID, "attn_bwd_shard_workspace_bytes: params or shard is NULL");
  return attn_bwd_workspace_bytes(*p, s, bytes);
}

int pcv_attn_bwd_shard(const pcv_attn_bwd_params* p, const pcv_key_shard* s, void* stream) {
  PCV_REQUIRE(p != nullptr && s != nullptr, PCV_ERR_INVALID, "attn_bwd_shard: params or shard is NULL");
  return launch_attn_bwd(*p, s, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_dropout_mask(uint8_t* keep, int32_t B, int32_t H, int32_t N, int32_t M, float dropout_p,
                          uint64_t dropout_seed, void* stream) {
  return launch_dropout_mask(keep, B, H, N, 0, M, dropout_p, dropout_seed, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_dropout_mask_range(uint8_t* keep, int32_t B, int32_t H, int32_t N, int32_t key_begin, int32_t key_end,
                                float dropout_p, uint64_t dropout_seed, void* stream) {
  return launch_dropout_mask(keep, B, H, N, key_begin, key_end, dropout_p, dropout_seed,
                             reinterpret_cast<cudaStream_t>(stream));
}

int pcv_sample_supported(const pcv_sample_params* p) { return sample_check(p) == PCV_OK ? 1 : 0; }

int pcv_sample(const pcv_sample_params* p, void* stream) {
  const int rc = sample_check(p);
  if (rc != PCV_OK) return rc;
  return launch_sample(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_sample_uniforms(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int32_t R,
                        int32_t rows_per_batch, void* stream) {
  return launch_sample_uniforms(out, seeds, positions, R, rows_per_batch, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_spec_verify_supported(const pcv_spec_verify_params* p) { return spec_verify_check(p) == PCV_OK ? 1 : 0; }

int pcv_spec_verify(const pcv_spec_verify_params* p, void* stream) {
  const int rc = spec_verify_check(p);
  if (rc != PCV_OK) return rc;
  return launch_spec_verify(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_spec_uniforms(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int32_t R, int32_t rows_per_batch,
                      int32_t stream_id, void* stream) {
  return launch_spec_uniforms(out, seeds, positions, R, rows_per_batch, stream_id,
                              reinterpret_cast<cudaStream_t>(stream));
}

int pcv_beam_step_supported(const pcv_beam_step_params* p) { return beam_step_check(p) == PCV_OK ? 1 : 0; }

int pcv_beam_step(const pcv_beam_step_params* p, void* stream) {
  const int rc = beam_step_check(p);
  if (rc != PCV_OK) return rc;
  return launch_beam_step(*p, false, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_beam_step_logprobs_supported(const pcv_beam_step_params* p) {
  return beam_step_check(p, true) == PCV_OK ? 1 : 0;
}

int pcv_beam_step_logprobs(const pcv_beam_step_params* p, void* stream) {
  const int rc = beam_step_check(p, true);
  if (rc != PCV_OK) return rc;
  return launch_beam_step(*p, true, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_logits_process_supported(const pcv_logits_process_params* p) {
  return logits_process_check(p) == PCV_OK ? 1 : 0;
}

int pcv_logits_process(const pcv_logits_process_params* p, void* stream) {
  const int rc = logits_process_check(p);
  if (rc != PCV_OK) return rc;
  return launch_logits_process(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_prompt_lookup_supported(const pcv_prompt_lookup_params* p) {
  return prompt_lookup_check(p) == PCV_OK ? 1 : 0;
}

int pcv_prompt_lookup(const pcv_prompt_lookup_params* p, void* stream) {
  const int rc = prompt_lookup_check(p);
  if (rc != PCV_OK) return rc;
  return launch_prompt_lookup(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_kv_gather_rows_supported(const pcv_kv_gather_params* p, const pcv_dev_rows* rows) {
  return kv_gather_check(p, rows) == PCV_OK ? 1 : 0;
}

int pcv_kv_gather_rows(const pcv_kv_gather_params* p, const pcv_dev_rows* rows, void* stream) {
  const int rc = kv_gather_check(p, rows);
  if (rc != PCV_OK) return rc;
  return launch_kv_gather(*p, *rows, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_contrastive_candidates_supported(const pcv_contrastive_candidates_params* p) {
  return contrastive_candidates_check(p) == PCV_OK ? 1 : 0;
}

int pcv_contrastive_candidates(const pcv_contrastive_candidates_params* p, void* stream) {
  const int rc = contrastive_candidates_check(p);
  if (rc != PCV_OK) return rc;
  return launch_contrastive_candidates(*p, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_contrastive_rank_supported(const pcv_contrastive_rank_params* p) {
  return contrastive_rank_check(p) == PCV_OK ? 1 : 0;
}

int pcv_contrastive_rank(const pcv_contrastive_rank_params* p, void* stream) {
  const int rc = contrastive_rank_check(p);
  if (rc != PCV_OK) return rc;
  return launch_contrastive_rank(*p, reinterpret_cast<cudaStream_t>(stream));
}

static int partial_dropout_check(const pcv_attn_params* p, float dropout_p, bool shard) {
  if (validate_attn(p) != PCV_OK) return 0;
  const char* why = "";
  const bool ok = partial_dropout_supported(*p, dropout_p, shard, &why);
  if (!ok) set_error("one-pass dropout forward not applicable: %s", why);
  return ok ? 1 : 0;
}

static int partial_dropout_launch(const pcv_attn_params* p, float dropout_p, uint64_t dropout_seed, bool shard,
                                  void* stream) {
  int rc = validate_attn(p);
  if (rc != PCV_OK) return rc;
  const char* why = "";
  PCV_REQUIRE(partial_dropout_supported(*p, dropout_p, shard, &why), PCV_ERR_UNSUPPORTED,
              "attn_fwd_partial_dropout: %s", why);
  const DropoutRule drop = dropout_rule(dropout_p, dropout_seed);
  return launch_attn_tc(*p, reinterpret_cast<cudaStream_t>(stream), nullptr, &drop);
}

int pcv_attn_fwd_partial_dropout_supported(const pcv_attn_params* p, float dropout_p) {
  return partial_dropout_check(p, dropout_p, false);
}

int pcv_attn_fwd_partial_dropout(const pcv_attn_params* p, float dropout_p, uint64_t dropout_seed, void* stream) {
  return partial_dropout_launch(p, dropout_p, dropout_seed, false, stream);
}

int pcv_attn_fwd_partial_dropout_shard_supported(const pcv_attn_params* p, float dropout_p) {
  return partial_dropout_check(p, dropout_p, true);
}

int pcv_attn_fwd_partial_dropout_shard(const pcv_attn_params* p, float dropout_p, uint64_t dropout_seed, void* stream) {
  return partial_dropout_launch(p, dropout_p, dropout_seed, true, stream);
}

int pcv_kv_project_fp8_supported(const pcv_kvproj_params* p, const pcv_kvproj_fp8* f) {
  if (p == nullptr || f == nullptr) {
    set_error("kv_project_fp8: params are NULL");
    return 0;
  }
  const char* why = "";
  const bool ok = kv_project_fp8_supported(*p, *f, &why);
  if (!ok) set_error("kv_project_fp8 not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_kv_project_fp8(const pcv_kvproj_params* p, const pcv_kvproj_fp8* f, void* stream) {
  PCV_REQUIRE(p != nullptr && f != nullptr, PCV_ERR_INVALID, "kv_project_fp8: params are NULL");
  return launch_kv_project_fp8(*p, *f, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_fwd_fp8_supported(const pcv_attn_params* p, const pcv_fp8_attn* f) {
  if (f == nullptr) {
    set_error("attn_fwd_fp8: fp8 params are NULL");
    return 0;
  }
  if (validate_attn(p, true) != PCV_OK) return 0;
  const char* why = "";
  const bool ok = attn_tc_fp8_supported(*p, *f, &why);
  if (!ok) set_error("FP8 attention forward not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_attn_fwd_fp8(const pcv_attn_params* p, const pcv_fp8_attn* f, void* stream) {
  PCV_REQUIRE(f != nullptr, PCV_ERR_INVALID, "attn_fwd_fp8: fp8 params are NULL");
  int rc = validate_attn(p, true);
  if (rc != PCV_OK) return rc;
  return launch_attn_tc_fp8(*p, *f, reinterpret_cast<cudaStream_t>(stream));
}

// The e4m3-row (fp8: f) and device-row (window: rows) decode entry points; each refuses a NULL f / rows it takes.
static int decode_check(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows, bool fp8,
                        bool window) {
  if ((fp8 && f == nullptr) || (window && rows == nullptr)) {
    if (fp8 && f == nullptr) set_error("%s: fp8 params are NULL", window ? "attn_decode_window_fp8" : "attn_decode_fp8");
    else set_error("attn_decode_window: rows is NULL");
    return 0;
  }
  if (validate_attn(p) != PCV_OK) return 0;
  const char* why = "";
  const bool ok = attn_decode_supported(*p, f, rows, &why);
  if (!ok) set_error("%s decode attention not applicable: %s", window ? "window" : "e4m3", why);
  return ok ? 1 : 0;
}

static int decode_launch(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows, bool fp8,
                         bool window, void* stream) {
  PCV_REQUIRE((f != nullptr || !fp8) && (rows != nullptr || !window), PCV_ERR_INVALID, "%s",
              !window ? "attn_decode_fp8: fp8 params are NULL"
                      : (fp8 ? "attn_decode_window_fp8: fp8 params or rows are NULL" : "attn_decode_window: rows is NULL"));
  int rc = validate_attn(p);
  if (rc != PCV_OK) return rc;
  const char* why = "";
  PCV_REQUIRE(attn_decode_supported(*p, f, rows, &why), PCV_ERR_UNSUPPORTED, "%s decode attention: %s",
              window ? "window" : "e4m3", why);
  return launch_attn_decode(*p, f, rows, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_decode_fp8_supported(const pcv_attn_params* p, const pcv_decode_fp8* f) {
  return decode_check(p, f, nullptr, true, false);
}

int pcv_attn_decode_fp8_workspace_bytes(const pcv_attn_params* p, size_t* bytes) {
  int rc = validate_attn(p);
  if (rc != PCV_OK) return rc;
  PCV_REQUIRE(bytes != nullptr, PCV_ERR_INVALID, "attn_decode_fp8: bytes is NULL");
  return attn_decode_workspace_bytes(*p, bytes);
}

int pcv_attn_decode_fp8(const pcv_attn_params* p, const pcv_decode_fp8* f, void* stream) {
  return decode_launch(p, f, nullptr, true, false, stream);
}

// The tensor-core attention of 1 to 64 query rows (pcv_attn_cached.cu) on a whole e4m3 cache or, for the window
// entries (window), on a device-resident window of an arena; the e4m3 entries (fp8) refuse a NULL f.
static int cached_check(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows, int32_t band,
                        bool fp8, bool window) {
  const char* name = !window ? "attn_cached_fp8" : (fp8 ? "attn_cached_window_fp8" : "attn_cached_window");
  PCV_REQUIRE(!fp8 || f != nullptr, PCV_ERR_INVALID, "%s: fp8 params are NULL", name);
  PCV_REQUIRE(!window || rows != nullptr, PCV_ERR_INVALID, "%s: rows is NULL", name);
  int rc = validate_attn(p);
  if (rc != PCV_OK) return rc;
  const char* why = "";
  PCV_REQUIRE(attn_cached_supported(*p, f, rows, band, &why), PCV_ERR_UNSUPPORTED, "%s not applicable: %s",
              window ? name : "cached e4m3 attention", why);
  return PCV_OK;
}

static int cached_workspace(const pcv_attn_params* p, size_t* bytes, const char* name) {
  int rc = validate_attn(p);
  if (rc != PCV_OK) return rc;
  PCV_REQUIRE(bytes != nullptr, PCV_ERR_INVALID, "%s: bytes is NULL", name);
  return attn_cached_workspace_bytes(*p, bytes);
}

int pcv_attn_cached_fp8_supported(const pcv_attn_params* p, const pcv_decode_fp8* f) {
  return cached_check(p, f, nullptr, 0, true, false) == PCV_OK ? 1 : 0;
}

int pcv_attn_cached_fp8_workspace_bytes(const pcv_attn_params* p, size_t* bytes) {
  return cached_workspace(p, bytes, "attn_cached_fp8");
}

int pcv_attn_cached_fp8(const pcv_attn_params* p, const pcv_decode_fp8* f, void* stream) {
  const int rc = cached_check(p, f, nullptr, 0, true, false);
  if (rc != PCV_OK) return rc;
  return launch_attn_cached(*p, f, nullptr, 0, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_kv_append_fp8_supported(const pcv_kv_append_params* p, const pcv_kv_fp8_scales* f) {
  if (p == nullptr || f == nullptr) {
    set_error("kv_append_fp8: params are NULL");
    return 0;
  }
  const char* why = "";
  const bool ok = kv_append_fp8_supported(*p, *f, &why);
  if (!ok) set_error("kv_append_fp8 not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_kv_append_fp8(const pcv_kv_append_params* p, const pcv_kv_fp8_scales* f, void* stream) {
  PCV_REQUIRE(p != nullptr && f != nullptr, PCV_ERR_INVALID, "kv_append_fp8: params are NULL");
  return launch_kv_append(*p, f, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_rotary_fp8_supported(const pcv_rotary_params* p, const pcv_rotary_fp8* f) {
  if (p == nullptr || f == nullptr) {
    set_error("rotary_fp8: params are NULL");
    return 0;
  }
  const char* why = "";
  const bool ok = rotary_fp8_supported(*p, *f, &why);
  if (!ok) set_error("rotary_fp8 not applicable: %s", why);
  return ok ? 1 : 0;
}

int pcv_rotary_apply_fp8(const pcv_rotary_params* p, const pcv_rotary_fp8* f, void* stream) {
  PCV_REQUIRE(p != nullptr && f != nullptr, PCV_ERR_INVALID, "rotary_fp8: params are NULL");
  return launch_rotary(*p, f, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_decode_window_supported(const pcv_attn_params* p, const pcv_dev_rows* rows) {
  return decode_check(p, nullptr, rows, false, true);
}

int pcv_attn_decode_window_fp8_supported(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows) {
  return decode_check(p, f, rows, true, true);
}

int pcv_attn_decode_window_workspace_bytes(const pcv_attn_params* p, size_t* bytes) {
  int rc = validate_attn(p);
  if (rc != PCV_OK) return rc;
  PCV_REQUIRE(bytes != nullptr, PCV_ERR_INVALID, "attn_decode_window: bytes is NULL");
  return attn_decode_workspace_bytes(*p, bytes);
}

int pcv_attn_decode_window(const pcv_attn_params* p, const pcv_dev_rows* rows, void* stream) {
  return decode_launch(p, nullptr, rows, false, true, stream);
}

int pcv_attn_decode_window_fp8(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows,
                               void* stream) {
  return decode_launch(p, f, rows, true, true, stream);
}

int pcv_attn_cached_window_supported(const pcv_attn_params* p, const pcv_dev_rows* rows, int32_t band) {
  return cached_check(p, nullptr, rows, band, false, true) == PCV_OK ? 1 : 0;
}

int pcv_attn_cached_window_fp8_supported(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows,
                                         int32_t band) {
  return cached_check(p, f, rows, band, true, true) == PCV_OK ? 1 : 0;
}

int pcv_attn_cached_window_workspace_bytes(const pcv_attn_params* p, size_t* bytes) {
  return cached_workspace(p, bytes, "attn_cached_window");
}

int pcv_attn_cached_window_fp8_workspace_bytes(const pcv_attn_params* p, size_t* bytes) {
  return cached_workspace(p, bytes, "attn_cached_window_fp8");
}

int pcv_attn_cached_window(const pcv_attn_params* p, const pcv_dev_rows* rows, int32_t band, void* stream) {
  const int rc = cached_check(p, nullptr, rows, band, false, true);
  if (rc != PCV_OK) return rc;
  return launch_attn_cached(*p, nullptr, rows, band, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_attn_cached_window_fp8(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows,
                               int32_t band, void* stream) {
  const int rc = cached_check(p, f, rows, band, true, true);
  if (rc != PCV_OK) return rc;
  return launch_attn_cached(*p, f, rows, band, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_kv_append_at(const pcv_kv_append_params* p, const pcv_dev_rows* rows, void* stream) {
  PCV_REQUIRE(p != nullptr && rows != nullptr, PCV_ERR_INVALID, "kv_append_at: params or rows are NULL");
  return launch_kv_append(*p, nullptr, rows, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_kv_append_at_fp8(const pcv_kv_append_params* p, const pcv_kv_fp8_scales* f, const pcv_dev_rows* rows,
                         void* stream) {
  PCV_REQUIRE(p != nullptr && f != nullptr && rows != nullptr, PCV_ERR_INVALID, "kv_append_at_fp8: params are NULL");
  return launch_kv_append(*p, f, rows, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_rotary_apply_at(const pcv_rotary_params* p, const pcv_dev_rows* rows, void* stream) {
  PCV_REQUIRE(p != nullptr && rows != nullptr, PCV_ERR_INVALID, "rotary_at: params or rows are NULL");
  return launch_rotary(*p, nullptr, rows, reinterpret_cast<cudaStream_t>(stream));
}

int pcv_rotary_apply_at_fp8(const pcv_rotary_params* p, const pcv_rotary_fp8* f, const pcv_dev_rows* rows,
                            void* stream) {
  PCV_REQUIRE(p != nullptr && f != nullptr && rows != nullptr, PCV_ERR_INVALID, "rotary_at_fp8: params are NULL");
  return launch_rotary(*p, f, rows, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
