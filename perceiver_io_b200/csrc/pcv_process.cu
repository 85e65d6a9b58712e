// pcv_process.cu — logits processors on the device (pcv_logits_process): the repetition penalty, n-gram blocking and
// minimum new tokens of the Hugging Face logits processors, on fp32 rows, before the sampler, the beam step or the
// contrastive candidates read them.  The rule is stated in include/pcv_attn.h.
//
// process_kernel, one 512-thread CTA per processed row: stages the row as fp32 in V floats of dynamic shared memory
// (optionally replaced by its log-softmax, with beam_rows_kernel's arithmetic), marks the history's ids in a V-bit
// shared bitmap and rescales the marked ids once each (so duplicates apply once, without any order between threads),
// then lets the threads over the n-gram starts write -inf to the banned ids (a benign race: every writer writes the
// same value), then the EOS ids, then writes the row out.  The history lengths are read from device memory when the
// kernel runs.  No floating-point atomics: a row's output is a pure function of its inputs.
#include "pcv_vocab.cuh"

namespace pcv {

namespace {

constexpr int kMaxNgram = PCV_PROCESS_MAX_NGRAM;

__device__ __forceinline__ int clamp_len(int n, int cap) { return n < 0 ? 0 : n > cap ? cap : n; }

template <typename T>
__global__ void __launch_bounds__(kThreads) process_kernel(const pcv_logits_process_params p) {
  extern __shared__ __align__(16) float xs[];
  __shared__ uint32_t seen[PCV_SAMPLE_MAX_VOCAB / 32];
  __shared__ int64_t suffix[kMaxNgram - 1];   // the history's last N - 1 ids
  const int V = p.V, tid = threadIdx.x, r = blockIdx.x;
  const int64_t row = p.row_map ? (int64_t)r * p.row_group + p.row_map[r] : r;
  const T* src = static_cast<const T*>(p.logits) + row * p.stride_row;

  // ---- the fp32 row, or its log-softmax ----
  if (p.log_softmax) {
    const RowStats st = stage_max_sum(src, V, xs);
    const double logS = log(st.S);
    for (int i = tid; i < V; i += kThreads) {
      const double d = (double)xs[i] - (double)st.m;
      xs[i] = __double2float_rn(d - logS);
    }
  } else {
    for (int i = tid; i < V; i += kThreads) xs[i] = load_f(src + i);
  }

  // ---- the history: prefix then tail ----
  const int h = r / p.rows_per_hist;
  const int Lp = clamp_len(p.prefix_len ? p.prefix_len[(int64_t)r * p.prefix_len_stride] : p.prefix_count,
                           p.prefix_cap);
  const int Lt = p.tail_len ? clamp_len(p.tail_len[(int64_t)r * p.tail_len_stride], p.tail_cap) : 0;
  const int L = Lp + Lt;
  const int64_t* pre = p.prefix + (int64_t)h * p.prefix_stride;
  const int64_t* tail = p.tail ? p.tail + (int64_t)h * p.tail_stride : nullptr;
  auto tok = [&](int j) -> int64_t { return j < Lp ? pre[j] : tail[j - Lp]; };

  // ---- 1. repetition penalty: mark, then rescale each marked id once ----
  if (p.repetition_penalty != 1.0f) {
    const int words = (V + 31) / 32;
    for (int w = tid; w < words; w += kThreads) seen[w] = 0u;
    __syncthreads();
    for (int j = tid; j < L; j += kThreads) {
      const int64_t id = tok(j);
      if (id >= 0 && id < V) atomicOr(seen + (id >> 5), 1u << (id & 31));
    }
    __syncthreads();
    const float theta = p.repetition_penalty;
    for (int i = tid; i < V; i += kThreads) {
      if ((seen[i >> 5] >> (i & 31)) & 1u) {
        const float x = xs[i];
        xs[i] = x < 0.0f ? __fmul_rn(x, theta) : __fdiv_rn(x, theta);
      }
    }
  }
  __syncthreads();

  // ---- 2. n-gram blocking: start s bans hist[s + N - 1] when hist[s .. s+N-1) equals the last N - 1 ids ----
  const int N = p.no_repeat_ngram;
  if (N > 0 && L + 1 >= N) {   // uniform over the CTA
    if (tid < N - 1) suffix[tid] = tok(L - N + 1 + tid);
    __syncthreads();
    for (int s = tid; s < L - N + 1; s += kThreads) {
      bool match = true;
      for (int j = 0; j < N - 1 && match; ++j) match = tok(s + j) == suffix[j];
      const int64_t id = tok(s + N - 1);
      if (match && id >= 0 && id < V) xs[id] = -INFINITY;
    }
  }

  // ---- 3. minimum new tokens ----
  if (p.min_new_tokens > 0 && L - p.prompt_len < p.min_new_tokens && tid < p.n_eos) xs[p.eos[tid]] = -INFINITY;
  __syncthreads();

  float* out = p.out + row * p.out_stride_row;
  for (int i = tid; i < V; i += kThreads) out[i] = xs[i];
}

}  // namespace

int logits_process_check(const pcv_logits_process_params* p) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "logits_process: params is NULL");
  PCV_REQUIRE(p->logits && p->out && p->prefix, PCV_ERR_INVALID, "logits_process: a pointer is NULL");
  PCV_REQUIRE(p->tail || !p->tail_len, PCV_ERR_INVALID, "logits_process: tail_len is set without a tail");
  PCV_REQUIRE(p->dtype == PCV_BF16 || p->dtype == PCV_F16 || p->dtype == PCV_F32, PCV_ERR_INVALID,
              "logits_process: unknown dtype %d (bf16, fp16 or fp32 logits)", p->dtype);
  PCV_REQUIRE(p->V >= 1 && p->V <= PCV_SAMPLE_MAX_VOCAB, PCV_ERR_UNSUPPORTED,
              "logits_process: V=%d must be in [1, %d]", p->V, PCV_SAMPLE_MAX_VOCAB);
  PCV_REQUIRE(p->R >= 1, PCV_ERR_INVALID, "logits_process: R=%d must be >= 1", p->R);
  PCV_REQUIRE(p->stride_row >= p->V && p->out_stride_row >= p->V, PCV_ERR_INVALID,
              "logits_process: stride_row=%lld and out_stride_row=%lld must be >= V=%d", (long long)p->stride_row,
              (long long)p->out_stride_row, p->V);
  PCV_REQUIRE(!p->row_map || p->row_group >= 1, PCV_ERR_INVALID,
              "logits_process: row_group=%d must be >= 1 with a row map", p->row_group);
  PCV_REQUIRE(p->rows_per_hist >= 1, PCV_ERR_INVALID, "logits_process: rows_per_hist=%d must be >= 1",
              p->rows_per_hist);
  PCV_REQUIRE(p->log_softmax == 0 || p->log_softmax == 1, PCV_ERR_INVALID,
              "logits_process: log_softmax=%d must be 0 or 1", p->log_softmax);
  PCV_REQUIRE(p->prefix_count >= 0 && p->prefix_cap >= 0 && p->tail_cap >= 0 && p->prefix_stride >= 0 &&
                  p->tail_stride >= 0 && p->prefix_len_stride >= 0 && p->tail_len_stride >= 0,
              PCV_ERR_INVALID, "logits_process: history counts, caps and strides must be >= 0");
  PCV_REQUIRE(isfinite(p->repetition_penalty) && p->repetition_penalty > 0.0f, PCV_ERR_INVALID,
              "logits_process: repetition_penalty=%g must be finite and > 0 (1: off)", (double)p->repetition_penalty);
  PCV_REQUIRE(p->no_repeat_ngram >= 0 && p->no_repeat_ngram <= PCV_PROCESS_MAX_NGRAM, PCV_ERR_UNSUPPORTED,
              "logits_process: no_repeat_ngram=%d must be in [0, %d] (0: off)", p->no_repeat_ngram,
              PCV_PROCESS_MAX_NGRAM);
  PCV_REQUIRE(p->min_new_tokens >= 0, PCV_ERR_INVALID, "logits_process: min_new_tokens=%d must be >= 0 (0: off)",
              p->min_new_tokens);
  PCV_REQUIRE(p->n_eos >= 0 && p->n_eos <= PCV_PROCESS_MAX_EOS, PCV_ERR_UNSUPPORTED,
              "logits_process: n_eos=%d must be in [0, %d]", p->n_eos, PCV_PROCESS_MAX_EOS);
  PCV_REQUIRE(p->min_new_tokens == 0 || p->n_eos > 0, PCV_ERR_INVALID,
              "logits_process: min_new_tokens=%d needs EOS ids (it bans them until enough tokens are new)",
              p->min_new_tokens);
  for (int e = 0; e < p->n_eos; ++e)
    PCV_REQUIRE(p->eos[e] >= 0 && p->eos[e] < p->V, PCV_ERR_INVALID,
                "logits_process: EOS id %d is outside [0, V=%d)", p->eos[e], p->V);
  return PCV_OK;
}

int launch_logits_process(const pcv_logits_process_params& p, cudaStream_t stream) {
  void (*const kern[3])(pcv_logits_process_params) = {process_kernel<__nv_bfloat16>, process_kernel<__half>,
                                                      process_kernel<float>};
  return launch_row_kernel(kern, p.dtype, p.V, p.R, p, stream);
}

}  // namespace pcv
