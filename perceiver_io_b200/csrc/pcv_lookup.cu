// pcv_lookup.cu — prompt-lookup drafts on the device (pcv_prompt_lookup): each batch row's drafts are the ids that
// followed the first earlier occurrence of its latest n-gram, with the rule of the Hugging Face
// PromptLookupCandidateGenerator; round mode first settles the speculative round that just ran.  The rule is stated in
// include/pcv_attn.h.
//
// lookup_kernel, one 256-thread CTA per batch row: thread 0 settles the round (round mode), the row's last N ids are
// staged in shared memory, the threads stride over window ends e and compute the backward match length l(e) <= N
// against them; a window of n ids ends at e exactly when l(e) >= n, and each thread keeps, per n, its first such e (its
// ends ascend).  A block-min per n (warp reductions, then one warp over the warps) gives the first window of every
// size; thread 0 takes the largest size that has one and writes the draft.  Integer comparisons and minima only: the
// result does not depend on the order in which threads finish.
#include "pcv_common.cuh"

namespace pcv {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxNgram = PCV_LOOKUP_MAX_NGRAM;
constexpr int kNone = 0x7fffffff;

__device__ __forceinline__ bool is_eos(const pcv_prompt_lookup_params& p, int64_t id) {
  bool hit = false;
  for (int e = 0; e < p.n_eos; ++e) hit |= id == p.eos[e];
  return hit;
}

__global__ void __launch_bounds__(kThreads) lookup_kernel(const pcv_prompt_lookup_params p) {
  __shared__ int64_t suffix[kMaxNgram];     // suffix[j] = h[len - 1 - j]
  __shared__ int first[kWarps][kMaxNgram];  // per warp and window size, the first window end
  __shared__ int row_state[3];              // [L, limit, search]
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int64_t* ids = p.ids + (int64_t)b * p.ids_stride;
  const int base = p.length[(int64_t)b * p.length_stride] + p.length_offset;

  // ---- round mode: settle the round that fed k tokens (thread 0), write t where it will be fed ----
  if (tid == 0) {
    int L = base, limit = p.limit ? p.limit[b] : p.G, search = 1;
    if (p.k > 0) {
      const int64_t* fed = p.fed + (int64_t)b * p.k;
      const int64_t* draws = p.draws + (int64_t)b * p.k;
      const int c = min(max(p.counts[b], 0), p.k - 1);
      int n = 0;
      int64_t t = fed[0];
      if (p.unfinished[b] != 0 && p.left[b] > 0) {
        while (n < c && fed[n + 1] == draws[n]) ++n;
        t = draws[n];
        p.left[b] -= n + 1;
        if (is_eos(p, t)) p.unfinished[b] = 0;
        L = base + n;
        const int row = min(max(L - 1, 0), p.cap - 1);
        ids[row] = t;
        search = p.unfinished[b] != 0 && p.left[b] > 0;
        limit = p.left[b] - 1;
      } else {
        L = base - 1;   // the history ends at t_0: its filler is t_0
        search = 0;
      }
      p.accepted[b] = n;
      p.t0[(int64_t)b * p.t0_stride] = t;
    }
    row_state[0] = min(max(L, 0), p.cap);
    row_state[1] = min(max(limit, 0), p.G);
    row_state[2] = search;
  }
  __syncthreads();   // also makes thread 0's write of t visible to the CTA
  const int L = row_state[0], limit = row_state[1];
  const int s = p.start ? min(max(p.start[b], 0), L) : 0;
  const int64_t* h = ids + s;
  const int len = L - s;
  const int nmax = row_state[2] ? min(p.N, len - 1) : 0;   // uniform over the CTA

  // ---- the first window end of every size ----
  if (tid < nmax) suffix[tid] = h[len - 1 - tid];
  __syncthreads();
  int best[kMaxNgram];
#pragma unroll
  for (int q = 0; q < kMaxNgram; ++q) best[q] = kNone;
  if (nmax > 0) {
    const int64_t last = suffix[0];
    for (int e = tid; e <= len - 2; e += kThreads) {
      if (h[e] != last) continue;
      int m = 1;
      while (m < nmax && m <= e && h[e - m] == suffix[m]) ++m;
#pragma unroll
      for (int q = 0; q < kMaxNgram; ++q)
        if (q < m && best[q] == kNone) best[q] = e;   // a window of q + 1 ids ends at e
    }
  }
#pragma unroll
  for (int q = 0; q < kMaxNgram; ++q) {
    const int w = __reduce_min_sync(0xffffffffu, best[q]);
    if (lane == 0) first[warp][q] = w;
  }
  __syncthreads();

  // ---- the draft of the largest size that has a window ----
  if (tid == 0) {
    int e = kNone;
    for (int q = nmax - 1; q >= 0 && e == kNone; --q) {
      int w = kNone;
      for (int i = 0; i < kWarps; ++i) w = min(w, first[i][q]);
      e = w;
    }
    int count = 0;
    if (e != kNone) {
      const int end = min(e + 1 + p.G, len);
      while (e + 1 + count < end && !is_eos(p, h[e + 1 + count])) ++count;
      count = min(count, limit);
    }
    int64_t* d = p.drafts + (int64_t)b * p.drafts_stride;
    const int64_t filler = len > 0 ? h[len - 1] : 0;
    for (int j = 0; j < p.G; ++j) d[j] = j < count ? h[e + 1 + j] : filler;
    p.counts[b] = count;
  }
}

}  // namespace

int prompt_lookup_check(const pcv_prompt_lookup_params* p) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "prompt_lookup: params is NULL");
  PCV_REQUIRE(p->ids && p->length && p->drafts && p->counts, PCV_ERR_INVALID, "prompt_lookup: a pointer is NULL");
  PCV_REQUIRE(p->B >= 1, PCV_ERR_INVALID, "prompt_lookup: B=%d must be >= 1", p->B);
  PCV_REQUIRE(p->cap >= 1, PCV_ERR_INVALID, "prompt_lookup: cap=%d must be >= 1", p->cap);
  PCV_REQUIRE(p->ids_stride >= p->cap, PCV_ERR_INVALID, "prompt_lookup: ids_stride=%lld is below cap=%d",
              (long long)p->ids_stride, p->cap);
  PCV_REQUIRE(p->length_stride >= 0, PCV_ERR_INVALID, "prompt_lookup: length_stride=%d must be >= 0",
              p->length_stride);
  PCV_REQUIRE(p->G >= 1 && p->G <= PCV_LOOKUP_MAX_DRAFTS, PCV_ERR_UNSUPPORTED, "prompt_lookup: G=%d must be in [1, %d]",
              p->G, PCV_LOOKUP_MAX_DRAFTS);
  PCV_REQUIRE(p->N >= 1 && p->N <= PCV_LOOKUP_MAX_NGRAM, PCV_ERR_UNSUPPORTED, "prompt_lookup: N=%d must be in [1, %d]",
              p->N, PCV_LOOKUP_MAX_NGRAM);
  PCV_REQUIRE(p->n_eos >= 0 && p->n_eos <= PCV_LOOKUP_MAX_EOS, PCV_ERR_UNSUPPORTED,
              "prompt_lookup: n_eos=%d must be in [0, %d]", p->n_eos, PCV_LOOKUP_MAX_EOS);
  PCV_REQUIRE(p->drafts_stride >= p->G, PCV_ERR_INVALID, "prompt_lookup: drafts_stride=%lld is below G=%d",
              (long long)p->drafts_stride, p->G);
  PCV_REQUIRE(p->k >= 0 && p->k <= p->G + 1, PCV_ERR_INVALID, "prompt_lookup: k=%d must be in [0, G+1=%d]", p->k,
              p->G + 1);
  if (p->k > 0) {
    PCV_REQUIRE(p->fed && p->draws && p->t0 && p->accepted && p->unfinished && p->left, PCV_ERR_INVALID,
                "prompt_lookup: a round (k=%d) needs fed, draws, t0, accepted, unfinished and left", p->k);
    PCV_REQUIRE(p->t0_stride >= 1, PCV_ERR_INVALID, "prompt_lookup: t0_stride=%lld must be >= 1",
                (long long)p->t0_stride);
  }
  return PCV_OK;
}

int launch_prompt_lookup(const pcv_prompt_lookup_params& p, cudaStream_t stream) {
  lookup_kernel<<<p.B, kThreads, 0, stream>>>(p);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

}  // namespace pcv
