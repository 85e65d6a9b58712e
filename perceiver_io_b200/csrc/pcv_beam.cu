// pcv_beam.cu — beam search on the device: one beam step (pcv_beam_step) with the semantics of 🤗's
// GenerationMixin._beam_search (do_sample=False; logits processors through pcv_logits_process and
// pcv_beam_step_logprobs, which starts from processed log-probabilities), and the KV-arena gather of the generated rows
// that follows it (pcv_kv_gather_rows).  oracle/beam_oracle.py restates the step in numpy.
//
// pcv_beam_step, two launches, no host read:
//   beam_rows_kernel, one CTA of 512 threads per beam row (b, k): stages the row's fp32 logits in shared memory,
//     logp_i = fp32(d_i - log S) with d_i = (double)x_i - (double)max and S = Σ exp(d_i) in fp64 (fixed order),
//     acc_i = fp32(running_score + logp_i) in place, then the row's top beams_to_keep by a radix select over
//     order-preserving keys, the lowest index first on ties.  The item's top beams_to_keep take at most beams_to_keep
//     candidates from one row, so the row's top set holds every candidate the item's can take from it.
//   beam_item_kernel, one CTA per batch item: ranks the K * beams_to_keep row candidates (score descending, flat index
//     k * V + token ascending), then runs 🤗's running-beam selection, finished-set merge and early-stop heuristic on
//     the state buffers (serially, in one thread: at most 40 candidates), gathers the token histories by parent and
//     writes the next tokens and parents.  The last CTA to finish (an integer atomic counter) sets "every item done"
//     and advances the generated count, which every launch reads from device memory: one recorded graph serves every
//     step.
// A row's result is a pure function of its item's logit bits and state: independent of B, of the launch and of graph
// capture.  No floating-point atomics.
//
// pcv_kv_gather_rows: for every beam row whose parent is another row, copy the parent's generated rows [first row,
// current row) of every arena in the table into the child's, through a scratch region in two launches (parent ->
// scratch, scratch -> child), so cycles and many-to-one moves read only pre-step rows.  With last_rows > 0 only the
// newest last_rows of them move (contrastive search: the rows of an item differ only in the row just appended).
#include "pcv_vocab.cuh"

namespace pcv {

namespace {

constexpr int kMaxKeep = (PCV_BEAM_MAX_EOS + 1) * PCV_BEAM_MAX_BEAMS;   // beams_to_keep at most
constexpr int kMaxCand = PCV_BEAM_MAX_BEAMS * kMaxKeep;                 // row candidates of one item
constexpr float kNeg = -1.0e9f;

__device__ __forceinline__ int keep_count(const pcv_beam_step_params& p) {
  return (p.n_eos + 1 > 2 ? p.n_eos + 1 : 2) * p.K;
}

// the step's params, and whether its rows already are fp32 log-probabilities (pcv_beam_step_logprobs: logp_i = x_i)
struct BeamRows {
  pcv_beam_step_params p;
  int logprobs;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) beam_rows_kernel(const BeamRows a) {
  const pcv_beam_step_params& p = a.p;
  extern __shared__ __align__(16) float xs[];   // the row's x, then its acc (V floats)
  __shared__ uint32_t ckey[kMaxKeep];
  __shared__ int32_t cidx[kMaxKeep];
  const int V = p.V, tid = threadIdx.x;
  const int row = blockIdx.x, k = row % p.K, keep = keep_count(p);
  const T* src = static_cast<const T*>(p.logits) + (int64_t)row * p.stride_row;

  // ---- logp and acc ----
  const float run = p.running_scores[row];
  if (a.logprobs) {
    for (int i = tid; i < V; i += kThreads) xs[i] = __fadd_rn(run, load_f(src + i));
  } else {
    const RowStats st = stage_max_sum(src, V, xs);
    const double logS = log(st.S);
    for (int i = tid; i < V; i += kThreads) {
      const double d = (double)xs[i] - (double)st.m;
      xs[i] = __fadd_rn(run, __double2float_rn(d - logS));
    }
  }

  // ---- the nsel-th largest key, and the nsel candidates ----
  const int nsel = keep < V ? keep : V;
  const uint32_t thr = select_key(xs, V, (uint32_t)nsel);
  collect_top(xs, V, (uint32_t)nsel, thr, ckey, cidx);

  // ---- rank the nsel candidates (key descending, index ascending) and write them; fillers past nsel ----
  if (tid < keep) {
    float* out_s = p.cand_scores + (int64_t)row * keep;
    int32_t* out_i = p.cand_index + (int64_t)row * keep;
    if (tid < nsel) {
      const int idx = cidx[tid];
      const int rank = top_rank(ckey, cidx, nsel, tid);
      out_s[rank] = xs[idx];
      out_i[rank] = k * V + idx;
    } else {
      out_s[tid] = -INFINITY;
      out_i[tid] = -1;
    }
  }
}

// fp32(g ** lp): the fp64 power of the fp64 penalty, rounded once, as torch divides an fp32 tensor by a Python float
__device__ __forceinline__ float length_divisor(int g, double lp) {
  return __double2float_rn(pow((double)g, lp));
}

// the position of the largest of v[0 .. n) not yet taken (lowest position on ties); marks it taken
__device__ __forceinline__ int take_top(const float* v, int n, bool* taken) {
  int best = -1;
  uint32_t bk = 0;
  for (int c = 0; c < n; ++c) {
    if (taken[c]) continue;
    const uint32_t key = order_key(v[c]);
    if (best < 0 || key > bk) best = c, bk = key;
  }
  taken[best] = true;
  return best;
}

__global__ void __launch_bounds__(kThreads) beam_item_kernel(const pcv_beam_step_params p) {
  __shared__ uint32_t key_s[kMaxCand];
  __shared__ int32_t idx_s[kMaxCand];
  __shared__ float score_s[kMaxCand];
  __shared__ float top_s[kMaxKeep];   // the item's top beams_to_keep, ranked
  __shared__ int32_t top_i[kMaxKeep];
  __shared__ float merged[PCV_BEAM_MAX_BEAMS + kMaxKeep];
  __shared__ bool taken[PCV_BEAM_MAX_BEAMS + kMaxKeep];
  __shared__ int32_t run_par[PCV_BEAM_MAX_BEAMS], run_tok[PCV_BEAM_MAX_BEAMS];
  __shared__ int32_t fin_src[PCV_BEAM_MAX_BEAMS];   // < K: old finished slot; else K + candidate position
  __shared__ int32_t gen_s;
  __shared__ float div_s[2];   // the length-penalty divisors of the finished scores and of the heuristic
  const int tid = threadIdx.x, b = blockIdx.x;
  const int K = p.K, V = p.V, keep = keep_count(p), nc = K * keep, H = p.hist_len;

  if (tid == kThreads - 1) {   // a thread of the last warp, idle while the candidates load (nc <= 320)
    const int n = p.counters[1], g = p.counters[0] + 1;
    div_s[0] = length_divisor(g, p.length_penalty);
    div_s[1] = length_divisor(p.early_stopping == PCV_EARLY_STOP_NEVER && p.length_penalty > 0.0 ? n : g,
                              p.length_penalty);
  }

  for (int c = tid; c < nc; c += kThreads) {
    const float sc = p.cand_scores[(int64_t)b * nc + c];
    const int32_t ix = p.cand_index[(int64_t)b * nc + c];
    score_s[c] = sc;
    key_s[c] = ix < 0 ? 0u : order_key(sc);                 // fillers rank below every candidate
    idx_s[c] = ix < 0 ? 0x7fffffff - c : ix;
  }
  __syncthreads();
  for (int c = tid; c < nc; c += kThreads) {
    const uint32_t key = key_s[c];
    const int32_t ix = idx_s[c];
    int rank = 0;
    for (int j = 0; j < nc; ++j) rank += (key_s[j] > key || (key_s[j] == key && idx_s[j] < ix)) ? 1 : 0;
    if (rank < keep) top_s[rank] = score_s[c], top_i[rank] = ix;
  }
  __syncthreads();

  if (tid == 0) {
    const int gen = p.counters[0], n = p.counters[1], g = gen + 1, es = p.early_stopping;
    float* fin = p.finished_scores + b * K;
    int32_t* fflag = p.finished_flags + b * K;
    float* runs = p.running_scores + b * K;
    int32_t* item = p.item_flags + 2 * b;
    bool hit[kMaxKeep];
    float trun[kMaxKeep];
    for (int c = 0; c < keep; ++c) {
      const int tok = top_i[c] % V;
      bool h = g >= n;
      for (int e = 0; e < p.n_eos; ++e) h = h || tok == p.eos[e];
      hit[c] = h;
      trun[c] = h ? __fadd_rn(top_s[c], kNeg) : top_s[c];
    }
    // finished set, with the state before this step
    bool full = es == PCV_EARLY_STOP_TRUE;
    for (int j = 0; j < K; ++j) full = full && fflag[j] != 0;
    const bool unsat = item[0] != 0;
    const float div = div_s[0];
    for (int j = 0; j < K; ++j) merged[j] = fin[j], taken[j] = false;
    for (int c = 0; c < keep; ++c) {
      float s = __fdiv_rn(top_s[c], div);
      if (full) s = __fadd_rn(s, kNeg);
      if (!unsat) s = __fadd_rn(s, kNeg);
      if (!(hit[c] && c < K)) s = __fadd_rn(s, kNeg);
      merged[K + c] = s;
      taken[K + c] = false;
    }
    float nfin[PCV_BEAM_MAX_BEAMS];
    int32_t nflag[PCV_BEAM_MAX_BEAMS];
    for (int j = 0; j < K; ++j) {
      const int src = take_top(merged, K + keep, taken);
      fin_src[j] = src;
      nfin[j] = merged[src];
      // a candidate's flag is its eligibility: an ineligible one taken into an unfilled slot stays unfinished
      nflag[j] = src < K ? fflag[src] : (src - K < K && hit[src - K]) ? 1 : 0;
    }
    for (int j = 0; j < K; ++j) {
      fin[j] = nfin[j];
      fflag[j] = nflag[j];
    }
    // running beams
    for (int c = 0; c < keep; ++c) taken[c] = false;
    for (int j = 0; j < K; ++j) {
      const int c = take_top(trun, keep, taken);
      runs[j] = trun[c];
      run_par[j] = top_i[c] / V;
      run_tok[j] = top_i[c] % V;
      p.next_tokens[b * K + j] = run_tok[j];
      p.parents[b * K + j] = b * K + run_par[j];
    }
    // the early-stop heuristic after this step, and the item's done flag
    const float best = __fdiv_rn(runs[0], div_s[1]);
    float worst = nfin[0];
    bool all_fin = true;
    for (int j = 0; j < K; ++j) worst = fminf(worst, nfin[j]), all_fin = all_fin && nflag[j] != 0;
    bool improve = false;
    for (int j = 0; j < K; ++j) improve = improve || best > (nflag[j] ? worst : kNeg);
    const bool unsat_new = unsat && improve;
    item[0] = unsat_new ? 1 : 0;
    item[1] = (!unsat_new || (es == PCV_EARLY_STOP_TRUE && all_fin)) ? 1 : 0;
    gen_s = gen;
  }
  __syncthreads();

  // ---- histories: copy the old rows' columns [0, gen) to scratch, then gather them by source ----
  const int gen = gen_s;
  const int cols = gen < 0 ? 0 : gen < H ? gen : H;
  int64_t* run_h = p.running_hist + (int64_t)b * K * H;
  int64_t* fin_h = p.finished_hist + (int64_t)b * K * H;
  int64_t* scr = p.hist_scratch + (int64_t)b * 2 * K * H;   // [K running rows | K finished rows]
  for (int e = tid; e < 2 * K * cols; e += kThreads) {
    const int r = e / cols, c = e % cols;
    scr[(int64_t)r * H + c] = r < K ? run_h[(int64_t)r * H + c] : fin_h[(int64_t)(r - K) * H + c];
  }
  __syncthreads();
  for (int e = tid; e < 2 * K * cols; e += kThreads) {
    const int r = e / cols, c = e % cols;
    if (r < K) {
      run_h[(int64_t)r * H + c] = scr[(int64_t)run_par[r] * H + c];
    } else {
      const int src = fin_src[r - K];
      const int from = src < K ? K + src : top_i[src - K] / V;   // an old finished row, or a candidate's parent
      fin_h[(int64_t)(r - K) * H + c] = scr[(int64_t)from * H + c];
    }
  }
  if (gen >= 0 && gen < H && tid < 2 * K) {
    if (tid < K) {
      run_h[(int64_t)tid * H + gen] = run_tok[tid];
    } else {
      const int src = fin_src[tid - K];
      if (src >= K) fin_h[(int64_t)(tid - K) * H + gen] = top_i[src - K] % V;
    }
  }

  // ---- the last CTA: every item done, and the generated count ----
  if (tid == 0) {
    __threadfence();
    const int arrived = atomicAdd(p.counters + 3, 1);
    if (arrived == p.B - 1) {
      __threadfence();
      int all = 1;
      for (int i = 0; i < p.B; ++i) all &= ((volatile int32_t*)p.item_flags)[2 * i + 1];
      p.counters[2] = all;
      p.counters[0] = gen + 1;
      p.counters[3] = 0;
    }
  }
}

// ---- KV gather of the generated rows ----------------------------------------------------------------------------------
// CTA (entry e, beam row i): phase 0 copies the parent's rows [first, cur) of arena e into row i's scratch, phase 1
// copies them from the scratch into row i; first = first_row, or max(first_row, cur - last_rows) when last_rows > 0.
// Rows whose parent is themselves copy nothing.
__global__ void __launch_bounds__(256) kv_gather_kernel(const pcv_kv_gather_params p, const pcv_dev_rows rows,
                                                        int phase) {
  const pcv_kv_gather_entry e = p.table[blockIdx.x];
  const int i = blockIdx.y, par = p.parents[i];
  if (par == i || par < 0 || par >= p.R) return;
  const int cur = rows.bounds[(int64_t)i * rows.bounds_stride_b + e.bounds_col];
  const int last = min(cur, e.first_row + e.max_rows);
  const int first = p.last_rows > 0 ? max(e.first_row, cur - p.last_rows) : e.first_row;
  if (last <= first) return;
  const int64_t n16 = (int64_t)(last - first) * e.row_bytes / 16;
  const int64_t row0 = (int64_t)first * e.row_bytes;
  const uint4* src;
  uint4* dst;
  if (phase == 0) {
    src = reinterpret_cast<const uint4*>(static_cast<const char*>(e.arena) + par * e.arena_stride_b + row0);
    dst = reinterpret_cast<uint4*>(static_cast<char*>(e.scratch) + i * e.scratch_stride_b);
  } else {
    src = reinterpret_cast<const uint4*>(static_cast<const char*>(e.scratch) + i * e.scratch_stride_b);
    dst = reinterpret_cast<uint4*>(static_cast<char*>(e.arena) + i * e.arena_stride_b + row0);
  }
  for (int64_t j = threadIdx.x; j < n16; j += blockDim.x) dst[j] = src[j];
}

bool disjoint(const void* a, size_t na, const void* b, size_t nb) {
  const char *x = static_cast<const char*>(a), *y = static_cast<const char*>(b);
  return x + na <= y || y + nb <= x;
}

}  // namespace

int beam_step_check(const pcv_beam_step_params* p, bool logprobs) {
  PCV_REQUIRE(p != nullptr, PCV_ERR_INVALID, "beam_step: params is NULL");
  PCV_REQUIRE(!logprobs || p->dtype == PCV_F32, PCV_ERR_INVALID,
              "beam_step_logprobs: dtype %d must be fp32 (%d): the rows are processed log-probabilities", p->dtype,
              PCV_F32);
  PCV_REQUIRE(p->logits && p->running_scores && p->finished_scores && p->finished_flags && p->running_hist &&
                  p->finished_hist && p->hist_scratch && p->item_flags && p->counters && p->cand_scores &&
                  p->cand_index && p->next_tokens && p->parents,
              PCV_ERR_INVALID, "beam_step: a pointer is NULL");
  PCV_REQUIRE(p->dtype == PCV_BF16 || p->dtype == PCV_F16 || p->dtype == PCV_F32, PCV_ERR_INVALID,
              "beam_step: unknown dtype %d (bf16, fp16 or fp32 logits)", p->dtype);
  PCV_REQUIRE(p->V >= 1 && p->V <= PCV_SAMPLE_MAX_VOCAB, PCV_ERR_UNSUPPORTED, "beam_step: V=%d must be in [1, %d]",
              p->V, PCV_SAMPLE_MAX_VOCAB);
  PCV_REQUIRE(p->K >= 1 && p->K <= PCV_BEAM_MAX_BEAMS, PCV_ERR_UNSUPPORTED, "beam_step: K=%d must be in [1, %d]",
              p->K, PCV_BEAM_MAX_BEAMS);
  PCV_REQUIRE(p->B >= 1, PCV_ERR_INVALID, "beam_step: B=%d must be >= 1", p->B);
  PCV_REQUIRE(p->n_eos >= 0 && p->n_eos <= PCV_BEAM_MAX_EOS, PCV_ERR_UNSUPPORTED,
              "beam_step: n_eos=%d must be in [0, %d]", p->n_eos, PCV_BEAM_MAX_EOS);
  const int keep = (p->n_eos + 1 > 2 ? p->n_eos + 1 : 2) * p->K;
  PCV_REQUIRE((int64_t)p->K * p->V >= keep, PCV_ERR_UNSUPPORTED,
              "beam_step: K*V=%lld is below beams_to_keep=%d", (long long)p->K * p->V, keep);
  for (int e = 0; e < p->n_eos; ++e)
    PCV_REQUIRE(p->eos[e] >= 0 && p->eos[e] < p->V, PCV_ERR_INVALID, "beam_step: EOS id %d is outside [0, V=%d)",
                p->eos[e], p->V);
  PCV_REQUIRE(p->stride_row >= p->V, PCV_ERR_INVALID, "beam_step: stride_row=%lld is below V=%d",
              (long long)p->stride_row, p->V);
  PCV_REQUIRE(isfinite(p->length_penalty), PCV_ERR_INVALID, "beam_step: length_penalty must be finite, got %g",
              p->length_penalty);
  PCV_REQUIRE(p->early_stopping >= PCV_EARLY_STOP_FALSE && p->early_stopping <= PCV_EARLY_STOP_NEVER,
              PCV_ERR_INVALID, "beam_step: unknown early_stopping code %d (0: False, 1: True, 2: never)",
              p->early_stopping);
  PCV_REQUIRE(p->hist_len >= 1, PCV_ERR_INVALID, "beam_step: hist_len=%d must be >= 1", p->hist_len);
  const size_t BK = (size_t)p->B * p->K, H = (size_t)p->hist_len;
  const struct {
    const void* ptr;
    size_t bytes;
  } out[] = {{p->running_scores, BK * 4},     {p->finished_scores, BK * 4}, {p->finished_flags, BK * 4},
             {p->running_hist, BK * H * 8},   {p->finished_hist, BK * H * 8}, {p->hist_scratch, 2 * BK * H * 8},
             {p->item_flags, (size_t)p->B * 8}, {p->counters, 16},          {p->cand_scores, BK * keep * 4},
             {p->cand_index, BK * keep * 4},  {p->next_tokens, BK * 8},    {p->parents, BK * 4}};
  const int n = (int)(sizeof(out) / sizeof(out[0]));
  for (int i = 0; i < n; ++i)
    for (int j = i + 1; j < n; ++j)
      PCV_REQUIRE(disjoint(out[i].ptr, out[i].bytes, out[j].ptr, out[j].bytes), PCV_ERR_INVALID,
                  "beam_step: output buffers %d and %d overlap", i, j);
  return PCV_OK;
}

int launch_beam_step(const pcv_beam_step_params& p, bool logprobs, cudaStream_t stream) {
  void (*const kern[3])(BeamRows) = {beam_rows_kernel<__nv_bfloat16>, beam_rows_kernel<__half>,
                                     beam_rows_kernel<float>};
  const int rc = launch_row_kernel(kern, p.dtype, p.V, p.B * p.K, BeamRows{p, logprobs ? 1 : 0}, stream);
  if (rc != PCV_OK) return rc;
  beam_item_kernel<<<p.B, kThreads, 0, stream>>>(p);
  PCV_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PCV_OK;
}

int kv_gather_check(const pcv_kv_gather_params* p, const pcv_dev_rows* rows) {
  PCV_REQUIRE(p != nullptr && rows != nullptr, PCV_ERR_INVALID, "kv_gather_rows: params or rows is NULL");
  PCV_REQUIRE(p->table && p->parents && rows->bounds, PCV_ERR_INVALID,
              "kv_gather_rows: table / parents / bounds pointer is NULL");
  PCV_REQUIRE(p->n_entries >= 1 && p->n_entries <= 65535, PCV_ERR_INVALID,
              "kv_gather_rows: n_entries=%d must be in [1, 65535]", p->n_entries);
  PCV_REQUIRE(p->R >= 1 && p->R <= 65535, PCV_ERR_INVALID, "kv_gather_rows: R=%d must be in [1, 65535]", p->R);
  PCV_REQUIRE(rows->bounds_stride_b >= 0, PCV_ERR_INVALID, "kv_gather_rows: bounds_stride_b=%d is negative",
              rows->bounds_stride_b);
  PCV_REQUIRE(p->last_rows >= 0, PCV_ERR_INVALID, "kv_gather_rows: last_rows=%d is negative", p->last_rows);
  return PCV_OK;
}

int launch_kv_gather(const pcv_kv_gather_params& p, const pcv_dev_rows& rows, cudaStream_t stream) {
  const dim3 grid(p.n_entries, p.R);
  for (int phase = 0; phase < 2; ++phase) {
    kv_gather_kernel<<<grid, 256, 0, stream>>>(p, rows, phase);
    PCV_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  return PCV_OK;
}

}  // namespace pcv
