/*
 * pcv_attn.h — C ABI of libpcv_attn.so: the H100 (sm_90a) latent-attention hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8(b), level 2).  Every entry point takes plain
 * pointers and sizes; no torch types cross it.  The Python host side
 * (perceiver_io_b200/ops.py) binds these symbols with ctypes and passes
 * `tensor.data_ptr()` and the raw `cudaStream_t` of torch's current stream.
 *
 * What each entry point replaces in the reference (paths relative to /root/reference):
 *
 *   pcv_attn_fwd            perceiver/model/core/modules.py:146-164  (the head-chunk loop:
 *                           einsum QK^T -> masked_fill_(pad) -> masked_fill_(causal) ->
 *                           softmax -> einsum PV) plus the head split/merge rearranges at
 *                           :123 and :166-167 (done by strides, never materialised) and the
 *                           q*dp_scale at :124 (folded into the softmax exponent).
 *   pcv_attn_combine        no counterpart: merges per-shard partial softmax states
 *                           (numerator, row max, denominator) when M is split inside one GPU
 *                           or across GPUs (SURVEY.md §8(e)).
 *   pcv_rotary_apply        perceiver/model/core/position.py:30-50
 *                           (RotaryPositionEmbedding.rotate + _rotate_half).
 *   pcv_kv_append           perceiver/model/core/modules.py:117-121 (torch.cat onto the cache).
 *
 * Conventions
 *   - All device pointers must belong to the current CUDA device of the calling thread.
 *   - All work is enqueued on `stream` (a cudaStream_t passed as void*); nothing synchronises.
 *   - Return value 0 = success; non-zero = failure, message via pcv_last_error() (thread local).
 *   - Strides are in ELEMENTS of the tensor's dtype.
 *   - Inputs are borrowed and never written; outputs are caller-allocated.
 */
#ifndef PCV_ATTN_H_
#define PCV_ATTN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCV_ABI_VERSION 2

#if defined(__GNUC__)
#define PCV_API __attribute__((visibility("default")))
#else
#define PCV_API
#endif

/* element type of q/k/v/out */
enum pcv_dtype { PCV_BF16 = 0, PCV_F16 = 1, PCV_F32 = 2 /* pcv_kv_append only */, PCV_E4M3 = 3 /* the *_fp8 entry points only */ };

/* kernel selection; AUTO picks the tensor-core kernel whenever the shape is supported (the names are historical) */
enum pcv_impl {
  PCV_IMPL_AUTO = 0,         /* decode kernel for N <= 4 and M >= 1024, single-CTA tensor-core kernel when the shape fits, else SIMT */
  PCV_IMPL_TCGEN05 = 1,      /* single-CTA tensor-core (sm_90a wgmma) kernel or error */
  PCV_IMPL_SIMT = 2,         /* CUDA-core coverage kernel */
  PCV_IMPL_TCGEN05_PAIR = 3, /* CTA-pair kernel: 2-CTA cluster sharing K/V tiles by multicast (qk and v head dims <= 128; 256 query rows per unit) or error */
  PCV_IMPL_DECODE = 4        /* streaming kernel for N <= 4 query rows against a long cache (HBM-bound) or error */
};

/* status codes */
enum pcv_status {
  PCV_OK = 0,
  PCV_ERR_INVALID = 1,      /* bad argument (message says which)              */
  PCV_ERR_UNSUPPORTED = 2,  /* shape/dtype not supported by the requested impl */
  PCV_ERR_CUDA = 3,         /* a CUDA runtime/driver call failed               */
  PCV_ERR_WORKSPACE = 4     /* workspace missing or too small                  */
};

/*
 * Fused attention forward for one MultiHeadAttention call.
 *
 *   q   : (Bq, N, H, dqk)  Bq is B or 1 (q_stride_b == 0 broadcasts the latents, the
 *                           encoder case: adapter.py:82-83 returns a batch-1 latent array)
 *   k   : (B,  M, H, dqk)
 *   v   : (B,  M, H, dv)
 *   out : (B,  N, H, dv)   normalised attention output, same dtype as q
 *
 * Score of query i / key j (before softmax), with jg = m_offset + j the key's global index:
 *     s_ij = scale * <q_i, k_j>
 *     masked (set to -FLT_MAX, the reference's finite fill, modules.py:152-158) when
 *         pad_mask[b, j] != 0, or
 *         causal != 0 and jg > i + (m_total - N)      (right-aligned causal, modules.py:135-140)
 *   A fully masked row therefore becomes the uniform average of all M value rows, exactly as
 *   in the reference.
 *
 * M-sharding: a shard passes its local M keys, the global key count m_total and its first
 * key's global index m_offset; with write_partial != 0 the kernel emits the un-normalised
 * state instead of `out`:
 *     part_o (B,H,N,dv) f32 = sum_j exp2(t_ij - m_i) v_j,   part_m (B,H,N) f32 = m_i (log2 domain,
 *     t = s*log2(e)),   part_l (B,H,N) f32 = sum_j exp2(t_ij - m_i)
 * which pcv_attn_combine merges exactly.
 */
typedef struct pcv_attn_params {
  const void* q;
  const void* k;
  const void* v;
  void* out;
  int64_t q_stride_b, q_stride_n, q_stride_h;
  int64_t k_stride_b, k_stride_m, k_stride_h;
  int64_t v_stride_b, v_stride_m, v_stride_h;
  int64_t o_stride_b, o_stride_n, o_stride_h;
  int32_t B, H, N, M;
  int32_t dqk, dv;
  float scale;             /* dp_scale = dqk^-0.5 (modules.py:73)                       */
  int32_t dtype;           /* enum pcv_dtype                                            */
  int32_t causal;          /* 0 / 1                                                     */
  int32_t m_total;         /* global number of keys (== M when not sharded)             */
  int32_t m_offset;        /* global index of this call's key 0                         */
  const uint8_t* pad_mask; /* (B, M) bytes, non-zero = padding key; NULL = none         */
  int64_t pad_stride_b;    /* bytes between batch rows of pad_mask                      */
  int32_t write_partial;   /* 0: write `out`; 1: write part_o/part_m/part_l             */
  float* part_o;
  float* part_m;
  float* part_l;
  void* workspace;         /* device scratch of at least pcv_attn_workspace_bytes()     */
  size_t workspace_bytes;
  int32_t impl;            /* enum pcv_impl                                             */
  int32_t reserved;
} pcv_attn_params;

/*
 * Merge `num_parts` partial softmax states of identical shape into the final output.
 *   part_o : (num_parts, B, H, N, dv) f32   part_m, part_l : (num_parts, B, H, N) f32
 *   out    : (B, N, H, dv) in `dtype`, strides as in pcv_attn_params
 *   m = max_g m_g ;  l = sum_g l_g 2^(m_g-m) ;  out = sum_g part_o_g 2^(m_g-m) / l
 */
typedef struct pcv_combine_params {
  const float* part_o;
  const float* part_m;
  const float* part_l;
  void* out;
  int64_t o_stride_b, o_stride_n, o_stride_h;
  int32_t num_parts;
  int32_t B, H, N, dv;
  int32_t dtype;
} pcv_combine_params;

/*
 * Rotary position embedding of a (B, n, H, d) tensor (position.py:30-50).
 *   angles : (Ba, n_angles, rotate_dim) f32, Ba is B or 1 — the `frq_pos_enc` tensor the
 *            reference's RotaryPositionEmbedding holds (position.py:23-28)
 *   row i of x uses angle row `angle_row0 + i`  (right_align: n_angles - n, else 0)
 *   channels [0, rotate_dim) of every head are rotated pairwise, the rest pass through:
 *     y[2p]   = x[2p]  *cos(a[2p])   - x[2p+1]*sin(a[2p])
 *     y[2p+1] = x[2p+1]*cos(a[2p+1]) + x[2p]  *sin(a[2p+1])
 *   y is written with its own strides (may alias neither x nor angles).
 */
typedef struct pcv_rotary_params {
  const void* x;
  void* y;
  const float* angles;
  int64_t x_stride_b, x_stride_n, x_stride_h;
  int64_t y_stride_b, y_stride_n, y_stride_h;
  int64_t a_stride_b, a_stride_n; /* a_stride_b == 0 broadcasts */
  int32_t B, n, H, d;
  int32_t rotate_dim;
  int32_t angle_row0;
  int32_t dtype;
  int32_t reserved;
} pcv_rotary_params;

/*
 * KV-cache append (modules.py:117-121): dst[:, :L_old] = cache, dst[:, L_old:L_old+n] = fresh
 * for both K and V in one launch.  Tensors are (B, L, C) with explicit batch/row strides.
 * A cache pointer may equal its dst pointer (in-place arena append): that half is skipped.
 */
typedef struct pcv_kv_append_params {
  const void* k_cache; const void* v_cache;   /* (B, L_old, Ck) / (B, L_old, Cv); may be NULL if L_old == 0 */
  const void* k_new;   const void* v_new;     /* (B, n, Ck) / (B, n, Cv) */
  void* k_dst;         void* v_dst;           /* (B, L_old + n, Ck) / (.., Cv) */
  int64_t kc_stride_b, kc_stride_l, vc_stride_b, vc_stride_l;
  int64_t kn_stride_b, kn_stride_l, vn_stride_b, vn_stride_l;
  int64_t kd_stride_b, kd_stride_l, vd_stride_b, vd_stride_l;
  int32_t B, L_old, n, Ck, Cv;
  int32_t dtype;
} pcv_kv_append_params;

/*
 * Merge `num_parts` partial states into ONE partial state (still un-normalised): the local step of a two-level
 * merge (chunks of a host-streamed shard on one GPU, then pcv_attn_combine_peers / an all-reduce across GPUs).
 *   part_* : (num_parts, rows[, dv]) f32, rows = B*H*N;   out_* : (rows[, dv]) f32
 *   out_m = max_g m_g ;  out_l = sum_g l_g 2^(m_g - out_m) ;  out_o = sum_g part_o_g 2^(m_g - out_m)
 */
typedef struct pcv_merge_params {
  const float* part_o;
  const float* part_m;
  const float* part_l;
  float* out_o;
  float* out_m;
  float* out_l;
  int64_t rows;
  int32_t num_parts, dv;
} pcv_merge_params;

/*
 * In-place change of reference maximum of a partial state (used between the two all-reduces of the
 * M-sharded path, perceiver_io_b200/dist.py):  w = 2^(part_m[r] - new_m[r]);  part_o[r,:] *= w;
 * part_l[r] *= w;  part_m[r] = new_m[r].   rows = B*H*N.  new_m[r] >= part_m[r] is expected.
 * part_o rows are read and written as float4 when dv % 4 == 0 and part_o is 16-byte aligned, element-wise otherwise.
 */
typedef struct pcv_rescale_params {
  float* part_o;        /* (rows, dv) */
  float* part_m;        /* (rows)     */
  float* part_l;        /* (rows)     */
  const float* new_m;   /* (rows)     */
  int64_t rows;
  int32_t dv;
  int32_t reserved;
} pcv_rescale_params;

/*
 * Merge of M-shard partial states held in PEER-ACCESSIBLE memory (NVLink / NVSwitch), no NCCL on the data
 * path: rank `rank` owns rows [row_begin, row_end) of the flattened (B*H*N) row space; for each owned row it
 * loads (part_o, part_m, part_l) of that row from all `num_peers` ranks through their mapped pointers, merges
 * them exactly as pcv_attn_combine does, and stores the normalised row into the output buffer of EVERY rank
 * (so all ranks end up with the full (B, N, H, dv) result after a barrier).  The caller provides the barriers
 * (before: all partial states written; after: all outputs written) — perceiver_io_b200/dist.py uses the
 * symmetric-memory signal pads for that.
 * Fast path (every lane issues all its loads of a row before it consumes one): taken when dv % 4 == 0, dv <= 128,
 * the three output strides are multiples of 4 elements, every part_o[g] is 16-byte aligned and every out[g] 8-byte
 * aligned.  Any other call runs the general path (element-wise loads and stores), with the same result.
 */
#define PCV_MAX_PEERS 8
typedef struct pcv_peer_combine_params {
  const float* part_o[PCV_MAX_PEERS]; /* per rank: (B, H, N, dv) f32 */
  const float* part_m[PCV_MAX_PEERS]; /* per rank: (B, H, N) f32     */
  const float* part_l[PCV_MAX_PEERS]; /* per rank: (B, H, N) f32     */
  void* out[PCV_MAX_PEERS];           /* per rank: (B, N, H, dv) in `dtype`, strides below */
  int64_t o_stride_b, o_stride_n, o_stride_h;
  int64_t row_begin, row_end;
  int32_t num_peers, rank;
  int32_t B, H, N, dv;
  int32_t dtype;
  int32_t reserved;
} pcv_peer_combine_params;

/*
 * Fused K/V producer of the cross-attention module (SURVEY.md §8(f)1): replaces, for inference,
 *   perceiver/model/core/modules.py:226      x_kv = self.kv_norm(x_kv)
 *   perceiver/model/core/modules.py:114-115  k = self.k_proj(x_kv); v = self.v_proj(x_kv)
 * with ONE pass over the raw input on the tcgen05 tensor cores.  LayerNorm is folded around the GEMM:
 *     LN(x) W^T + b  =  rstd * ( x (gamma.W)^T - mean * s ) + t
 * The caller prepares, once per set of weights,
 *     w      : (n_k + n_v, C)  = [gamma.Wk ; gamma.Wv] rounded to `dtype`, row-major (the nn.Linear layout)
 *     col_st : (n_k + n_v, 2) f32, per output column (s, t):  s = sum_c w[n, c] (of the ROUNDED w),
 *              t = sum_c beta_c W[n, c] + bias[n]
 * The row statistics (mean, 1/sqrt(var + eps)) come either from pcv_ln_stats (row_stats (rows, 2) f32: two-pass, one
 * extra read of x) or — row_stats == NULL and ln_eps > 0 — from the GEMM kernel itself, which computes them in one
 * pass (shifted by the row's first element) from the input tiles it stages anyway.
 * row_stats == NULL and ln_eps == 0 means "no LayerNorm": out = x w^T + t (a plain projection with bias).
 * A zero-variance row has x_hat == 0, so its output is t exactly (the fold would otherwise scale the fp32 residue of
 * x.w - mean * s by eps^-1/2).  The in-kernel statistics detect such rows exactly.  With row_stats, pass their eps as
 * ln_eps: a row whose rstd equals 1 / sqrtf(ln_eps), the value pcv_ln_stats writes when var + eps rounds to eps in
 * fp32 (var < ~2^-24 eps, |x_hat| < 2^-12 in RMS), is written as t.
 *   x      : (rows, C) with an element row stride (rows = B*M flattened)
 *   k_out  : (rows, n_k), v_out : (rows, n_v), each with its own row stride — the un-rotated, pre-head-split
 *            K / V rows the reference would have produced (and caches, modules.py:117-121)
 * Constraints (else PCV_ERR_UNSUPPORTED; the host side then uses the library GEMM): C, n_v and the strides multiples
 * of 8 elements, n_k a multiple of 64, 16-byte aligned pointers.
 */
typedef struct pcv_kvproj_params {
  const void* x;
  const void* w;
  const float* col_st;
  const float* row_stats;
  void* k_out;
  void* v_out;
  int64_t x_stride_row, k_stride_row, v_stride_row;
  int64_t rows;
  int32_t C, n_k, n_v;
  int32_t dtype;       /* PCV_BF16 / PCV_F16 */
  int32_t cta_group;   /* 0 = library default (1), 1 = one CTA per tile, 2 = CTA pairs (2-CTA cluster sharing the weight tile) */
  float ln_eps;        /* row_stats == NULL: > 0 = LayerNorm with statistics computed INSIDE the GEMM kernel from the
                          staged input tiles (no separate pass over x), 0 = no LayerNorm.  With row_stats: the eps
                          they were computed with (0 = unknown: zero-variance rows are not detected) */
} pcv_kvproj_params;

/* LayerNorm row statistics (nn.LayerNorm semantics: biased variance): stats[r] = (mean, 1/sqrt(var + eps)) */
typedef struct pcv_ln_stats_params {
  const void* x;       /* (rows, C) */
  float* stats;        /* (rows, 2) f32 */
  int64_t x_stride_row;
  int64_t rows;
  int32_t C;
  float eps;
  int32_t dtype;
  int32_t reserved;
} pcv_ln_stats_params;

/*
 * M-sharded attention with the cross-GPU merge FUSED INTO THE KERNEL TAIL (SURVEY.md §8(e) option 3): one launch per
 * rank computes the partial softmax state of this rank's key shard, publishes it to its peers through NVLink-mapped
 * symmetric memory, merges the rows it owns from all ranks and pushes the normalised rows into every rank's output
 * buffer.  No NCCL and no host-launched barrier is on the path; the kernel returns when this rank's output buffer is
 * complete.  All ranks must call with the same shapes and the same `epoch` (1, 2, 3, ... per call on one set of
 * buffers); `p` is a pcv_attn_params with write_partial = 1 (part_* are ignored: the state lives in part[rank]).
 *   part[g]  : rank g's buffer, f32 [ numerator (B,H,N,dv) | row max (B,H,N) | denominator (B,H,N) ]
 *   out[g]   : rank g's output (B,N,H,dv) in p->dtype with the strides below; every rank ends with the full result
 *   flags[g] : rank g's flag block, >= 32 zero-initialised uint32 words (never reset: values are epochs)
 * Rank r merges rows [R*r/G, R*(r+1)/G) of the flattened (b,h,n) space, R = B*H*N.
 * The merge loads 16 bytes of part rows and stores 4 channels (8 bytes) of output rows at once, so every part[g] must
 * be 16-byte aligned, every out[g] 8-byte aligned, o_stride_b / o_stride_n / o_stride_h multiples of 4 elements and
 * every flags[g] 4-byte aligned; other calls are refused with PCV_ERR_INVALID before any CUDA call.
 */
typedef struct pcv_shard_fuse {
  void* part[PCV_MAX_PEERS];
  void* out[PCV_MAX_PEERS];
  uint32_t* flags[PCV_MAX_PEERS];
  int64_t o_stride_b, o_stride_n, o_stride_h;
  int32_t num_peers, rank;
  uint32_t epoch;
  int32_t reserved;
} pcv_shard_fuse;

/*
 * Backward of the attention core (autograd through modules.py:141-167): from the forward's operands, its output and
 * its saved row statistics (part_m / part_l of a write_partial forward over ALL keys, log2 domain) compute
 *   grad_q = scale * dS K,  grad_k = scale * dS^T Q,  grad_v = P^T grad_out,   dS = P * (grad_out V^T - rowsum(grad_out*out))
 * with the masks of the forward (finite fill: a filled score carries no gradient).  Tensors are laid out as in
 * pcv_attn_params ((B, rows, H, d) by strides, in `dtype`); q_stride_b == 0 broadcasts one latent array over the batch and
 * grad_q is then the SUM over the batch, shape (1, N, H*dqk).  Two tcgen05 kernels (dK/dV: key-tile outer; dQ: query-tile
 * outer) — no (B, H, N, M) tensor is ever materialised.  Head dims: multiples of 8, at most 192.  Above 128 grad_q is
 * summed from per-(batch contribution, key split) fp32 partials in a fixed order (bitwise reproducible); the workspace
 * then holds those partials.
 */
typedef struct pcv_attn_bwd_params {
  const void* q;
  const void* k;
  const void* v;
  const void* out;        /* forward output (B, N, H, dv)                               */
  const void* grad_out;   /* gradient of the loss w.r.t. out, same shape                */
  const float* stat_m;    /* (B, H, N) row maxima of the forward (log2 domain)          */
  const float* stat_l;    /* (B, H, N) softmax denominators relative to stat_m          */
  void* grad_q;           /* (B or 1, N, H, dqk)                                        */
  void* grad_k;           /* (B, M, H, dqk)                                             */
  void* grad_v;           /* (B, M, H, dv)                                              */
  int64_t q_stride_b, q_stride_n, q_stride_h;
  int64_t k_stride_b, k_stride_m, k_stride_h;
  int64_t v_stride_b, v_stride_m, v_stride_h;
  int64_t o_stride_b, o_stride_n, o_stride_h;
  int64_t go_stride_b, go_stride_n, go_stride_h;
  int64_t gq_stride_b, gq_stride_n, gq_stride_h;
  int64_t gk_stride_b, gk_stride_m, gk_stride_h;
  int64_t gv_stride_b, gv_stride_m, gv_stride_h;
  int32_t B, H, N, M;
  int32_t dqk, dv;
  float scale;
  int32_t dtype;           /* enum pcv_dtype (bf16 / fp16)                              */
  int32_t causal;          /* right-aligned causal mask as in the forward               */
  float dropout_p;         /* attention-probability dropout of the forward (0 = none)   */
  uint64_t dropout_seed;
  const uint8_t* pad_mask; /* (B, M) bytes, non-zero = padding key; NULL = none         */
  int64_t pad_stride_b;
  void* workspace;         /* >= pcv_attn_bwd_workspace_bytes(), 256-byte aligned       */
  size_t workspace_bytes;
} pcv_attn_bwd_params;

/* library / device introspection */
typedef struct pcv_device_info {
  int32_t device;
  int32_t sm_major, sm_minor;
  int32_t num_sms;
  int32_t smem_optin_bytes;
  int32_t tcgen05_ok;      /* 1 when the tensor-core (sm_90a wgmma) kernels can run on this device */
} pcv_device_info;

PCV_API int pcv_abi_version(void);
PCV_API const char* pcv_last_error(void);
PCV_API int pcv_get_device_info(pcv_device_info* info);

/* 1 if the tcgen05 kernel family covers this problem (shape, dtype, alignment), else 0 */
PCV_API int pcv_attn_supported_tcgen05(const pcv_attn_params* p);
PCV_API int pcv_attn_workspace_bytes(const pcv_attn_params* p, size_t* bytes);
PCV_API int pcv_attn_fwd(const pcv_attn_params* p, void* stream);
PCV_API int pcv_attn_combine(const pcv_combine_params* p, void* stream);
PCV_API int pcv_attn_combine_peers(const pcv_peer_combine_params* p, void* stream);
PCV_API int pcv_attn_merge_partials(const pcv_merge_params* p, void* stream);
/* 1 if pcv_attn_fwd_sharded covers this problem (tcgen05 kernel, head dims <= 128 / 256, dv % 4 == 0) */
PCV_API int pcv_attn_fwd_sharded_supported(const pcv_attn_params* p);
PCV_API int pcv_attn_fwd_sharded(const pcv_attn_params* p, const pcv_shard_fuse* fuse, void* stream);
PCV_API int pcv_partial_rescale(const pcv_rescale_params* p, void* stream);
PCV_API int pcv_rotary_apply(const pcv_rotary_params* p, void* stream);
PCV_API int pcv_kv_append(const pcv_kv_append_params* p, void* stream);
/* 1 if pcv_kv_project covers this problem (alignment, widths, device), else 0 (reason via pcv_last_error) */
PCV_API int pcv_kv_project_supported(const pcv_kvproj_params* p);
PCV_API int pcv_ln_stats(const pcv_ln_stats_params* p, void* stream);
PCV_API int pcv_kv_project(const pcv_kvproj_params* p, void* stream);
/* 1 if the tcgen05 backward kernels cover this problem, else 0 (reason via pcv_last_error) */
PCV_API int pcv_attn_bwd_supported(const pcv_attn_bwd_params* p);
PCV_API int pcv_attn_bwd_workspace_bytes(const pcv_attn_bwd_params* p, size_t* bytes);
PCV_API int pcv_attn_bwd(const pcv_attn_bwd_params* p, void* stream);
/*
 * The keep mask of attention-probability dropout (modules.py:161, nn.Dropout on the softmax output) as (B, H, N, M)
 * bytes, 1 = the element survives (tests / debugging).  Each element (b, h, query, key) is dropped with probability
 * round(256 p)/256 by a pure function of (dropout_seed, b, h, query, key): the mask pcv_attn_fwd_partial_dropout applies
 * and pcv_attn_bwd regenerates from the same seed.
 */
PCV_API int pcv_attn_dropout_mask(uint8_t* keep, int32_t B, int32_t H, int32_t N, int32_t M, float dropout_p,
                                  uint64_t dropout_seed, void* stream);
/*
 * The keys [key_begin, key_end) of the same keep mask: keep is (B, H, N, key_end - key_begin) bytes, 1 = the element
 * survives.  pcv_attn_dropout_mask is the range [0, M).  Arguments are checked before any CUDA call.
 */
PCV_API int pcv_attn_dropout_mask_range(uint8_t* keep, int32_t B, int32_t H, int32_t N, int32_t key_begin,
                                        int32_t key_end, float dropout_p, uint64_t dropout_seed, void* stream);
/*
 * One-pass training forward WITH attention-probability dropout, for every head dim the tensor-core forward takes (up
 * to 512).  A write_partial pcv_attn_fwd over all keys (m_total == M, m_offset == 0; impl AUTO or TCGEN05, not the CTA
 * pair) whose part_o is the numerator with dropout, scaled by 1/(1 - p): every element (b, h, query, key) is dropped
 * with probability round(256 p)/256 by the same pure function of (dropout_seed, b, h, query, key) that
 * pcv_attn_dropout_mask exports and pcv_attn_bwd regenerates.  part_m / part_l are the statistics of the dropout-free
 * softmax, so pcv_attn_combine of the state gives out = dropout(P) V and the backward takes part_m / part_l as its
 * stat_m / stat_l.  p->workspace must hold pcv_attn_workspace_bytes() of the call with impl = PCV_IMPL_TCGEN05 (with
 * AUTO and at most 4 query rows it would size the decode kernel's workspace).  Arguments are checked before any CUDA call.
 */
PCV_API int pcv_attn_fwd_partial_dropout_supported(const pcv_attn_params* p, float dropout_p);
PCV_API int pcv_attn_fwd_partial_dropout(const pcv_attn_params* p, float dropout_p, uint64_t dropout_seed, void* stream);

/*
 * Training through a key-sharded attention (each rank holds keys [m_offset, m_offset + M) of m_total).
 *
 * pcv_attn_fwd_partial_dropout_shard: pcv_attn_fwd_partial_dropout on the keys [p->m_offset, p->m_offset + p->M) of
 * p->m_total.  The causal mask and the dropout mask take global key indices: element (b, h, q, m_offset + j) is
 * dropped exactly as pcv_attn_dropout_mask_range exports it, so the shards of one call drop what the unsharded call
 * drops.  part_m / part_l are the dropout-free statistics of the local keys.  m_offset must be even (the mask hashes
 * key pairs).
 *
 * pcv_attn_bwd_shard: the backward of one key shard.  stat_m / stat_l are the statistics MERGED over all m_total keys
 * (the exact merge of every shard's partial state) and out is the merged output.  grad_k / grad_v receive the local
 * keys' gradients, complete.  grad_q in `p` is ignored (may be NULL): the shard's fp32 contribution to grad_q is
 * written to s->grad_q32, (B or 1, N, H, dqk) dense (for a batch-1 q already summed over the batch); grad_q is the sum
 * of the contributions of all shards.  Up to head dim 128 the contribution is accumulated with atomics, above that
 * summed in a fixed order (bitwise reproducible).  Head dims and alignment as pcv_attn_bwd; s->grad_q32 16-byte
 * aligned.  The workspace (pcv_attn_bwd_shard_workspace_bytes, computed without a device) holds no dQ accumulator up
 * to head dim 128.
 * Every argument is checked before any CUDA call.
 */
typedef struct pcv_key_shard {
  int32_t m_total;   /* keys of the whole problem (all shards)                                   */
  int32_t m_offset;  /* global index of this call's key 0 (even)                                 */
  float* grad_q32;   /* (Bq, N, H, dqk) fp32 dense: this shard's contribution to grad_q, WRITTEN  */
} pcv_key_shard;

PCV_API int pcv_attn_fwd_partial_dropout_shard_supported(const pcv_attn_params* p, float dropout_p);
PCV_API int pcv_attn_fwd_partial_dropout_shard(const pcv_attn_params* p, float dropout_p, uint64_t dropout_seed,
                                               void* stream);
PCV_API int pcv_attn_bwd_shard_supported(const pcv_attn_bwd_params* p, const pcv_key_shard* s);
PCV_API int pcv_attn_bwd_shard_workspace_bytes(const pcv_attn_bwd_params* p, const pcv_key_shard* s, size_t* bytes);
PCV_API int pcv_attn_bwd_shard(const pcv_attn_bwd_params* p, const pcv_key_shard* s, void* stream);

/*
 * FP8 (e4m3) inference forward on the tensor cores: S = Q K^T and O = P V on the e4m3 wgmma, softmax in fp32.
 * `p` is a pcv_attn_params with dtype = PCV_E4M3 whose q / k are e4m3 (strides in elements = bytes) and whose v is
 * V TRANSPOSED, vt (B, H, dv, M_pad) e4m3 with the strides of `f` (keys contiguous, in order; M_pad >= M and a
 * multiple of 16; keys beyond M are never read).  v_stride_* of `p` are ignored.  With the dequantisation factors
 *     q = q8 * q_descale[h],   k = k8 * k_descale[h],   v = vt8[b, h, c, :] * v_descale[h, c]
 * the result is that of pcv_attn_fwd on (q, k, v) except that each probability (relative to the running row maximum
 * of its 128-key tile) is rounded to e4m3 as e4m3(P * 256) before P V; the denominators are the fp32 sums of the
 * unrounded probabilities.  Masks, batch-1 q, key sharding (m_total / m_offset) and write_partial behave as in
 * pcv_attn_fwd; out is written in f->out_dtype (bf16 / fp16), and part_* are the same fp32 state, so pcv_attn_combine
 * merges it.  Head dims: multiples of 16, dqk <= 256, dv <= 512.  impl must be AUTO or TCGEN05: the CTA pair, the
 * fused cross-GPU merge, dropout and the decode kernel take no FP8 operands.  The workspace is
 * pcv_attn_workspace_bytes() of the same params.  Arguments are checked before any CUDA call.
 */
typedef struct pcv_fp8_attn {
  const float* q_descale;  /* (H) f32                                                  */
  const float* k_descale;  /* (H) f32                                                  */
  const float* v_descale;  /* (H, dv) f32, dense                                       */
  int64_t vt_stride_b, vt_stride_h, vt_stride_c;  /* element strides of vt; its key stride is 1 */
  int32_t out_dtype;       /* PCV_BF16 / PCV_F16: dtype of `out`                      */
  int32_t reserved;
} pcv_fp8_attn;

PCV_API int pcv_attn_fwd_fp8_supported(const pcv_attn_params* p, const pcv_fp8_attn* f);
PCV_API int pcv_attn_fwd_fp8(const pcv_attn_params* p, const pcv_fp8_attn* f, void* stream);

/*
 * The fused producer (pcv_kv_project) with e4m3 outputs, for pcv_attn_fwd_fp8: the same LayerNorm-folded GEMM with a
 * bf16 / fp16 mainloop (p->dtype is that of x and w); in the epilogue output column n is multiplied by
 * inv_scale[n] (1 / its descale) and rounded to e4m3 (nearest even, saturating at +-448).
 *   K columns [0, n_k)        -> p->k_out, e4m3 rows with the row stride p->k_stride_row (bytes, a multiple of 16)
 *   V columns [n_k, n_k + n_v) -> vt_out, V transposed: (B, H, v_head_dim, keys) with the strides below, where input
 *                                row r is key r % keys_per_batch of batch row r / keys_per_batch
 * p->v_out / p->v_stride_row are unused.  q is produced the same way with n_v = 0.  One CTA per tile (cta_group 0 or
 * 1).  Arguments are checked before any CUDA call.
 */
typedef struct pcv_kvproj_fp8 {
  const float* inv_scale;  /* (n_k + n_v) f32                                          */
  void* vt_out;            /* e4m3 V^T; may be NULL when n_v == 0                      */
  int64_t vt_stride_b, vt_stride_h, vt_stride_c;  /* byte strides of vt_out; keys contiguous */
  int32_t keys_per_batch;  /* keys per batch row (rows = B * keys_per_batch)           */
  int32_t v_head_dim;      /* V channels per head (a multiple of 16)                   */
} pcv_kvproj_fp8;

PCV_API int pcv_kv_project_fp8_supported(const pcv_kvproj_params* p, const pcv_kvproj_fp8* f);
PCV_API int pcv_kv_project_fp8(const pcv_kvproj_params* p, const pcv_kvproj_fp8* f, void* stream);

/*
 * FP8 (e4m3) KV cache of cached generation: the three kernels below keep a cache's K and V rows as e4m3 codes
 * (strides in elements = bytes) with scales that are not stored in the cache (the caller derives them from the
 * weights).  k / v hold the codes of k_true[h, c] / k_descale[h] and v_true[h, c] / v_descale[h, c].
 *
 * pcv_attn_decode_fp8: the streaming decode kernel (PCV_IMPL_DECODE's) on an e4m3 cache.  `p` is a pcv_attn_params in
 * which dtype (PCV_BF16 / PCV_F16) is that of q and out, and k / v are e4m3 rows whose strides are multiples of 16
 * (16 channels per 16-byte load).  The result is pcv_attn_fwd's on (q, k8 * k_descale[h], v8 * v_descale[h, c]) with
 * fp32 probabilities: k_descale is folded into the scaled q, v_descale multiplies the accumulator once.  Masks and
 * batch-1 q as in pcv_attn_fwd.  N <= 4 query rows, any M >= 1, head dims multiples of 16 and at most 256; impl AUTO or
 * DECODE.  It writes `out` only: write_partial and key shards (m_total != M or m_offset != 0) are refused.  The
 * workspace is pcv_attn_decode_fp8_workspace_bytes() of the same params.  Arguments are checked before any CUDA call.
 */
typedef struct pcv_decode_fp8 {
  const float* k_descale;  /* (H) f32                                                  */
  const float* v_descale;  /* (H, dv) f32, dense                                       */
} pcv_decode_fp8;

PCV_API int pcv_attn_decode_fp8_supported(const pcv_attn_params* p, const pcv_decode_fp8* f);
PCV_API int pcv_attn_decode_fp8_workspace_bytes(const pcv_attn_params* p, size_t* bytes);
PCV_API int pcv_attn_decode_fp8(const pcv_attn_params* p, const pcv_decode_fp8* f, void* stream);

/*
 * pcv_attn_cached_fp8: attention of 1 to 64 query rows on an e4m3 cache on the tensor cores: a cached step that
 * appends several tokens at once.  Operands, descales and result as in pcv_attn_decode_fp8: attention on (q,
 * k8 * k_descale[h], v8 * v_descale[h, c]), with q and out bf16 / fp16 (dtype) and k / v e4m3 rows whose strides are
 * multiples of 16.  The e4m3 tiles are converted to q's 16-bit type in shared memory (exact); q enters unrounded;
 * scale * k_descale[h] multiplies the fp32 scores once, in the exponent; P is rounded to q's 16-bit type before P V
 * (as in pcv_attn_fwd's tensor-core kernel) and v_descale multiplies the fp32 accumulator once.  Masks and batch-1 q
 * as in pcv_attn_fwd.  N <= 64 query rows, any M >= 1, head dims multiples of 16 and at most 256 (independently);
 * impl AUTO.  It writes `out` only: write_partial and key shards are refused, as are an e4m3 q and NULL descales.
 * The workspace is pcv_attn_cached_fp8_workspace_bytes() of the same params; one launch, bitwise reproducible.
 * Arguments are checked before any CUDA call.
 */
PCV_API int pcv_attn_cached_fp8_supported(const pcv_attn_params* p, const pcv_decode_fp8* f);
PCV_API int pcv_attn_cached_fp8_workspace_bytes(const pcv_attn_params* p, size_t* bytes);
PCV_API int pcv_attn_cached_fp8(const pcv_attn_params* p, const pcv_decode_fp8* f, void* stream);

/*
 * pcv_kv_append_fp8: pcv_kv_append onto e4m3 caches.  p->dtype (PCV_BF16 / PCV_F16) is that of k_new / v_new; k_cache,
 * v_cache, k_dst and v_dst are e4m3 (strides in bytes).  The old rows are copied byte for byte (skipped for a half
 * whose cache pointer equals its dst pointer, as in pcv_kv_append); new row channel c becomes
 * e4m3(x[c] * inv_scale[c]) (fp32 product, round to nearest even, saturating at +-448).  Ck and Cv multiples of 16,
 * every pointer (the scales included) 16-byte aligned, e4m3 strides multiples of 16, new-row strides multiples of 8
 * elements.  pcv_kv_append refuses e4m3.  Arguments are checked before any CUDA call.
 */
typedef struct pcv_kv_fp8_scales {
  const float* k_inv_scale;  /* (Ck) f32: 1 / descale of every K channel               */
  const float* v_inv_scale;  /* (Cv) f32                                               */
} pcv_kv_fp8_scales;

PCV_API int pcv_kv_append_fp8_supported(const pcv_kv_append_params* p, const pcv_kv_fp8_scales* f);
PCV_API int pcv_kv_append_fp8(const pcv_kv_append_params* p, const pcv_kv_fp8_scales* f, void* stream);

/*
 * pcv_rotary_apply_fp8: pcv_rotary_apply with e4m3 output: y = e4m3(rotate(x)[h, c] * y_inv_scale[h]).  p->dtype is that
 * of x: PCV_BF16 / PCV_F16, or PCV_E4M3 with x = codes * x_descale[h].  The rotation is computed in fp32 and rounded once.
 * d and every stride even (a channel pair is one 16-bit store).  Arguments are checked before any CUDA call.
 */
typedef struct pcv_rotary_fp8 {
  const float* x_descale;    /* (H) f32, read when p->dtype == PCV_E4M3, else may be NULL */
  const float* y_inv_scale;  /* (H) f32                                                  */
} pcv_rotary_fp8;

PCV_API int pcv_rotary_fp8_supported(const pcv_rotary_params* p, const pcv_rotary_fp8* f);
PCV_API int pcv_rotary_apply_fp8(const pcv_rotary_params* p, const pcv_rotary_fp8* f, void* stream);

/*
 * Device-resident rows: the entry points below read the rows they work on from device memory when the kernel runs, so
 * one recorded CUDA graph serves every step of a decode loop whose lengths change each token.  Every pointer and size
 * in their params is fixed for the life of a graph; only the int32s behind `bounds` change (in-graph tensor ops write
 * them).  None of these entry points synchronises or reads device memory on the host.
 *
 * Every batch row has its own bounds when `bounds_stride_b` > 0: batch row b (the arena's batch row; also with a batch-1
 * q, q_stride_b == 0) reads bounds + b * bounds_stride_b, so each row of a batched decode loop can sit at its own rows
 * (per-row rewind of speculative decoding).  bounds_stride_b == 0: every row reads the same bounds.  A negative stride
 * is refused before any CUDA call.  The grid and the workspace do not depend on the bounds either way.
 *
 * pcv_attn_decode_window (_fp8): the streaming decode kernel on the key window [bounds[0], bounds[1]) of an arena.
 * k, v and pad_mask point at arena row 0 and M == capacity (the arena's rows); pad bytes are indexed by the absolute
 * arena row.  The split count is planned on the host from `capacity`, so the grid and the workspace
 * (pcv_attn_decode_window_workspace_bytes) do not depend on the window; each split takes an equal share of the window's
 * keys when the kernel runs.  The causal mask is right-aligned to the window's end: query i sits at row end - N + i.
 * Any window length >= 1 is valid (the pcv_attn_fwd decode kernel's 1024-key floor does not apply); a window of length
 * <= 0 writes zeros.  The window is clamped to [0, capacity).  N <= 4, head dims multiples of 8 (bf16 / fp16 rows) or
 * 16 (e4m3 rows, with pcv_decode_fp8 as in pcv_attn_decode_fp8) and at most 256; no write_partial, no key shard.
 *
 * pcv_kv_append_at (_fp8): pcv_kv_append (_fp8) of the n new rows to arena rows bounds[0] .. bounds[0] + n - 1, with
 * k_cache = v_cache = NULL and L_old = 0; k_dst / v_dst point at arena row 0.  Rows that would land before row 0 or
 * at or past `capacity` are skipped.
 *
 * pcv_rotary_apply_at (_fp8): pcv_rotary_apply (_fp8) with the angle rows of a precomputed (capacity, rotate_dim) fp32
 * table (`angles`, a_stride_b = 0): input row i uses table row bounds[0] + i and is written to output row bounds[0] + i
 * when bounds[1] != 0 (a new key rotated straight into a rotated-key arena), else to row i (q into a fixed buffer).
 * angle_row0 is ignored; rows whose table row is negative or at or past `capacity` are skipped, whichever output row
 * they would go to.
 */
typedef struct pcv_dev_rows {
  const int32_t* bounds;   /* device int32s; meaning per entry point above                  */
  int32_t capacity;        /* rows of the arena (host-known, fixed for the life of a graph) */
  int32_t bounds_stride_b; /* int32s between the bounds of batch rows b and b + 1; 0: shared */
} pcv_dev_rows;

PCV_API int pcv_attn_decode_window_supported(const pcv_attn_params* p, const pcv_dev_rows* rows);
PCV_API int pcv_attn_decode_window_workspace_bytes(const pcv_attn_params* p, size_t* bytes);
PCV_API int pcv_attn_decode_window(const pcv_attn_params* p, const pcv_dev_rows* rows, void* stream);
PCV_API int pcv_attn_decode_window_fp8_supported(const pcv_attn_params* p, const pcv_decode_fp8* f,
                                                 const pcv_dev_rows* rows);
PCV_API int pcv_attn_decode_window_fp8(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows,
                                       void* stream);

/*
 * pcv_attn_cached_window (_fp8): attention of 1 to 64 query rows on the key window [bounds[0], bounds[1]) of an arena on
 * the tensor cores, with an optional causal band: a k-token step of a decode loop in which every token sees exactly the
 * keys a one-token step gives it.  k, v and pad_mask point at arena row 0 and M == rows->capacity (>= 1); pad bytes
 * are indexed by the absolute arena row.  The window is clamped to [0, capacity); a window of length <= 0 writes zeros.
 * The split count is planned on the host from capacity, so the grid and the workspace
 * (pcv_attn_cached_window (_fp8)_workspace_bytes) do not depend on the window; each split takes an equal share of the
 * window's 64-key tiles when the kernel runs.  Query i sits at row r_i = end - N + i.
 *   band == 0: the causal mask (if set) is right-aligned to the window's end; padded and causally masked keys take the
 *              finite fill, as in pcv_attn_cached_fp8 (a fully masked row is the uniform average of the window);
 *   band  > 0: causal only; query i sees the keys [r_i + 1 - band, r_i] of the window and nothing else: a key outside
 *              that band contributes nothing (no fill), padded keys inside it take the fill.
 * pcv_attn_cached_window: k / v are rows of q's type (dtype PCV_BF16 / PCV_F16), head dims multiples of 8.
 * pcv_attn_cached_window_fp8: k / v are e4m3 rows with pcv_decode_fp8 descales as in pcv_attn_cached_fp8, head dims
 * multiples of 16.  Arithmetic as pcv_attn_cached_fp8: q unrounded, P rounded to q's type before P V, fp32
 * denominators, v_descale applied to the accumulator once; with the window [0, capacity) and no band the e4m3 entry
 * computes pcv_attn_cached_fp8's result bit for bit.  Head dims at most 256; impl AUTO; no write_partial, no key shard.
 * One launch, bitwise reproducible.  Arguments are checked before any CUDA call.
 */
PCV_API int pcv_attn_cached_window_supported(const pcv_attn_params* p, const pcv_dev_rows* rows, int32_t band);
PCV_API int pcv_attn_cached_window_workspace_bytes(const pcv_attn_params* p, size_t* bytes);
PCV_API int pcv_attn_cached_window(const pcv_attn_params* p, const pcv_dev_rows* rows, int32_t band, void* stream);
PCV_API int pcv_attn_cached_window_fp8_supported(const pcv_attn_params* p, const pcv_decode_fp8* f,
                                                 const pcv_dev_rows* rows, int32_t band);
PCV_API int pcv_attn_cached_window_fp8_workspace_bytes(const pcv_attn_params* p, size_t* bytes);
PCV_API int pcv_attn_cached_window_fp8(const pcv_attn_params* p, const pcv_decode_fp8* f, const pcv_dev_rows* rows,
                                       int32_t band, void* stream);
PCV_API int pcv_kv_append_at(const pcv_kv_append_params* p, const pcv_dev_rows* rows, void* stream);
PCV_API int pcv_kv_append_at_fp8(const pcv_kv_append_params* p, const pcv_kv_fp8_scales* f, const pcv_dev_rows* rows,
                                 void* stream);
PCV_API int pcv_rotary_apply_at(const pcv_rotary_params* p, const pcv_dev_rows* rows, void* stream);
PCV_API int pcv_rotary_apply_at_fp8(const pcv_rotary_params* p, const pcv_rotary_fp8* f, const pcv_dev_rows* rows,
                                    void* stream);

/*
 * Token sampling: pcv_sample draws one token per row of R logits rows of V entries, with temperature, top-k and top-p
 * filtering in the semantics of the Hugging Face TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper, then
 * softmax + multinomial.  Row r belongs to batch row b = r / rows_per_batch.
 *   x_i = float(logit_i) / temperature (a true fp32 division); temperature == 0 is greedy: the argmax, the lowest index
 *   on ties, log-probability 0, nothing random drawn.  A row whose largest x is -inf or +inf (every logit -inf, e.g.
 *   after n-gram blocking has banned the whole vocabulary, or logit / temperature overflowing fp32) has no finite
 *   softmax and is taken as greedy too: the lowest index of the largest x (index 0 when every x is -inf, as
 *   torch.argmax), log-probability 0.  The Hugging Face warpers raise an error on such a row.
 *   top_k > 0: keep every token with x_i >= the k-th largest x (all ties with it); 0 or >= V: off.
 *   top_p < 1: with masses w_i = round(2^40 exp(x_i - max x)) (uint64) of the kept tokens, Z their sum and
 *   W<=(v) the mass of the kept tokens with x <= v, token i is removed iff W<=(x_i) <= floor((1 - top_p) Z) (fp64
 *   product); a tie group straddling the cut is kept whole, and the top group always stays.  1: off.
 *   The token is the first index, in vocabulary order, whose kept prefix mass exceeds hi64(u * Z_kept), with u the 64
 *   bits pcv_sample_uniforms exports for (seeds[b], b, positions[r]).
 * A row's token is a pure function of its logit bits, the three filter values, seeds[b], b and positions[r]:
 * independent of R, of the other rows, of the launch and of graph capture.  Seeds and positions are read from device
 * memory when the kernel runs, so one recorded CUDA graph serves every seed and position.  Logits must be free of NaN
 * and +inf.  Refusals (NULL pointers, V outside [1, PCV_SAMPLE_MAX_VOCAB], stride_row < V, R not a multiple of
 * rows_per_batch, temperature < 0 or NaN, top_k < 0, top_p outside (0, 1] or NaN, an unknown dtype) come before any
 * CUDA call, with the reason in pcv_last_error.
 */
#define PCV_SAMPLE_MAX_VOCAB 32768

typedef struct pcv_sample_params {
  const void* logits;        /* (R, V) rows of `dtype` (PCV_BF16 / PCV_F16 / PCV_F32), unit element stride */
  int64_t stride_row;        /* elements between rows, >= V                                                */
  int32_t R, V;
  int32_t dtype;
  int32_t rows_per_batch;    /* R / rows_per_batch batch rows                                              */
  const uint64_t* seeds;     /* device, one per batch row                                                  */
  const int32_t* positions;  /* device, one per row: the counter of the row's draw                          */
  float temperature;         /* >= 0; 0: greedy                                                            */
  int32_t top_k;             /* >= 0; 0: off                                                               */
  float top_p;               /* (0, 1]; 1: off                                                             */
  int32_t reserved;
  int64_t* tokens;           /* device (R) out: token ids                                                  */
  float* logprobs;           /* device (R) out or NULL: the token's log-probability under the filtered distribution */
} pcv_sample_params;

/* 1 if pcv_sample takes these params, else 0 (reason via pcv_last_error) */
PCV_API int pcv_sample_supported(const pcv_sample_params* p);
PCV_API int pcv_sample(const pcv_sample_params* p, void* stream);
/* out[r] (device, R) = the 64 random bits of row r's draw: (seeds[r / rows_per_batch], r / rows_per_batch,
 * positions[r]).  Arguments are checked before any CUDA call. */
PCV_API int pcv_sample_uniforms(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int32_t R,
                                int32_t rows_per_batch, void* stream);

/*
 * Speculative sampling with a draft model's probabilities (Leviathan et al. 2023; Chen et al. 2023): pcv_spec_verify
 * decides one round of G drafts for each of B batch rows.  Row b fed tokens t_0 .. t_G (tokens[b]) to both models; t_1
 * .. t_G are the draft's draws.  Target row i (i = 0 .. G) holds the target's logits after t_i, draft row i (i < G) the
 * logits the draft drew t_{i+1} from.  P_i / Zp_i are the kept masses of target row i and their sum under (temperature,
 * top_k, top_p), exactly as pcv_sample computes them (greedy, and a row pcv_sample takes as greedy because its largest
 * scaled value is not finite: 2^40 at the first maximal index, 0 elsewhere); Q_i / Zq_i those of draft row i under the
 * draft_* values, by the same rule, so that Q is the distribution pcv_sample drew the draft from.  All arithmetic is exact integer arithmetic:
 *   accept t_{i+1} = x iff hi64(u_a * Q_i(x) * Zp_i) < P_i(x) * Zq_i   (min(1, p/q) to 2^-64), with u_a the accept
 *   stream's bits at (seeds[b], b, positions[b, i]).  A draft with Q_i(x) = 0 (one not drawn from Q) is accepted iff
 *   P_i(x) > 0; a token outside [0, V) is rejected.
 *   n_b = the first rejected i, or G.
 *   n_b < G: the correction is the first index, in vocabulary order, whose prefix sum of
 *   R(y) = max(0, P(y) Zq - Q(y) Zp) (row n_b) exceeds hi64(u_r * ΣR), u_r the residual stream's bits at
 *   positions[b, n_b].  ΣR = 0 (reached only by a draft that neither P nor Q gives mass): a draw from P with u_r.
 *   n_b = G: the bonus token, the first index whose prefix P_G mass exceeds hi64(u_r * Zp_G), u_r at positions[b, G].
 *   out_tokens[b, :n_b] = t_1 .. t_{n_b}, out_tokens[b, n_b] = the correction or bonus token, the rest -1;
 *   accepted[b] = n_b.
 * The accept and residual streams are counter-based hashes independent of each other and of pcv_sample's draw stream
 * at equal (seed, b, position), so the draft may share the target's seeds; pcv_spec_uniforms exports them.  A row's
 * result is a pure function of its logit bits, both sets of filter values, its tokens, seeds[b], b and its positions:
 * independent of B, of the launch and of graph capture.  Two kernels, no host read: one CTA per (b, i), then one thread
 * per batch row resolves n_b in place in out_tokens, which is the only scratch.  Refusals (NULL pointers, V outside
 * [1, PCV_SAMPLE_MAX_VOCAB], G outside [1, PCV_SPEC_MAX_DRAFTS], B < 1, a stride below V, draft_dtype != dtype, an
 * unknown dtype, out_tokens overlapping tokens, either set of filter values out of range) come before any CUDA call,
 * with the reason in pcv_last_error.
 */
#define PCV_SPEC_MAX_DRAFTS 63

typedef struct pcv_spec_verify_params {
  const void* target;          /* (B, G+1, V) target logits of `dtype`, unit element stride                       */
  int64_t t_stride_b, t_stride_row;
  const void* draft;           /* (B, G, V) draft logits of `draft_dtype` (== dtype), unit element stride           */
  int64_t d_stride_b, d_stride_row;
  const int64_t* tokens;       /* device (B, G+1) contiguous: the fed tokens t_0 .. t_G                             */
  const uint64_t* seeds;       /* device (B)                                                                        */
  const int32_t* positions;    /* device (B, G+1) contiguous: the counter of a token decided by target row i        */
  int32_t B, G, V;
  int32_t dtype, draft_dtype;  /* PCV_BF16 / PCV_F16 / PCV_F32                                                      */
  int32_t reserved;
  float temperature;           /* the target's filter values, as pcv_sample takes them                              */
  int32_t top_k;
  float top_p;
  float draft_temperature;     /* the draft's                                                                       */
  int32_t draft_top_k;
  float draft_top_p;
  int64_t* out_tokens;         /* device (B, G+1) out                                                               */
  int32_t* accepted;           /* device (B) out: n_b                                                               */
} pcv_spec_verify_params;

/* 1 if pcv_spec_verify takes these params, else 0 (reason via pcv_last_error) */
PCV_API int pcv_spec_verify_supported(const pcv_spec_verify_params* p);
PCV_API int pcv_spec_verify(const pcv_spec_verify_params* p, void* stream);
/* out[r] (device, R) = the 64 bits of stream stream_id (0: accept, 1: residual) at (seeds[r / rows_per_batch],
 * r / rows_per_batch, positions[r]).  Arguments are checked before any CUDA call. */
PCV_API int pcv_spec_uniforms(uint64_t* out, const uint64_t* seeds, const int32_t* positions, int32_t R,
                              int32_t rows_per_batch, int32_t stream_id, void* stream);

/*
 * Beam search: pcv_beam_step runs one step of the Hugging Face GenerationMixin._beam_search (do_sample=False; logits
 * processors through pcv_logits_process and pcv_beam_step_logprobs) for B items of K beams each, on state buffers that live on the device.  Beam k of item b is logits row
 * b*K + k.  E = n_eos, beams_to_keep = max(2, E + 1) * K (as the Hugging Face code keeps them).  For each item:
 *   1. logp = log_softmax(fp32 logits) per beam row: d_i = (double)x_i - (double)max, S = Σ exp(d_i) in fp64,
 *      logp_i = fp32(d_i - log S);
 *   2. acc = fp32(running_scores[b, k] + logp); the top beams_to_keep of the K*V values by score descending, then flat
 *      index k*V + token ascending (the tie rule);
 *   3. a candidate hits the stopping criteria if its token is an EOS id or it is the max_length-th generated token
 *      (generated count + 1 >= max_length);
 *   4. running beams: hitting candidates get -1e9 added (fp32) and the top K (ties by candidate position) give
 *      next_tokens, parents (global beam rows b*K + parent beam) and the running scores;
 *   5. finished set: of the first K candidates those that just hit are eligible; scores are divided in fp32 by
 *      fp32(pow(g, length_penalty)) (fp64 pow of the fp64 penalty, g = generated count + 1), get -1e9 if early_stopping is TRUE and the
 *      item's K finished flags are all set, -1e9 if the item's early-stop heuristic is satisfied, -1e9 if not eligible,
 *      and are merged with the K finished entries; the top K are kept, ties by position in [finished | candidates];
 *   6. the early-stop heuristic (sticky) on the new state, as the Hugging Face code computes it, and the item's done
 *      flag: heuristic satisfied, or early_stopping TRUE and every finished flag set.
 * Token histories (running and finished, hist_len columns per beam) are gathered by parent; column `generated count`
 * takes the new token.  The last item CTA to finish sets counters[2] = every item done and counters[0] += 1.  The
 * generated count and max_length are read from counters when the kernels run, so one recorded CUDA graph serves every
 * step.  Initial state: running scores 0 for beam 0 and -1e9 for the others, finished scores -1e9, flags 0, histories
 * filled with the output fill value, item_flags {1, 0}, counters {0, max_length, 0, 0}.  Two launches (one CTA per
 * beam row, one per item), no host read, integer atomics only; an item's result is a pure function of its logit bits
 * and state.  Refusals (NULL pointers, V outside [1, PCV_SAMPLE_MAX_VOCAB], K outside [1, PCV_BEAM_MAX_BEAMS], n_eos
 * outside [0, PCV_BEAM_MAX_EOS], K*V < beams_to_keep, an EOS id outside [0, V), a non-finite length_penalty, an
 * unknown early_stopping code or dtype, stride_row < V, overlapping outputs) come before any CUDA call, with the reason
 * in pcv_last_error.
 */
#define PCV_BEAM_MAX_BEAMS 8
#define PCV_BEAM_MAX_EOS 4
enum pcv_early_stopping { PCV_EARLY_STOP_FALSE = 0, PCV_EARLY_STOP_TRUE = 1, PCV_EARLY_STOP_NEVER = 2 };

typedef struct pcv_beam_step_params {
  const void* logits;          /* (B*K, V) rows of `dtype` (PCV_BF16 / PCV_F16 / PCV_F32), unit element stride */
  int64_t stride_row;          /* elements between rows, >= V                                                  */
  double length_penalty;       /* fp64, as the Hugging Face code raises the length to it                       */
  int32_t B, K, V, dtype;
  int32_t n_eos;
  int32_t eos[PCV_BEAM_MAX_EOS];
  int32_t early_stopping;      /* pcv_early_stopping                                                           */
  int32_t hist_len;            /* columns of every history row (>= max_length)                                 */
  float* running_scores;       /* (B, K) state                                                                  */
  float* finished_scores;      /* (B, K) state                                                                  */
  int32_t* finished_flags;     /* (B, K) state                                                                  */
  int64_t* running_hist;       /* (B, K, hist_len) state                                                        */
  int64_t* finished_hist;      /* (B, K, hist_len) state                                                        */
  int64_t* hist_scratch;       /* (B, 2K, hist_len) scratch                                                     */
  int32_t* item_flags;         /* (B, 2) state: [early-stop heuristic not satisfied, item done]                 */
  int32_t* counters;           /* 4 int32s: [generated count, max_length, every item done, arrivals (0)]        */
  float* cand_scores;          /* (B*K, beams_to_keep) scratch                                                  */
  int32_t* cand_index;         /* (B*K, beams_to_keep) scratch                                                  */
  int64_t* next_tokens;        /* (B*K) out                                                                     */
  int32_t* parents;            /* (B*K) out: the global beam row each beam continues                            */
} pcv_beam_step_params;

/* 1 if pcv_beam_step takes these params, else 0 (reason via pcv_last_error) */
PCV_API int pcv_beam_step_supported(const pcv_beam_step_params* p);
PCV_API int pcv_beam_step(const pcv_beam_step_params* p, void* stream);
/* pcv_beam_step on rows that already are fp32 log-probabilities (pcv_logits_process with log_softmax = 1): step 1 is
 * skipped, logp_i = x_i, and everything after it is the same.  The same params and refusals, and dtype must be
 * PCV_F32. */
PCV_API int pcv_beam_step_logprobs_supported(const pcv_beam_step_params* p);
PCV_API int pcv_beam_step_logprobs(const pcv_beam_step_params* p, void* stream);

/*
 * Logits processors: pcv_logits_process applies the Hugging Face RepetitionPenaltyLogitsProcessor (without
 * prompt_ignore_length), NoRepeatNGramLogitsProcessor and MinNewTokensLengthLogitsProcessor, in that order, to R rows,
 * one 512-thread CTA per row.  Processed row r reads logits row s = r (row_map NULL) or s = r * row_group + row_map[r]
 * and writes out row s, fp32:
 *   0. x = the fp32 logits; with log_softmax = 1, x_i = fp32(d_i - log S), d_i = (double)x_i - (double)max and
 *      S = Σ exp(d_i) in fp64, exactly as step 1 of pcv_beam_step;
 *   1. repetition_penalty θ (1: off): every distinct id of the history in [0, V) once, x = x < 0 ? fp32(x * fp32(θ))
 *      : fp32(x / fp32(θ));
 *   2. no_repeat_ngram N (0: off), L the history length: if L + 1 >= N, for every start s in [0, L - N + 1) with
 *      hist[s .. s+N-1) == hist[L-N+1 .. L), x[hist[s+N-1]] = -inf (N = 1 bans every id of the history);
 *   3. min_new_tokens M (0: off): if L - prompt_len < M, x[eos] = -inf for every EOS id.
 * Ids outside [0, V) take part in the n-gram matching; their own score is never written.  The history of row r is
 * history row h = r / rows_per_hist: prefix[h * prefix_stride + 0 .. Lp) then tail[h * tail_stride + 0 .. Lt), where
 * Lp = prefix_len ? prefix_len[r * prefix_len_stride] : prefix_count and Lt = tail_len ? tail_len[r *
 * tail_len_stride] : 0 are read when the kernel runs (so one recorded CUDA graph serves every step), each clamped to
 * [0, its cap].  No floating-point atomics: a row's output is a pure function of its inputs.  Refusals (NULL pointers,
 * V outside [1, PCV_SAMPLE_MAX_VOCAB], R < 1, an unknown dtype, a stride below V, θ not finite and > 0, N outside [0,
 * PCV_PROCESS_MAX_NGRAM], M < 0, M > 0 without EOS ids, n_eos outside [0, PCV_PROCESS_MAX_EOS], an EOS id outside
 * [0, V), rows_per_hist < 1, negative caps, counts or strides) come before any CUDA call, with the reason in
 * pcv_last_error.
 */
#define PCV_PROCESS_MAX_NGRAM 8
#define PCV_PROCESS_MAX_EOS 4

typedef struct pcv_logits_process_params {
  const void* logits;          /* rows of `dtype` (PCV_BF16 / PCV_F16 / PCV_F32), unit element stride         */
  int64_t stride_row;          /* elements between logits rows, >= V                                          */
  float* out;                  /* fp32 rows, unit element stride                                              */
  int64_t out_stride_row;      /* elements between out rows, >= V                                             */
  const int32_t* row_map;      /* device (R) or NULL                                                          */
  const int64_t* prefix;       /* history prefixes                                                            */
  int64_t prefix_stride;       /* elements between history rows' prefixes                                     */
  const int64_t* tail;         /* history tails, or NULL (then tail_len must be NULL)                         */
  int64_t tail_stride;
  const int32_t* prefix_len;   /* device or NULL (then prefix_count)                                          */
  const int32_t* tail_len;     /* device or NULL (then 0)                                                     */
  int32_t prefix_len_stride, tail_len_stride;
  int32_t prefix_count, prefix_cap, tail_cap;
  int32_t R, V, dtype, row_group, rows_per_hist;
  int32_t log_softmax;         /* 0 or 1                                                                      */
  float repetition_penalty;
  int32_t no_repeat_ngram;
  int32_t min_new_tokens;
  int32_t prompt_len;          /* the prompt's padded width: new tokens = L - prompt_len                      */
  int32_t n_eos;
  int32_t eos[PCV_PROCESS_MAX_EOS];
} pcv_logits_process_params;

/* 1 if pcv_logits_process takes these params, else 0 (reason via pcv_last_error) */
PCV_API int pcv_logits_process_supported(const pcv_logits_process_params* p);
PCV_API int pcv_logits_process(const pcv_logits_process_params* p, void* stream);

/*
 * Prompt-lookup drafts: pcv_prompt_lookup finds each batch row's drafts in its own history, with the rule of the
 * Hugging Face PromptLookupCandidateGenerator.get_candidates (no logits processor) applied to each row alone.  One CTA
 * per row.  Row b's history is h = ids[b, s .. L), s = start[b] (its left-padding count; NULL: 0) clamped to [0, L],
 * L = length[b * length_stride] + length_offset (+ n_b in round mode) clamped to [0, cap]; len = L - s:
 *   1. for n = min(N, len - 1) down to 1: the first window h[e-n+1 .. e] (smallest e) equal to h[len-n .. len) with
 *      e <= len - 2 (it has a continuation);
 *   2. the draft is h[e+1 .. min(e+1+G, len)) of the largest n that has such a window, cut before its first EOS id
 *      (empty after the cut: no draft, and no other window is tried), then capped at the row's limit;
 *   3. counts[b] = its length, drafts[b, :counts[b]] = the draft, drafts[b, counts[b] .. G) = h[len-1] (filler; 0 for
 *      an empty history).
 * The limit is limit[b] (NULL: G) in search mode (k = 0).  Round mode (1 <= k <= G+1) first settles the round that fed
 * fed[b, 0 .. k) (t_0 and counts[b] drafts, then filler) and drew draws[b, i] after fed[b, i]: a row is live while
 * unfinished[b] != 0 and left[b] > 0.  A live row accepts n_b = the leading i < counts[b] with fed[b, i+1] ==
 * draws[b, i], emits those drafts and t = draws[b, n_b], sets left[b] -= n_b + 1, unfinished[b] = 0 if t is an EOS id,
 * writes t into ids at row L - 1 (the row it will be fed at) and searches with the limit left[b] - 1 if it is still
 * live.  A row that is not live keeps t = fed[b, 0], n_b = 0 and gets no draft (its history ends at t: L is one
 * less).  accepted[b] = n_b, t0[b] = t.
 * Integer comparisons only, a block-min over window ends and no atomics on results: a row's output is a pure
 * function of its ids, lengths, G, N, the EOS ids and its limit / state, independent of B, the launch and graph
 * capture.  Refusals (NULL pointers, B < 1, cap < 1, ids_stride < cap, G outside [1, PCV_LOOKUP_MAX_DRAFTS], N outside
 * [1, PCV_LOOKUP_MAX_NGRAM], n_eos outside [0, PCV_LOOKUP_MAX_EOS], drafts_stride < G, k outside [0, G+1], a round
 * without its state, t0_stride < 1) come before any CUDA call, with the reason in pcv_last_error.
 */
#define PCV_LOOKUP_MAX_DRAFTS 63
#define PCV_LOOKUP_MAX_NGRAM 16
#define PCV_LOOKUP_MAX_EOS 4

typedef struct pcv_prompt_lookup_params {
  int64_t* ids;                /* device (B, cap) history rows (round mode writes t into them)                    */
  int64_t ids_stride;          /* elements between rows, >= cap                                                  */
  const int32_t* start;        /* device (B) left-padding counts, or NULL (0)                                    */
  const int32_t* length;       /* device: L = length[b * length_stride] + length_offset                         */
  int32_t length_stride, length_offset;
  const int32_t* limit;        /* device (B) per-row draft caps, or NULL (G); search mode only                   */
  int32_t B, cap, G, N;
  int32_t n_eos;
  int32_t k;                   /* 0: search only; 1 .. G+1: settle the round that fed k tokens, then search      */
  int64_t eos[PCV_LOOKUP_MAX_EOS];
  int64_t* drafts;             /* device (B, drafts_stride) out                                                   */
  int64_t drafts_stride;
  int32_t* counts;             /* device (B) out (round mode: in first, the drafts the round fed)                 */
  int32_t reserved;
  const int64_t* fed;          /* round mode: device (B, k) contiguous, t_0 then the drafts and filler            */
  const int64_t* draws;        /* round mode: device (B, k) contiguous, the draw after each fed token             */
  int64_t* t0;                 /* round mode: device (B, t0_stride) out, the next t_0                              */
  int64_t t0_stride;
  int32_t* accepted;           /* round mode: device (B) out, n_b                                                  */
  int32_t* unfinished;         /* round mode: device (B) state                                                     */
  int32_t* left;               /* round mode: device (B) state, the tokens each row still emits                    */
} pcv_prompt_lookup_params;

/* 1 if pcv_prompt_lookup takes these params, else 0 (reason via pcv_last_error) */
PCV_API int pcv_prompt_lookup_supported(const pcv_prompt_lookup_params* p);
PCV_API int pcv_prompt_lookup(const pcv_prompt_lookup_params* p, void* stream);

/*
 * pcv_kv_gather_rows: after a beam step, every beam row i with parents[i] != i takes its parent's generated rows.  For
 * every arena of the device table and every such row i, rows [first_row, cur) with cur = rows->bounds[i *
 * bounds_stride_b + bounds_col] (clamped to first_row + max_rows) are copied from row parents[i] into row i, through
 * the entry's scratch (parent -> scratch, then scratch -> child, two launches), so cycles and many-to-one moves read
 * only the rows as they were before the call.  Rows whose parent is themselves, rows before first_row or at / past cur,
 * and every other arena byte are untouched.  The grid is (n_entries, R) whatever the bounds: the call can be recorded
 * in a CUDA graph.  Each entry's arena and scratch are 16-byte aligned, row_bytes and the strides multiples of 16, and
 * the scratch holds max_rows rows per beam row (the caller builds the table; only the params are checked).
 * last_rows = 0 moves every generated row as above; last_rows > 0 moves only [max(first_row, cur - last_rows), cur):
 * with 1, the row a step just appended (contrastive search, whose rows of an item share every earlier row).
 */
typedef struct pcv_kv_gather_entry {
  void* arena;                 /* batch row 0, arena row 0                                                      */
  void* scratch;               /* beam row 0's max_rows rows                                                    */
  int64_t arena_stride_b;      /* bytes between batch rows of the arena                                         */
  int64_t scratch_stride_b;    /* bytes between beam rows of the scratch                                        */
  int32_t row_bytes;
  int32_t first_row;           /* the first generated row of the arena's layer group                            */
  int32_t bounds_col;          /* the int32 of a beam row's bounds that holds its current row                   */
  int32_t max_rows;            /* generated rows the arena holds after first_row                                */
} pcv_kv_gather_entry;

typedef struct pcv_kv_gather_params {
  const pcv_kv_gather_entry* table;   /* device (n_entries)                                                     */
  int32_t n_entries, R;
  const int32_t* parents;             /* device (R): the global beam row each row continues                     */
  int32_t last_rows;                  /* >= 0; 0: every generated row, n: only the newest n                      */
  int32_t reserved;
} pcv_kv_gather_params;

PCV_API int pcv_kv_gather_rows_supported(const pcv_kv_gather_params* p, const pcv_dev_rows* rows);
PCV_API int pcv_kv_gather_rows(const pcv_kv_gather_params* p, const pcv_dev_rows* rows, void* stream);

/*
 * Contrastive search (Su et al. 2022) on the device, with the semantics of the Hugging Face 4.28
 * GenerationMixin.contrastive_search (no logits processors or warpers), for B items of K = top_k candidate rows each:
 * candidate j of item b is batch row b*K + j.  All arithmetic of the ranking is fp64 (the Hugging Face code computes it
 * in the model dtype, so on near-ties it may choose differently).  One step of item b:
 *   pcv_contrastive_candidates, one 512-thread CTA per item: x = the fp32 logits of row b*K + sel[b] (sel = 0 after the
 *     prompt, whose K rows are equal); the K largest x, value descending then index ascending on ties (-0 == +0), are
 *     the candidates cand[b, j]; p_j = exp(x_j - m) / Σ_i exp(x_i - m) in fp64 (m = max x); next_tokens[b*K + j] =
 *     cand[b, j].  A row with -inf entries ranks them last, in index order; a row whose every entry is -inf has no
 *     finite softmax (NaN probabilities, as in 4.28) and is unsupported.
 *   pcv_contrastive_rank, after the model ran row b*K + j on candidate j and produced its final hidden row h_j:
 *     1. cos(c_s, h_j) = (Σ_d c_sd h_jd) / (sqrt(‖c_s‖²) sqrt(‖h_j‖²)) in fp64 (16-bit products are exact; one fixed
 *        summation order), 0 when either norm is 0; c_s are the item's context rows;
 *     2. pen_j = the max of cos over the live context rows whose squared norm is not negative (negative: a padding row
 *        of the prompt, skipped); 0 when no row counts;
 *     3. score_j = (1 - α) p_j - α pen_j (fp64, each operation rounded); sel = the lowest j attaining the max;
 *     4. emit = unfinished[b] ? cand[b, sel] : pad_token, written to history[b, generated count];
 *        unfinished[b] &= emit is no EOS id; parents[b*K + j] = b*K + sel for every j;
 *     5. the context grows by h_sel (its squared norm computed once, by the order of step 1).
 *   The last item CTA sets counters[2] = every item finished and advances counters[0] (context length) and counters[1]
 *   (generated count); both are read when the kernels run, so one recorded CUDA graph serves every step.  The KV select
 *   that follows is pcv_kv_gather_rows with last_rows = 1 and these parents.  Initial state: context rows and squared
 *   norms of the prompt loaded, unfinished 1, sel 0, counters {prompt context length, 0, 0, 0}.  No floating-point
 *   atomics; the context is split across CTAs of PCV_CONTRASTIVE_ROWS_PER_CTA rows, each computing its rows' maxima,
 *   and a max is exact in any order, so an item's result is a pure function of its inputs and state.  Refusals (NULL
 *   pointers, V outside [1, PCV_SAMPLE_MAX_VOCAB], K outside [1, PCV_CONTRASTIVE_MAX_K] or above V, D outside [8,
 *   PCV_CONTRASTIVE_MAX_HIDDEN] or not a multiple of 8, α outside [0, 1], n_eos outside [0, PCV_CONTRASTIVE_MAX_EOS],
 *   an unknown dtype, misaligned hidden rows, overlapping outputs) come before any CUDA call, with the reason in
 *   pcv_last_error.
 */
#define PCV_CONTRASTIVE_MAX_K 16
#define PCV_CONTRASTIVE_MAX_HIDDEN 4096
#define PCV_CONTRASTIVE_MAX_EOS 4
#define PCV_CONTRASTIVE_ROWS_PER_CTA 32

typedef struct pcv_contrastive_candidates_params {
  const void* logits;          /* (B*K, V) rows of `dtype` (PCV_BF16 / PCV_F16 / PCV_F32), unit element stride */
  int64_t stride_row;          /* elements between rows, >= V                                                  */
  int32_t B, K, V, dtype;
  const int32_t* sel;          /* device (B): the selected candidate of each item                               */
  double* probs;               /* (B, K) out: p_j                                                               */
  int32_t* cand;               /* (B, K) out: candidate token ids                                               */
  int64_t* next_tokens;        /* (B*K) out                                                                     */
} pcv_contrastive_candidates_params;

typedef struct pcv_contrastive_rank_params {
  const void* hidden;          /* (B*K, D) rows of hidden_dtype (PCV_BF16 / PCV_F16), 16-byte aligned rows       */
  int64_t hidden_stride_row;   /* elements between rows, >= D, a multiple of 8                                 */
  void* context;               /* (B, cap, D) hidden_dtype, contiguous, 16-byte aligned                         */
  double* context_norm2;       /* (B, cap) squared norms; negative: a padding row                               */
  const double* probs;         /* (B, K) from pcv_contrastive_candidates                                        */
  const int32_t* cand;         /* (B, K) from pcv_contrastive_candidates                                        */
  double alpha;                /* penalty_alpha, in [0, 1]                                                       */
  int64_t pad_token;           /* emitted once an item is finished                                              */
  int32_t B, K, D, hidden_dtype;
  int32_t cap;                 /* context rows per item                                                         */
  int32_t hist_len;            /* columns of every history row                                                  */
  int32_t n_eos;
  int32_t eos[PCV_CONTRASTIVE_MAX_EOS];
  int32_t reserved;
  double* partial;             /* (B, ceil(cap / PCV_CONTRASTIVE_ROWS_PER_CTA), K) scratch                       */
  int32_t* sel;                /* (B) out                                                                       */
  int32_t* unfinished;         /* (B) state                                                                     */
  int64_t* history;            /* (B, hist_len) out: the emitted tokens                                         */
  int32_t* counters;           /* 4 int32s: [context length, generated count, every item finished, arrivals (0)] */
  int32_t* parents;            /* (B*K) out: the batch row each row continues                                   */
} pcv_contrastive_rank_params;

/* 1 if the call takes these params, else 0 (reason via pcv_last_error) */
PCV_API int pcv_contrastive_candidates_supported(const pcv_contrastive_candidates_params* p);
PCV_API int pcv_contrastive_candidates(const pcv_contrastive_candidates_params* p, void* stream);
PCV_API int pcv_contrastive_rank_supported(const pcv_contrastive_rank_params* p);
PCV_API int pcv_contrastive_rank(const pcv_contrastive_rank_params* p, void* stream);

/*
 * Backward of the LayerNorm -> Linear chain pcv_kv_project computes (training through kv_norm -> k_proj / v_proj,
 * q_norm -> q_proj, norm -> q/k/v_proj).  With x_hat = (x - mean) * rstd (row_stats of pcv_ln_stats),
 * y = x_hat * gamma + beta, out = y W^T + b, W = [W_k ; W_v] (n_k + n_v, C) and G = [grad_k | grad_v] (rows, n):
 *   grad_b = G^T 1,  grad_w = (G^T x_hat) diag(gamma) + grad_b beta^T,
 *   dy = G W,  grad_gamma = sum_rows dy * x_hat,  grad_beta = sum_rows dy,
 *   grad_x = rstd * (dx_hat - (a + x_hat * b) / C),  dx_hat = gamma * dy,  a = sum_c dx_hat,  b = sum_c dx_hat * x_hat.
 * Two wgmma GEMMs (dy = G W with dx_hat written to grad_x and per-tile fp32 row / column partials; G^T x_hat with x_hat
 * formed in registers from x and the statistics and rounded to 16 bits) and three small kernels that sum the partials
 * in a fixed order: no atomics, every gradient is bitwise reproducible.
 *   x          : (rows, C) with a row stride; w: (n_k + n_v, C) contiguous, the UNFOLDED weights
 *   gamma/beta : (C) or NULL (gamma NULL = 1, beta NULL = 0)
 *   grad_k/v   : (rows, n_k) / (rows, n_v), each with its own row stride (as k_out / v_out of pcv_kv_project)
 *   grad_x     : (rows, C) contiguous; grad_w (n_k + n_v, C) contiguous; grad_b (n_k + n_v); grad_gamma / grad_beta
 *                (C).  Each may be NULL when it is not needed.
 * All tensors are in `dtype`.  Widths and alignment as pcv_kv_project (C and n_v multiples of 8, n_k a multiple of 64,
 * strides multiples of 8 elements, 16-byte aligned x / w / grad_k / grad_v / grad_x).  The workspace
 * (pcv_ln_linear_bwd_workspace_bytes, a function of rows, C, n_k and n_v alone) is 256-byte aligned.  Arguments are
 * checked before any CUDA call.
 */
typedef struct pcv_ln_linear_bwd_params {
  const void* x;
  int64_t x_stride_row;
  const float* row_stats;  /* (rows, 2) f32 (mean, rstd) */
  const void* w;
  const void* gamma;
  const void* beta;
  const void* grad_k;
  const void* grad_v;
  int64_t gk_stride_row, gv_stride_row;
  void* grad_x;
  void* grad_w;
  void* grad_b;
  void* grad_gamma;
  void* grad_beta;
  int64_t rows;
  int32_t C, n_k, n_v;
  int32_t dtype;           /* PCV_BF16 / PCV_F16 */
  void* workspace;
  size_t workspace_bytes;
} pcv_ln_linear_bwd_params;

/* 1 if pcv_ln_linear_bwd covers this problem, else 0 (reason via pcv_last_error) */
PCV_API int pcv_ln_linear_bwd_supported(const pcv_ln_linear_bwd_params* p);
PCV_API int pcv_ln_linear_bwd_workspace_bytes(const pcv_ln_linear_bwd_params* p, size_t* bytes);
PCV_API int pcv_ln_linear_bwd(const pcv_ln_linear_bwd_params* p, void* stream);

/*
 * Live timing of the dominant kernel (bench.py's roofline leg): between pcv_profile_begin() and
 * pcv_profile_end() every attention main-kernel launch is bracketed by CUDA events on its own
 * stream; pcv_profile_end() synchronises those events and returns their summed duration.
 */
PCV_API int pcv_profile_begin(void);
PCV_API int pcv_profile_end(double* main_kernel_ms_total, int32_t* main_kernel_launches);

/*
 * Watchdog record of the tensor-core kernels (attention forward and its cross-GPU merge, backward, dropout
 * forward, K/V projection), one for the whole library: every in-kernel barrier wait is bounded (4 s); the first
 * wait that times out writes {1, site, blockIdx, threadIdx, parity or expected value, spins or seen value} to a
 * pinned host buffer and traps, so a pipeline bug surfaces as a CUDA error instead of a hung GPU.  Site numbers
 * are unique in the library and name the kernel and the wait.  Copies up to 16 words; word 0 == 0 means no timeout
 * was recorded.  Readable even after the context died.
 */
PCV_API int pcv_debug_read(uint32_t* out, int32_t n);
/* Kept for ABI compatibility: the kernels record no clock trace, so this always returns PCV_ERR_UNSUPPORTED. */
PCV_API int pcv_debug_trace_read(uint64_t* out, int32_t n);

/*
 * Host-only developer aid (no CUDA call, usable without a GPU): the stream-K work plan the tcgen05 kernels would
 * use for (B, H, N, M) on `workers` CTAs with `rows_per_unit` query rows per work unit (256: two 128-row tiles
 * per CTA; 128: wide-v / big-head kernels; 512: CTA pairs).  Writes counts = {segments, ctas, partial slots,
 * split units} and, if max_segs is large enough (else PCV_ERR_WORKSPACE with counts filled), one record of
 * 8 ints per segment: {cta, b, h, q0, active query tiles, first key tile, end key tile, slot (-1 = whole key
 * range, writes the final output)}.  Key tiles are 128 keys.
 */
PCV_API int pcv_debug_plan(int32_t B, int32_t H, int32_t N, int32_t M, int32_t workers, int32_t rows_per_unit,
                           int32_t rows_per_tile, int32_t* segs, int32_t max_segs, int32_t* counts);

/*
 * The current device's CTA-pair plan: *workers CTA pairs, of the *clusters_fit 2-CTA clusters of the pair kernel that
 * can be resident at once (cudaOccupancyMaxActiveClusters).
 */
PCV_API int pcv_debug_pair_workers(int32_t* workers, int32_t* clusters_fit);

/* number of kernel launches issued by this library in the calling process (for bench.py's
 * gpu_launches claim) */
PCV_API uint64_t pcv_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* PCV_ATTN_H_ */
