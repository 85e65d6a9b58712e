// pcv_attn_tc.cu — fused attention forward on the Hopper tensor cores (sm_90a, warpgroup MMA).
//
//   S = Q K^T  (wgmma SS: Q and K boxes in SWIZZLE_128B shared memory, S in registers)
//   P = 2^(S*scale*log2e - m)   (online softmax in registers, rows shared by the four lanes of a quad)
//   O += P V   (wgmma RS: P re-used in place as the 16-bit A fragment, V box read MN-major, O in registers)
//
// CTA = one 128-row query tile of one (batch, head) x a contiguous range of 128-key tiles; 384 threads:
// warpgroup 0 is the TMA producer (one lane), warpgroups 1 and 2 each own 64 query rows.  For head dims up to 128 a
// consumer warpgroup overlaps the P V of tile t - 1 with the softmax of tile t, and the two consumer warpgroups take
// turns at issuing their GEMMs, so the tensor cores work while the softmax runs (see kPipelined in attn_fwd_kernel).
// CTA-pair variant (PAIR, impl = PCV_IMPL_TCGEN05_PAIR): a 2-CTA cluster takes two adjacent query tiles of the same
// (b, h) and key range; each CTA loads one 64-key half of every K / V box and multicasts it to both, so the pair
// reads each key tile from L2 once.  A ring slot is refilled only after the consumers of BOTH CTAs released it.  Q stays in shared
// memory for the segment; K and V arrive as 128-key x 64-channel boxes through one ring of 16 KB slots guarded
// by full / empty mbarriers, so every head dim (up to 512 for Q/K) uses the same pipeline: at head dims up to 128 one
// pair per tile's K boxes and one per its V boxes, each released by one arrive per consumer warpgroup (and CTA of
// a pair), so a tile costs two waits and two releases.  V is processed in
// passes of at most 128 channels (one launch per pass) to keep the accumulators in registers.
//
// Work distribution is a host-built segment table (stream-K over the key axis): segments that cover a
// whole (b,h,query tile) write the final output; split ones write (numerator, max, denominator) slots that
// tc_combine_kernel merges.  Semantics are those of include/pcv_attn.h (finite mask fill, uniform rows).
#include "pcv_common.cuh"
#include "pcv_dropout.cuh"
#include "pcv_sm90.cuh"

#include <cstdlib>
#include <algorithm>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <tuple>
#include <vector>

namespace pcv {
namespace {

using namespace sm90;

constexpr int kTileM = 128;              // query rows per CTA tile (two warpgroups of 64)
constexpr int kTileN = 128;              // keys per tile
constexpr int kBoxBytes = kTileN * 128;  // one TMA box: 128 rows x 64 16-bit channels, SWIZZLE_128B
constexpr int kThreads = 384;            // producer warpgroup + 2 consumer warpgroups
constexpr int kMaxDvPass = 128;          // V channels per launch (O accumulators stay in registers)
constexpr int kSmemLimit = 227 * 1024;

struct Segment {
  int b, h;
  int q0;      // first query row of the tile
  int ntile;   // 128-row query tiles of the unit that hold rows < N (plan bookkeeping)
  int t0, t1;  // key tiles [t0, t1)
  int slot;    // >= 0: partial slot index; -1: the segment covers every key tile (final)
  int unit;    // >= 0: index of the split unit (UnitRec) this segment is a part of (host plan checks); -1: whole key range
};

struct UnitRec {  // a (b,h,query tile) whose key range was split over several segments
  int b, h, q0;
  int slot_begin, slot_count;
  int pad_[3];
};

// M-sharded launch with the cross-GPU merge fused into the kernel tail (pcv_attn_fwd_sharded): after its segments
// every CTA turns into a merge worker.  All pointers of index g are rank g's symmetric-memory buffers as mapped
// into THIS process (index `rank` is the local one).  Flag words per rank: [0, G) "partial state of rank i is
// complete" (written by rank i), [G, 2G) "rank i has pushed all its output rows" (written by rank i), [16, 19)
// grid-wide arrival counters of the local kernel.  All flags / counters are monotonic in the call epoch.
struct PeerTail {
  int enabled;
  int num_peers, rank;
  uint32_t epoch;
  const float* part_o[PCV_MAX_PEERS];
  const float* part_m[PCV_MAX_PEERS];
  const float* part_l[PCV_MAX_PEERS];
  void* out[PCV_MAX_PEERS];
  uint32_t* flags[PCV_MAX_PEERS];
  int64_t osb, osn, osh;
  int64_t row_begin, row_end;  // rows of the flattened (b, h, n) space this rank merges
};

struct TcParams {
  const Segment* segs;
  const int* cta_seg_begin;
  int B, H, N, M, dv;
  int dv_off, dv_pass;       // this launch writes output channels [dv_off, dv_off + dv_pass)
  float scale_log2;
  int causal, causal_shift;  // key j (local) masked for query n iff j > n + causal_shift
  const uint32_t* pad_bits;  // (B, pad_wpr) bit set = padding key; nullptr if no mask
  int pad_wpr;
  int q_bcast;
  void* out;
  int64_t osb, osn, osh;
  int write_partial;
  float *fin_o, *fin_m, *fin_l;     // caller's partial state (B,H,N,dv),(B,H,N),(B,H,N)
  float *slot_o, *slot_m, *slot_l;  // workspace slots [slot][slot_rows][DV], [slot][slot_rows]
  int rows_per_unit;
  int slot_rows;
  PeerTail tail;
  DropoutRule drop;  // attn_fwd_drop_kernel only; last, so that the other kernels' parameter offsets do not move
  int drop_key_base; // attn_fwd_drop_kernel: global index of local key 0 (m_offset, even); the mask hashes it + j
  // attn_fwd_fp8_kernel only (appended, as the dropout fields): per-head q / k and per-(head, channel) v descales
  const float *q_descale, *k_descale, *v_descale;
  int v_descale_stride;  // floats between heads of v_descale (the full dv)
};

// --------------------------------------------------------------------------------------------------
// M-sharded merge across GPUs (pcv_attn_fwd_sharded), run in stream order right after the attention kernel of the
// call: publish "partial state complete" to every rank, wait for all ranks, merge the owned rows of the flattened
// (b, h, n) space from every rank's state over peer memory and store the normalised rows into EVERY rank's output,
// then a grid-wide arrival and a second flag exchange so that the call returns when this rank's output is complete.
// No NCCL and no host barrier on the path.  Flag words per rank: [0, G) partial state of rank i complete, [G, 2G)
// rank i has pushed all its rows, [18] grid arrival counter, [24, 30) phase clock of CTA 0; all monotonic in the
// call epoch.  The grid-wide arrival needs every CTA co-resident: the grid is at most one CTA per SM.
// --------------------------------------------------------------------------------------------------
constexpr int kTailThreads = 256;

__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ float ld_relaxed_sys_f32(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_relaxed_sys_f32x4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void tail_wait_ge(const uint32_t* flag, uint32_t value, uint32_t site) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while ((int32_t)(ld_acquire_sys_u32(flag) - value) < 0) {
    if ((++spins & 0xFFu) == 0) {
      const uint64_t now = globaltimer_ns();
      if (t0 == 0) {
        t0 = now;
      } else if (now - t0 > kWaitTimeoutNs) {
        uint32_t* d = g_wait_diag;
        if (d != nullptr && atomicCAS(d, 0u, 1u) == 0u) {
          d[1] = site;
          d[2] = blockIdx.x;
          d[3] = threadIdx.x;
          d[4] = value;
          d[5] = ld_acquire_sys_u32(flag);
          __threadfence_system();
        }
        __trap();
      }
    }
  }
}

// all kTailThreads threads of every CTA call this; `counter` is a device-local word, monotonic over calls
__device__ __forceinline__ void tail_grid_arrive_wait(uint32_t* counter, uint32_t target, uint32_t site) {
  __threadfence_system();  // this thread's partial-state / output stores are visible system-wide before the arrival
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(counter, 1u);
    tail_wait_ge(counter, target, site);
  }
  __syncthreads();
}

template <bool BF16>
__global__ void __launch_bounds__(kTailThreads) peer_tail_kernel(const TcParams p) {
  const PeerTail& t = p.tail;
  const int G = t.num_peers;
  uint32_t* lf = t.flags[t.rank];
  const uint32_t target = t.epoch * gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kWarps = kTailThreads / 32;
  // phase clock of CTA 0 (ns since tail entry) in flag words [24, 30): cheap, always on, read by tools/dist_check.py
  const uint64_t t_in = globaltimer_ns();
#define PCV_TAIL_STAMP(i)                                                                      \
  do {                                                                                         \
    if (blockIdx.x == 0 && threadIdx.x == 0) lf[24 + (i)] = (uint32_t)(globaltimer_ns() - t_in); \
  } while (0)

  // the attention (and combine) kernels of this call ran before in stream order: the local partial state is complete
  PCV_TAIL_STAMP(0);
  PCV_TAIL_STAMP(1);

  // publish: flags[g][rank] = epoch on every rank g
  if (blockIdx.x == 0 && threadIdx.x < G) {
    __threadfence_system();
    st_release_sys_u32(t.flags[threadIdx.x] + t.rank, t.epoch);
  }
  if (threadIdx.x < G) tail_wait_ge(lf + threadIdx.x, t.epoch, 41);
  __syncthreads();
  PCV_TAIL_STAMP(2);

  // owned rows: pull, merge, push.  A warp keeps PCV_MAX_PEERS (row, rank) sources in flight at once — with 2 ranks
  // that is 4 rows per iteration — so that every lane always has 8 x 16 bytes of (mostly remote) loads outstanding;
  // with one row per warp iteration the phase is bound by the NVLink round trip, not by bandwidth.
  const int RB = PCV_MAX_PEERS / G;  // rows per warp iteration
  const int64_t nblk = (t.row_end - t.row_begin + RB - 1) / RB;
  for (int64_t blk = (int64_t)blockIdx.x * kWarps + warp; blk < nblk; blk += (int64_t)gridDim.x * kWarps) {
    const int64_t r0 = t.row_begin + blk * RB;
    for (int c = lane * 4; c < p.dv; c += 128) {
      float mg[PCV_MAX_PEERS], lg[PCV_MAX_PEERS];
      float4 x[PCV_MAX_PEERS];
#pragma unroll
      for (int j = 0; j < PCV_MAX_PEERS; ++j) {
        const int rr = j / G, g = j - rr * G;   // source j = row r0 + rr of rank g
        const int64_t r = r0 + rr;
        const bool live = rr < RB && r < t.row_end;
        mg[j] = -INFINITY;
        lg[j] = 0.f;
        x[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live) {
          mg[j] = ld_relaxed_sys_f32(t.part_m[g] + r);
          lg[j] = ld_relaxed_sys_f32(t.part_l[g] + r);
          x[j] = ld_relaxed_sys_f32x4(t.part_o[g] + r * p.dv + c);
        }
      }
      for (int rr = 0; rr < RB; ++rr) {
        const int64_t r = r0 + rr;
        if (r >= t.row_end) break;
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < PCV_MAX_PEERS; ++j)
          if (j / G == rr) m = fmaxf(m, mg[j]);
        float l = 0.f;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < PCV_MAX_PEERS; ++j) {
          if (j / G != rr) continue;
          const float w = (mg[j] != -INFINITY) ? exp2f(mg[j] - m) : 0.f;
          l = fmaf(lg[j], w, l);
          acc.x = fmaf(x[j].x, w, acc.x);
          acc.y = fmaf(x[j].y, w, acc.y);
          acc.z = fmaf(x[j].z, w, acc.z);
          acc.w = fmaf(x[j].w, w, acc.w);
        }
        const float inv = 1.f / l;
        uint2 packed;
        packed.x = pack2(acc.x * inv, acc.y * inv, BF16);
        packed.y = pack2(acc.z * inv, acc.w * inv, BF16);
        const int n = (int)(r % p.N);
        const int h = (int)((r / p.N) % p.H);
        const int b = (int)(r / ((int64_t)p.N * p.H));
        const int64_t o_off = (int64_t)b * t.osb + (int64_t)n * t.osn + (int64_t)h * t.osh;
#pragma unroll
        for (int g = 0; g < PCV_MAX_PEERS; ++g)
          if (g < G) *reinterpret_cast<uint2*>(reinterpret_cast<char*>(t.out[g]) + 2 * (o_off + c)) = packed;
      }
    }
  }

  PCV_TAIL_STAMP(3);
  tail_grid_arrive_wait(lf + 18, target, 42);
  PCV_TAIL_STAMP(4);
  if (blockIdx.x == 0) {
    if (threadIdx.x < G) {
      st_release_sys_u32(t.flags[threadIdx.x] + G + t.rank, t.epoch);
      tail_wait_ge(lf + G + threadIdx.x, t.epoch, 43);
    }
    __syncthreads();
  }
  PCV_TAIL_STAMP(5);
#undef PCV_TAIL_STAMP
}

// The pipelined schedule (NQB <= 2) uses a multiple of NQB + NVB ring slots: every key tile then starts at a ring
// index that is a multiple of NQB + NVB, so the V boxes of a tile are adjacent slots that never wrap and one
// m64n128 wgmma reads both (issue_pv).
template <int NQB, int NVB>
struct FwdCfg {
  static constexpr int kQBytes = NQB * kBoxBytes;
  static constexpr int kFit = (kSmemLimit - kQBytes - 2048) / kBoxBytes > 16 ? 16 : (kSmemLimit - kQBytes - 2048) / kBoxBytes;
  static constexpr int kSlots = NQB <= 2 ? kFit / (NQB + NVB) * (NQB + NVB) : kFit;
  static constexpr int kSmemBytes = kQBytes + kSlots * kBoxBytes + 2048;  // + barriers + 1024-byte alignment slack
  static_assert(kSlots >= 2, "shared memory budget");
};

// Position of a key tile in the pipelined schedule's ring: the slot of its first K box and the parity of that slot's
// current fill.  Tiles start at multiples of STEP (the K and V boxes of a tile), which divides NS, so the tile's V
// group (slot + NQB) has the same parity and one compare wraps the position: no division by the ring size, which is
// not a power of two.
template <int STEP, int NS>
struct RingPos {
  uint32_t slot = 0, phase = 0;
  __device__ __forceinline__ void advance() {
    slot += STEP;
    if (slot == NS) {
      slot = 0;
      phase ^= 1;
    }
  }
};

struct FwdBarriers {
  uint64_t full[16], empty[16];
  uint64_t q_full, q_empty;
};

// Scores of one 128-key tile (this thread's 64 accumulator registers) -> unnormalised probabilities in place: scale to
// the log2 domain, apply the masks, update the running row maxima and denominators.  alpha is the factor by which the
// running numerator has to be rescaled before this tile's P V is added.  `interior` (uniform over the warpgroup): no
// key of the tile is masked for any row of the warpgroup, so the per-element checks and pad-word loads are skipped.
// DROP: after the denominators took the tile's probabilities, the dropped elements of the numerator are zeroed (the
// statistics stay those of the dropout-free softmax; the survivors are scaled once, in the epilogue).  `qside` is the
// query side of the mask hash of rows n0 and n0 + 8; each thread hashes once per row and key pair (jb, jb + 1).
// FP8: the scores are scaled by `fp8_scale_log2` (p.scale_log2 * q_descale[h] * k_descale[h]) instead of p.scale_log2.
// The scale c is folded into the exponent, 2^(s c - m) with the raw score s, and the row maximum is taken on the raw
// scores: c > 0 (attn_tc_supported) and rounding is monotonic, so the raw maximum times c is exactly the maximum of the
// scaled scores.  Where a thread holds a padded or causally masked score of a row in the tile, it writes that row's
// scores scaled and masked (the finite fill kMaskedScore) and takes 2^(x - m) instead.  Which formula a score gets
// depends on the masked set alone, so an all-false pad mask gives the unmasked result bit for bit.
template <bool DROP, bool FP8 = false>
__device__ __forceinline__ void tile_softmax(float (&s)[64], float (&m_run)[2], float (&l_run)[2], float (&alpha)[2],
                                             const TcParams& p, int b, int j0, int n0, int cq, bool interior,
                                             const uint32_t (&qside)[2], float fp8_scale_log2 = 0.f) {
  const float c = FP8 ? fp8_scale_log2 : p.scale_log2;
  float mx[2] = {-INFINITY, -INFINITY};
  bool filled[2] = {false, false};  // this thread holds a padded or causally masked score of row r
  if (interior) {
    // four independent chains per row: one chain of 32 dependent FMNMX would put its latency on the critical path
    float m4[2][4] = {{-INFINITY, -INFINITY, -INFINITY, -INFINITY}, {-INFINITY, -INFINITY, -INFINITY, -INFINITY}};
#pragma unroll
    for (int i = 0; i < 64; ++i) m4[(i >> 1) & 1][((i >> 2) & 1) * 2 + (i & 1)] = fmaxf(m4[(i >> 1) & 1][((i >> 2) & 1) * 2 + (i & 1)], s[i]);
#pragma unroll
    for (int r = 0; r < 2; ++r) mx[r] = fmaxf(fmaxf(m4[r][0], m4[r][1]), fmaxf(m4[r][2], m4[r][3]));
  } else {
    // element e of the 8-key group g: 0 live, 1 padded or causally masked, 2 past M
    auto pad_word = [&](int g) { return p.pad_bits != nullptr ? p.pad_bits[(int64_t)b * p.pad_wpr + ((j0 + 8 * g + cq) >> 5)] : 0u; };
    auto kind = [&](int g, int e, uint32_t padw) {
      const int j = j0 + 8 * g + cq + (e & 1);
      if (j >= p.M) return 2;
      return (((padw >> (j & 31)) & 1u) || (p.causal && j > n0 + 8 * (e >> 1) + p.causal_shift)) ? 1 : 0;
    };
#pragma unroll
    for (int g = 0; g < 16; ++g) {
      const uint32_t padw = pad_word(g);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kd = kind(g, e, padw);
        if (kd == 0) mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * g + e]);
        else if (kd == 2) s[4 * g + e] = -INFINITY;
        else filled[e >> 1] = true;
      }
    }
    if (filled[0] || filled[1]) {
#pragma unroll
      for (int g = 0; g < 16; ++g) {
        const uint32_t padw = pad_word(g);
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (filled[e >> 1]) {
            const int kd = kind(g, e, padw);
            if (kd == 0) s[4 * g + e] *= c;
            else if (kd == 1) s[4 * g + e] = kMaskedScore;
          }
      }
    }
  }
  float mref[2], cr[2];  // the exponent of score s of row r is s * cr[r] - mref[r]
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] *= c;
    if (filled[r]) mx[r] = fmaxf(mx[r], kMaskedScore);
    cr[r] = filled[r] ? 1.f : c;
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float mn = fmaxf(m_run[r], mx[r]);
    alpha[r] = (mn == -INFINITY) ? 1.f : ex2(m_run[r] - mn);
    mref[r] = (mn == -INFINITY) ? 0.f : mn;
    m_run[r] = mn;
    l_run[r] *= alpha[r];
  }
  float lsum[2][2] = {{0.f, 0.f}, {0.f, 0.f}};  // two partial row sums: half the dependent FADD chain
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    float e0 = ex2(fmaf(s[4 * g + 0], cr[0], -mref[0])), e1 = ex2(fmaf(s[4 * g + 1], cr[0], -mref[0]));
    float e2 = ex2(fmaf(s[4 * g + 2], cr[1], -mref[1])), e3 = ex2(fmaf(s[4 * g + 3], cr[1], -mref[1]));
    lsum[0][g & 1] += e0 + e1;
    lsum[1][g & 1] += e2 + e3;
    if constexpr (DROP) {
      const uint32_t jb = (uint32_t)(p.drop_key_base + j0 + 8 * g + cq), n = (uint32_t)n0;
      const uint32_t ks = drop_kside(p.drop.seed_hi, jb);
      const uint32_t x0 = drop_finish(qside[0], ks), x1 = drop_finish(qside[1], ks);
      if (!drop_keep(x0, n, jb, p.drop.thresh)) e0 = 0.f;
      if (!drop_keep(x0, n, jb + 1, p.drop.thresh)) e1 = 0.f;
      if (!drop_keep(x1, n + 8, jb, p.drop.thresh)) e2 = 0.f;
      if (!drop_keep(x1, n + 8, jb + 1, p.drop.thresh)) e3 = 0.f;
    }
    s[4 * g + 0] = e0;
    s[4 * g + 1] = e1;
    s[4 * g + 2] = e2;
    s[4 * g + 3] = e3;
  }
  l_run[0] += lsum[0][0] + lsum[0][1];
  l_run[1] += lsum[1][0] + lsum[1][1];
}

// probabilities -> the 16-bit A fragments of the P V wgmma (k-step kk covers keys [16 kk, 16 kk + 16))
template <bool BF16>
__device__ __forceinline__ void pack_p(const float (&s)[64], uint32_t (&pa)[8][4]) {
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    pa[g >> 1][(g & 1) * 2 + 0] = pack2(s[4 * g + 0], s[4 * g + 1], BF16);
    pa[g >> 1][(g & 1) * 2 + 1] = pack2(s[4 * g + 2], s[4 * g + 3], BF16);
  }
}

// probabilities -> the e4m3 A fragments of the FP8 P V wgmma (k-step kk covers keys [32 kk, 32 kk + 32)), each
// rounded as e4m3(P * 2^8).  This thread's scores hold keys 8j + 2q + {0, 1} of rows r and r + 8 (q = lane % 4), the
// fragment wants keys 4q .. 4q + 3 and 16 + 4q .. 16 + 4q + 3 of the same rows, so the four lanes of a quad exchange
// halves: per k-step and row, lane q receives from lanes a = q/2 + 2 (q%2) and a ^ 1 the two-key halves it needs.
// Sources with odd q send their 8 + 2q / 24 + 2q keys first, even ones their 2q / 16 + 2q keys, so that each of the
// two shuffles reads one value per source lane.
__device__ __forceinline__ void pack_p_e4m3(const float (&s)[64], uint32_t (&pa)[4][4], int lane) {
  const int q = lane & 3;
  const uint32_t sel_a = (q & 1) ? 0x7632u : 0x5410u, sel_b = (q & 1) ? 0x5410u : 0x7632u;
  const uint32_t sel_lo = (q & 2) ? 0x1054u : 0x5410u, sel_hi = (q & 2) ? 0x3276u : 0x7632u;
  const int src_a = (lane & ~3) | (q >> 1) | ((q & 1) << 1), src_b = src_a ^ 1;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float* x = s + 16 * kk + 2 * r;  // groups 4kk .. 4kk + 3 (8 keys each), row half r
      const uint32_t x0 = cvt_e4m3x2(x[0] * 256.f, x[1] * 256.f) | (cvt_e4m3x2(x[4] * 256.f, x[5] * 256.f) << 16);
      const uint32_t x1 = cvt_e4m3x2(x[8] * 256.f, x[9] * 256.f) | (cvt_e4m3x2(x[12] * 256.f, x[13] * 256.f) << 16);
      const uint32_t a = __shfl_sync(0xffffffffu, __byte_perm(x0, x1, sel_a), src_a);
      const uint32_t b = __shfl_sync(0xffffffffu, __byte_perm(x0, x1, sel_b), src_b);
      pa[kk][r] = __byte_perm(a, b, sel_lo);
      pa[kk][2 + r] = __byte_perm(a, b, sel_hi);
    }
}

// Skipped when no row of the warp moved its maximum (alpha is exactly 1, and o * 1 is o): after the first few key tiles
// that is the common case.
template <int NVB>
__device__ __forceinline__ void rescale_o(float (&o)[NVB][32], const float (&alpha)[2]) {
  if (__all_sync(0xffffffffu, alpha[0] == 1.f && alpha[1] == 1.f)) return;
#pragma unroll
  for (int v = 0; v < NVB; ++v)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[v][i] *= alpha[(i >> 1) & 1];
}

// The body of attn_fwd_kernel (DROP = false) and of attn_fwd_drop_kernel (DROP = true: attention-probability dropout,
// see tile_softmax; write_partial = 1 without key sharding, no CTA pair), and of attn_fwd_fp8_kernel (FP8 = true:
// e4m3 q / k and V^T, (B, H, dv, keys).  A Q or K box is 128 rows x 128 e4m3 channels; the V^T box of a tile is 128
// channels x 128 keys, one ring slot, with the 64-channel halves v at byte offset 8192 v.  BF16 is the output dtype).
template <int NQB, int NVB, bool BF16, bool PAIR, bool DROP, bool FP8 = false>
__device__ __forceinline__ void attn_fwd_body(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                                              const TcParams& p) {
  static_assert(!(DROP && PAIR), "no dropout in the CTA-pair kernel");
  static_assert(!FP8 || (NQB <= 2 && !PAIR && !DROP), "the FP8 kernel: qk head dims up to 256, no CTA pair, no dropout");
  using C = FwdCfg<NQB, NVB>;
  constexpr int NS = C::kSlots;
  constexpr int KVB = FP8 ? 1 : NVB;  // ring boxes of V per key tile
  constexpr int kQkCh = FP8 ? 128 : 64;  // qk channels per box
  // Head dims up to 128 (NQB <= 2) run the pipelined schedule: per tile one commit group for S = Q K^T and one for
  // O += P V, the P V of tile t - 1 runs under the softmax of tile t, and the two warpgroups take turns at issuing
  // their GEMMs (ping-pong), so that one warpgroup's MMAs run while the other computes its softmax.  It holds the K
  // boxes of tile t and the V boxes of tile t - 1 at once, which larger head dims do not leave ring slots for; they
  // keep the serial schedule (per box: wait, issue, drain, release).
  constexpr bool kPipelined = NQB <= 2;
  static_assert(!kPipelined || NQB + KVB <= NS, "the pipelined schedule holds NQB + KVB ring slots");
  static_assert(!kPipelined || NS % (NQB + KVB) == 0, "a key tile's V boxes must not wrap around the ring");
  // registers per thread: producer + 2 x consumer = 504 = the launch bound's 168 x 3; the pipelined consumers keep
  // S, P and O live at once, the serial schedule's producer (ring index arithmetic by a non-power-of-two) spills at 24
  constexpr int kProducerRegs = kPipelined ? 24 : 40, kConsumerRegs = kPipelined ? 240 : 232;
  static_assert(kProducerRegs + 2 * kConsumerRegs == 504, "register split");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sRing = smem + C::kQBytes;
  FwdBarriers& bar = *reinterpret_cast<FwdBarriers*>(sRing + NS * kBoxBytes);
  const int wg = threadIdx.x / 128;
  const int worker = PAIR ? blockIdx.x / 2 : blockIdx.x;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
  const int qoff = 128 * (int)rank;  // this CTA's query tile within the pair's 256-row unit
  const int seg_lo = p.cta_seg_begin[worker], seg_hi = p.cta_seg_begin[worker + 1];

  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&bar.full[s], 1);
      mbar_init(&bar.empty[s], PAIR ? 4 : 2);  // one arrive per consumer warpgroup (of both CTAs of a pair)
    }
    mbar_init(&bar.q_full, 1);
    mbar_init(&bar.q_empty, 8);
    fence_mbar_init();
  }
  if (PAIR)
    cluster_sync_all();
  else
    __syncthreads();

  if (wg == 0) {
    reg_dealloc<kProducerRegs>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;  // serial schedule: ring index of the next box
      RingPos<NQB + KVB, NS> pos;  // pipelined schedule: the next tile's box groups
      for (int si = seg_lo; si < seg_hi; ++si) {
        const Segment sg = p.segs[si];
        mbar_wait(&bar.q_empty, ((si - seg_lo) & 1) ^ 1, 1);
        mbar_arrive_expect_tx(&bar.q_full, C::kQBytes);
        for (int c = 0; c < NQB; ++c)
          tma_load_4d(sQ + c * kBoxBytes, &tq, &bar.q_full, c * kQkCh, sg.q0 + qoff, sg.h, p.q_bcast ? 0 : sg.b);
        for (int t = sg.t0; t < sg.t1; ++t) {
          // box c of the tile into ring slot s, its bytes counted on full barrier fb
          auto load_box = [&](int c, uint32_t s, uint64_t* fb) {
            uint8_t* dst = sRing + s * kBoxBytes;
            const CUtensorMap* tm = c < NQB ? &tk : &tv;
            const int ch = (c < NQB ? c : c - NQB) * 64;
            if constexpr (FP8) {  // K: (channel box c, keys of tile t); V^T: (keys of tile t, channels of the pass)
              if (c < NQB) tma_load_4d(dst, tm, fb, c * kQkCh, t * kTileN, sg.h, sg.b);
              else tma_load_4d(dst, tm, fb, t * kTileN, 0, sg.h, sg.b);
            } else if (PAIR)  // 64-key half `rank` of the box, into both CTAs
              tma_load_4d_mc(dst + rank * (kBoxBytes / 2), tm, fb, ch, t * kTileN + 64 * (int)rank, sg.h, sg.b, 0x3);
            else
              tma_load_4d(dst, tm, fb, ch, t * kTileN, sg.h, sg.b);
          };
          // nb boxes from ring slot g on, whose fill has parity ph: wait until the slots are free, expect their bytes
          auto begin_group = [&](uint32_t g, uint32_t ph, int nb) {
            mbar_wait(&bar.empty[g], ph ^ 1, 2);
            mbar_arrive_expect_tx(&bar.full[g], nb * kBoxBytes);
          };
          // The pipelined schedule guards the K boxes of a tile with one full / empty pair and its V boxes with
          // another, those of the group's first slot (a tile's boxes never wrap around the ring); the serial schedule
          // every box with its own.
          if constexpr (kPipelined) {
            const uint32_t gk = pos.slot, gv = pos.slot + NQB;
            begin_group(gk, pos.phase, NQB);
#pragma unroll
            for (int c = 0; c < NQB; ++c) load_box(c, gk + c, &bar.full[gk]);
            begin_group(gv, pos.phase, KVB);
#pragma unroll
            for (int c = 0; c < KVB; ++c) load_box(NQB + c, gv + c, &bar.full[gv]);
            pos.advance();
          } else {
#pragma unroll 1
            for (int c = 0; c < NQB + KVB; ++c, ++it) {
              const uint32_t s = it % NS;
              begin_group(s, (it / NS) & 1, 1);
              load_box(c, s, &bar.full[s]);
            }
          }
        }
      }
    }
    if (PAIR) {
      __syncwarp();
      cluster_sync_all();  // the peer may still multicast into / arrive on this CTA's shared memory until here
    }
    return;
  }

  reg_alloc<kConsumerRegs>();
  const int cw = (int)warp_uniform(wg) - 1;  // consumer warpgroup: query rows [64*cw, 64*cw + 64) of the tile
  const int tid = threadIdx.x - 128 * wg;
  const int warp = tid >> 5, lane = tid & 31;
  const int rloc = 64 * cw + 16 * warp + (lane >> 2);  // rows rloc and rloc + 8
  const int cq = 2 * (lane & 3);                      // first of the two columns of every 8-column group
  // wgmma descriptors: a warp-uniform low word set up outside the GEMM turn plus a compile-time byte offset (desc_at),
  // so that each wgmma costs one uniform add.  Q stays at one place for the whole kernel; ring slot g has the low word
  // ring_lo + g * kSlotLo.  On the pipelined schedule the 16-bit P V at NVB == 2 reads both V boxes of a tile
  // (adjacent slots) in one m64n128 wgmma: LBO = one box.
  constexpr uint32_t kSlotLo = kBoxBytes >> 4;
  constexpr uint32_t kPvLbo = (kPipelined && !FP8 && NVB == 2) ? kBoxBytes : 16;
  const uint32_t q_lo = warp_uniform(desc_lo(smem_u32(sQ) + cw * 64 * 128));
  const uint32_t ring_lo = warp_uniform(desc_lo(smem_u32(sRing)));
  const uint32_t ring_lo_v = warp_uniform(desc_lo(smem_u32(sRing), kPvLbo));
  // low word of the K group at ring slot g.  Marked uniform it is built in the uniform datapath; at NVB == 1 the mark
  // makes ptxas spill the segment bounds (8 bytes), so those kernels leave it unmarked.
  auto k_lo = [&](uint32_t g) {
    const uint32_t lo = ring_lo + g * kSlotLo;
    return NVB == 2 ? warp_uniform(lo) : lo;
  };
  RingPos<NQB + KVB, NS> pos;  // pipelined schedule: the next tile's box groups (the producer's order)
  uint32_t it = 0;  // serial schedule: ring index of the next box (the NQB K boxes, then the NVB V boxes of a tile)

  // releases the box group (see the producer) whose first box is ring slot g
  auto release = [&](uint32_t g) {
    if (PAIR) wg_arrive_pair(&bar.empty[g]);
    else wg_arrive(&bar.empty[g]);
  };
  // S (+)= Q box c K^T with the K box at low word kb: four k16 steps of 16-bit channels or k32 steps of e4m3 ones,
  // 32 bytes each.  FP8 issues all four k32 steps of a box even past dqk (TMA zero fill): a runtime guard around the
  // wgmma makes ptxas serialise every wgmma of the kernel (C7515)
  auto qk_box = [&](float (&s)[64], int c, uint32_t kb) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      if constexpr (FP8)
        wgmma_ss_e4m3_n128(s, desc_at(q_lo, c * kBoxBytes + kk * 32), desc_at(kb, kk * 32), (c | kk) != 0);
      else
        wgmma_ss<128, BF16>(s, desc_at(q_lo, c * kBoxBytes + kk * 32), desc_at(kb, kk * 32), (c | kk) != 0);
    }
  };
  // O += P V box at low word vb (16-bit, 64 channels): eight k16 steps of 16 key rows, 2048 bytes each
  auto pv_box = [&](float (&ov)[32], const uint32_t (&pa)[8][4], uint32_t vb) {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_rs<64, BF16>(ov, pa[kk], desc_at(vb, kk * 2048));
  };
  // S = Q K^T of the tile whose K group starts at ring slot g (low word kb), filled with parity ph: one commit group
  auto issue_qk = [&](float (&s)[64], uint32_t g, uint32_t ph, uint32_t kb) {
    mbar_wait(&bar.full[g], ph, 6);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NQB; ++c) qk_box(s, c, kb + c * kSlotLo);
    wgmma_commit();
  };
  // P as the A operand of P V: 16-bit fragments of 8 k16 steps, or e4m3 fragments of 4 k32 steps
  using PFrag = uint32_t[FP8 ? 4 : 8][4];
  // O += P V of the tile whose V group starts at ring slot g (low word vb), filled with parity ph: one commit group
  auto issue_pv = [&](float (&o)[NVB][32], const PFrag& pa, uint32_t g, uint32_t ph, uint32_t vb) {
    mbar_wait(&bar.full[g], ph, 7);
    wgmma_fence();
    if constexpr (FP8) {  // the V^T box of a tile: 64-channel halves 8192 bytes apart, k32 steps of 32 bytes
#pragma unroll
      for (int v = 0; v < NVB; ++v)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_e4m3_n64(o[v], pa[kk], desc_at(vb, v * 8192 + kk * 32));
    } else if constexpr (NVB == 2) {  // both V boxes in one m64n128 per k16 step (adjacent slots, see FwdCfg)
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        wgmma_rs<128, BF16>(reinterpret_cast<float(&)[64]>(o), pa[kk], desc_at(vb, kk * 2048));
    } else {
      pv_box(o[0], pa, vb);
    }
    wgmma_commit();
  };
  auto pack = [&](const float (&s)[64], PFrag& pa) {
    if constexpr (FP8) pack_p_e4m3(s, pa, lane);
    else pack_p<BF16>(s, pa);
  };
  // after the P V whose V group starts at ring slot g completed: O is final in registers, release the V boxes
  auto pv_done = [&](float (&o)[NVB][32], uint32_t g) {
#pragma unroll
    for (int v = 0; v < NVB; ++v) fence_regs(o[v]);
    release(g);
  };
  // Ping-pong turns.  Warpgroup cw waits on its own named barrier (id 1 + cw) before it issues its GEMMs and hands
  // the turn over by arriving on the other's (id 2 - cw) after it committed them; a phase counts 256 threads (128
  // syncing + 128 arriving).  Invariant: both warpgroups run the same segments with the same key tiles (the plan is
  // per CTA, and every segment has at least one tile), so each takes exactly nt + 1 turns per segment of nt tiles.
  // Warpgroup 1 hands warpgroup 0 the first turn and skips the hand-over after its own last turn, so that both
  // barriers see as many arrivals as syncs:  id 1: n syncs (wg 0), 1 + (n - 1) arrivals (wg 1);  id 2: n and n.
  constexpr int kTurnThreads = 256;
  auto turn_begin = [&] {
    if (cw == 0) named_bar_sync<1, kTurnThreads>();
    else named_bar_sync<2, kTurnThreads>();
  };
  auto turn_end = [&](bool last) {
    if (cw == 0) named_bar_arrive<2, kTurnThreads>();
    else if (!last) named_bar_arrive<1, kTurnThreads>();
  };
  if (kPipelined && cw == 1 && seg_lo < seg_hi) named_bar_arrive<1, kTurnThreads>();

  // PAIR: the consumers' closing cluster barrier (the peer may still arrive on this CTA's ring barriers until both
  // CTAs reach it) is issued inside the segment loop, after the last segment: a barrier after the loop makes ptxas
  // budget the whole consumer path at the launch bound (168 registers) and serialise the wgmmas.
  if (PAIR && seg_lo == seg_hi) cluster_sync_all();
  for (int si = seg_lo; si < seg_hi; ++si) {
    const Segment sg = p.segs[si];
    mbar_wait(&bar.q_full, (si - seg_lo) & 1, 3);
    float o[NVB][32];
#pragma unroll
    for (int v = 0; v < NVB; ++v)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[v][i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const int n0 = sg.q0 + qoff + rloc;
    const int n_wg = sg.q0 + qoff + 64 * cw;  // first query row of this warpgroup
    uint32_t qside[2] = {0u, 0u};
    if constexpr (DROP) {
      const uint32_t bh = (uint32_t)(sg.b * p.H + sg.h);
#pragma unroll
      for (int r = 0; r < 2; ++r) qside[r] = drop_qside(p.drop.seed_lo, drop_qword(bh, (uint32_t)(n0 + 8 * r)));
    }
    // no key of the tile starting at j0 is masked for any row of this warpgroup
    auto interior = [&](int j0) {
      return p.pad_bits == nullptr && j0 + kTileN <= p.M && (!p.causal || j0 + kTileN - 1 <= n_wg + p.causal_shift);
    };

    // FP8: q_descale * k_descale of the head factors out of every score of the segment
    float sl2 = 0.f;
    if constexpr (FP8) sl2 = p.scale_log2 * p.q_descale[sg.h] * p.k_descale[sg.h];
    if constexpr (kPipelined) {
      float s[64], alpha[2];
      PFrag pa;
      if (sg.t1 > sg.t0) {
        // prologue: S of the first tile, its softmax (O is still zero: nothing to rescale)
        uint32_t kb = k_lo(pos.slot);
        turn_begin();
        issue_qk(s, pos.slot, pos.phase, kb);
        turn_end(false);
        wgmma_wait<0>();
        fence_regs(s);
        release(pos.slot);
        tile_softmax<DROP, FP8>(s, m_run, l_run, alpha, p, sg.b, sg.t0 * kTileN, n0, cq, interior(sg.t0 * kTileN), qside,
                                sl2);
        pack(s, pa);
        for (int t = sg.t0 + 1; t < sg.t1; ++t) {
          const uint32_t gv = pos.slot + NQB, vph = pos.phase;  // V boxes of tile t - 1
          const uint32_t vb = ring_lo_v + gv * kSlotLo;
          pos.advance();
          kb = k_lo(pos.slot);
          turn_begin();
          issue_qk(s, pos.slot, pos.phase, kb);
          issue_pv(o, pa, gv, vph, vb);
          turn_end(false);
          wgmma_wait<1>();  // S of tile t is ready; P V of tile t - 1 still runs under the softmax below
          fence_regs(s);
          release(pos.slot);
          tile_softmax<DROP, FP8>(s, m_run, l_run, alpha, p, sg.b, t * kTileN, n0, cq, interior(t * kTileN), qside, sl2);
          wgmma_wait<0>();
          pv_done(o, gv);
          rescale_o(o, alpha);
          pack(s, pa);
        }
        // epilogue: P V of the last tile
        const uint32_t gv = pos.slot + NQB;
        const uint32_t vb = ring_lo_v + gv * kSlotLo;
        turn_begin();
        issue_pv(o, pa, gv, pos.phase, vb);
        turn_end(si + 1 == seg_hi);  // the last turn of this CTA
        wgmma_wait<0>();
        pv_done(o, gv);
        pos.advance();
      }
    } else {
      for (int t = sg.t0; t < sg.t1; ++t) {
        float s[64];
#pragma unroll
        for (int c = 0; c < NQB; ++c, ++it) {
          const uint32_t sl = it % NS;
          mbar_wait(&bar.full[sl], (it / NS) & 1, 4);
          wgmma_fence();
          qk_box(s, c, ring_lo + sl * kSlotLo);
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(s);
          release(sl);
        }
        float alpha[2];
        tile_softmax<DROP>(s, m_run, l_run, alpha, p, sg.b, t * kTileN, n0, cq, interior(t * kTileN), qside);
        rescale_o(o, alpha);
        uint32_t pa[8][4];
        pack_p<BF16>(s, pa);
#pragma unroll
        for (int v = 0; v < NVB; ++v, ++it) {
          const uint32_t sl = it % NS;
          mbar_wait(&bar.full[sl], (it / NS) & 1, 5);
          wgmma_fence();
          pv_box(o[v], pa, ring_lo + sl * kSlotLo);
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(o[v]);
          release(sl);
        }
      }
    }
    warp_arrive(&bar.q_empty);  // every wgmma reading Q of this segment has completed

    // epilogue: quad-reduce the denominators, write final rows / caller's partial state / split slots
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    if constexpr (DROP) {  // the survivors' scale, once for every store below (tc_combine_kernel is linear in o)
#pragma unroll
      for (int v = 0; v < NVB; ++v)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[v][i] *= p.drop.scale;
    }
    if constexpr (FP8) {  // P was scaled by 2^8 before rounding; v_descale of the channel, once for every store below
      const float* vd = p.v_descale + (int64_t)sg.h * p.v_descale_stride + p.dv_off;
#pragma unroll
      for (int v = 0; v < NVB; ++v)
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const int c = v * 64 + 8 * g + cq;  // dv_pass is a multiple of 16: c and c + 1 are both in or both out
          const float d0 = c < p.dv_pass ? vd[c] * (1.f / 256.f) : 0.f;
          const float d1 = c < p.dv_pass ? vd[c + 1] * (1.f / 256.f) : 0.f;
          o[v][4 * g + 0] *= d0;
          o[v][4 * g + 1] *= d1;
          o[v][4 * g + 2] *= d0;
          o[v][4 * g + 3] *= d1;
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int rr = qoff + rloc + 8 * r;  // row within the unit (slot row)
      const int n = sg.q0 + rr;
      if (n >= p.N) continue;
      if (sg.slot >= 0) {
        const int64_t row = (int64_t)sg.slot * p.slot_rows + rr;
        float* dst = p.slot_o + row * (NVB * 64);
#pragma unroll
        for (int v = 0; v < NVB; ++v)
#pragma unroll
          for (int g = 0; g < 8; ++g)
            *reinterpret_cast<float2*>(dst + v * 64 + 8 * g + cq) = make_float2(o[v][4 * g + 2 * r], o[v][4 * g + 2 * r + 1]);
        if ((lane & 3) == 0) {
          p.slot_m[row] = m_run[r];
          p.slot_l[row] = l_run[r];
        }
      } else if (p.write_partial) {
        const int64_t row = ((int64_t)sg.b * p.H + sg.h) * p.N + n;
        float* dst = p.fin_o + row * p.dv + p.dv_off;
#pragma unroll
        for (int v = 0; v < NVB; ++v)
#pragma unroll
          for (int g = 0; g < 8; ++g) {
            const int c = v * 64 + 8 * g + cq;
            if (c < p.dv_pass) *reinterpret_cast<float2*>(dst + c) = make_float2(o[v][4 * g + 2 * r], o[v][4 * g + 2 * r + 1]);
          }
        if ((lane & 3) == 0) {
          p.fin_m[row] = m_run[r];
          p.fin_l[row] = l_run[r];
        }
      } else {
        const float inv = 1.f / l_run[r];
        char* orow = reinterpret_cast<char*>(p.out) +
                     2 * ((int64_t)sg.b * p.osb + (int64_t)n * p.osn + (int64_t)sg.h * p.osh + p.dv_off);
#pragma unroll
        for (int v = 0; v < NVB; ++v)
#pragma unroll
          for (int g = 0; g < 8; ++g) {
            const int c = v * 64 + 8 * g + cq;
            if (c < p.dv_pass)
              *reinterpret_cast<uint32_t*>(orow + 2 * c) = pack2(o[v][4 * g + 2 * r] * inv, o[v][4 * g + 2 * r + 1] * inv, BF16);
          }
      }
    }
    if (PAIR && si + 1 == seg_hi) cluster_sync_all();
  }
}

template <int NQB, int NVB, bool BF16, bool PAIR>
__global__ void __launch_bounds__(kThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                const __grid_constant__ CUtensorMap tv, const TcParams p) {
  attn_fwd_body<NQB, NVB, BF16, PAIR, false>(tq, tk, tv, p);
}

// One-pass forward with attention-probability dropout (pcv_attn_fwd_partial_dropout): a separate kernel, so that the
// inference kernel's code is unchanged.
template <int NQB, int NVB, bool BF16>
__global__ void __launch_bounds__(kThreads, 1)
attn_fwd_drop_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                     const __grid_constant__ CUtensorMap tv, const TcParams p) {
  attn_fwd_body<NQB, NVB, BF16, false, true>(tq, tk, tv, p);
}

// FP8 inference forward (pcv_attn_fwd_fp8): e4m3 Q / K and V^T, output / partial state as attn_fwd_kernel's; a
// separate kernel, so that the 16-bit kernels' code is unchanged.
template <int NQB, int NVB, bool BF16>
__global__ void __launch_bounds__(kThreads, 1)
attn_fwd_fp8_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                    const __grid_constant__ CUtensorMap tv, const TcParams p) {
  attn_fwd_body<NQB, NVB, BF16, false, false, true>(tq, tk, tv, p);
}

// --------------------------------------------------------------------------------------------------
// merge of split units (one warp per query row)
// --------------------------------------------------------------------------------------------------
template <int DV, bool BF16>
__global__ void __launch_bounds__(256) tc_combine_kernel(const UnitRec* __restrict__ units, const TcParams p) {
  const UnitRec u = units[blockIdx.x];
  const int row = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int n = u.q0 + row;
  if (n >= p.N || row >= p.rows_per_unit) return;
  float m = -INFINITY;
  for (int s = 0; s < u.slot_count; ++s) m = fmaxf(m, p.slot_m[(int64_t)(u.slot_begin + s) * p.slot_rows + row]);
  float l = 0.f;
  for (int s = 0; s < u.slot_count; ++s) {
    const int64_t r = (int64_t)(u.slot_begin + s) * p.slot_rows + row;
    l += p.slot_l[r] * exp2f(p.slot_m[r] - m);
  }
  for (int c = lane * 4; c < DV; c += 128) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < u.slot_count; ++s) {
      const int64_t r = (int64_t)(u.slot_begin + s) * p.slot_rows + row;
      const float w = exp2f(p.slot_m[r] - m);
      const float4 x = *reinterpret_cast<const float4*>(p.slot_o + r * DV + c);
      acc.x = fmaf(x.x, w, acc.x);
      acc.y = fmaf(x.y, w, acc.y);
      acc.z = fmaf(x.z, w, acc.z);
      acc.w = fmaf(x.w, w, acc.w);
    }
    if (c >= p.dv_pass) continue;
    if (!p.write_partial) {
      const float inv = 1.f / l;
      uint2 w2;
      w2.x = pack2(acc.x * inv, acc.y * inv, BF16);
      w2.y = pack2(acc.z * inv, acc.w * inv, BF16);
      char* orow = reinterpret_cast<char*>(p.out) + 2 * ((int64_t)u.b * p.osb + (int64_t)n * p.osn + (int64_t)u.h * p.osh);
      *reinterpret_cast<uint2*>(orow + 2 * (p.dv_off + c)) = w2;
    } else {
      const int64_t r = ((int64_t)u.b * p.H + u.h) * p.N + n;
      *reinterpret_cast<float4*>(p.fin_o + r * p.dv + p.dv_off + c) = acc;
    }
  }
  if (p.write_partial && lane == 0) {
    const int64_t r = ((int64_t)u.b * p.H + u.h) * p.N + n;
    p.fin_m[r] = m;
    p.fin_l[r] = l;
  }
}

// --------------------------------------------------------------------------------------------------
// host: plan (segment table), tensor maps, launch
// --------------------------------------------------------------------------------------------------
struct Plan {
  int num_ctas = 0, num_slots = 0, num_units = 0;
  std::vector<Segment> segs;
  std::vector<int> cta_seg_begin;
  std::vector<UnitRec> units;
  Segment* d_segs = nullptr;
  int* d_cta = nullptr;
  UnitRec* d_units = nullptr;
  int dev = 0;
  uint64_t seq = 0;  // last use (LRU eviction)
};

void build_plan(Plan& pl, int B, int H, int N, int M, int num_sms, int rows_per_unit, int rows_per_tile) {
  // num_sms = number of workers (CTAs)
  const int QB = (N + rows_per_unit - 1) / rows_per_unit;
  const int T = (M + kTileN - 1) / kTileN;
  const int BH = B * H;
  auto ntile_of = [&](int qb) { return (rows_per_unit > rows_per_tile && (N - qb * rows_per_unit) > rows_per_tile) ? 2 : 1; };
  std::vector<std::vector<Segment>> per_cta;
  const bool split_mode = QB * 2 <= num_sms;  // groups of QB workers share their K/V stream; else whole units per worker
  if (split_mode) {
    // groups of QB CTAs walk the flattened (b*h, key tile) space together, one query block each, so that
    // the members of a group stream the same K/V tiles at the same time (they meet in L2)
    int ngroups = num_sms / QB;
    const int64_t W = (int64_t)BH * T;
    if (ngroups > W) ngroups = (int)W;
    per_cta.resize((size_t)ngroups * QB);
    std::map<std::pair<int, int>, std::vector<int>> unit_slots;  // (bh, qb) -> slots
    for (int g = 0; g < ngroups; ++g) {
      int64_t pos = W * g / ngroups;
      const int64_t end = W * (g + 1) / ngroups;
      while (pos < end) {
        const int bh = (int)(pos / T), t0 = (int)(pos % T);
        const int t1 = (int)std::min<int64_t>(T, t0 + (end - pos));
        for (int r = 0; r < QB; ++r) {
          Segment s{};
          s.b = bh / H; s.h = bh % H; s.q0 = r * rows_per_unit; s.ntile = ntile_of(r); s.t0 = t0; s.t1 = t1;
          s.unit = -1;
          if (t0 == 0 && t1 == T) {
            s.slot = -1;
          } else {
            s.slot = pl.num_slots++;
            unit_slots[{bh, r}].push_back(s.slot);
          }
          per_cta[(size_t)g * QB + r].push_back(s);
        }
        pos += t1 - t0;
      }
    }
    // slots of one unit must be contiguous for the combine kernel: renumber
    std::map<int, int> remap, unit_of;
    int next = 0;
    for (auto& kv : unit_slots) {
      UnitRec u{};
      u.b = kv.first.first / H; u.h = kv.first.first % H; u.q0 = kv.first.second * rows_per_unit;
      u.slot_begin = next; u.slot_count = (int)kv.second.size();
      for (int old : kv.second) {
        unit_of[old] = (int)pl.units.size();
        remap[old] = next++;
      }
      pl.units.push_back(u);
    }
    for (auto& v : per_cta)
      for (auto& s : v)
        if (s.slot >= 0) {
          s.unit = unit_of[s.slot];
          s.slot = remap[s.slot];
        }
  } else {
    // many query blocks: whole (b,h,query-block) units, contiguous chunks per CTA, no splitting
    const int64_t U = (int64_t)BH * QB;
    const int nctas = (int)std::min<int64_t>(num_sms, U);
    per_cta.resize(nctas);
    for (int c = 0; c < nctas; ++c) {
      for (int64_t u = U * c / nctas; u < U * (c + 1) / nctas; ++u) {
        const int bh = (int)(u / QB), qb = (int)(u % QB);
        Segment s{};
        s.b = bh / H; s.h = bh % H; s.q0 = qb * rows_per_unit; s.ntile = ntile_of(qb); s.t0 = 0; s.t1 = T; s.slot = -1;
        s.unit = -1;
        per_cta[c].push_back(s);
      }
    }
  }
  pl.num_ctas = (int)per_cta.size();
  pl.cta_seg_begin.assign(1, 0);
  for (auto& v : per_cta) {
    for (auto& s : v) pl.segs.push_back(s);
    pl.cta_seg_begin.push_back((int)pl.segs.size());
  }
  pl.num_units = (int)pl.units.size();
}

std::mutex g_plan_mu;
// The plan depends on (N, M) only through the number of query blocks, whether the last block holds one or two
// query tiles, and the number of 128-key tiles, so the cache is keyed on those: a decode loop whose key count
// grows by one per step hits the cache for 128 consecutive steps (no cudaMalloc / blocking copy on the step path).
using PlanKey = std::tuple<int, int, int, int, int, int, int, int, int>;  // device, B, H, QB, last ntile, T, workers, rows/unit, rows/tile
std::map<PlanKey, std::shared_ptr<Plan>> g_plans;
uint64_t g_plan_seq = 0;
constexpr size_t kMaxPlans = 256;


struct Mode {
  int rows_per_unit, rows_per_tile, slot_rows;
  bool pair;  // 2-CTA clusters: workers are CTA pairs, 256 query rows per unit
};

void free_plan_tables(Plan& pl) {
  // a kernel in flight on ANY stream of the plan's device may still read the tables
  int cur = 0;
  cudaGetDevice(&cur);
  if (cur != pl.dev) cudaSetDevice(pl.dev);
  cudaDeviceSynchronize();
  cudaFree(pl.d_segs);
  cudaFree(pl.d_cta);
  cudaFree(pl.d_units);
  pl.d_segs = nullptr;
  pl.d_cta = nullptr;
  pl.d_units = nullptr;
  if (cur != pl.dev) cudaSetDevice(cur);
}

// Workers of the CTA-pair plan: SMs / 2, capped at the 2-CTA clusters of the pair kernel that can be resident at
// once.  Both CTAs of a cluster must sit in one GPC, so a GPC with an odd number of SMs leaves one of them idle; a pair
// past that cap would start only when another has finished all its work, doubling the kernel time.  Every pair
// instantiation takes one CTA per SM (more than half the shared memory), so one of them stands for all.
int pair_workers(int dev, int* workers, int* fit_out = nullptr) {
  static std::mutex mu;
  static std::map<int, std::pair<int, int>> cache;  // device -> (workers, clusters that fit)
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(dev);
  if (it != cache.end()) {
    *workers = it->second.first;
    if (fit_out != nullptr) *fit_out = it->second.second;
    return PCV_OK;
  }
  int sms = 0;
  PCV_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  auto kernel = attn_fwd_kernel<2, 2, true, true>;
  constexpr int smem = FwdCfg<2, 2>::kSmemBytes;
  const int rc = set_smem_limit(reinterpret_cast<const void*>(kernel), smem);
  if (rc != PCV_OK) return rc;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(sms / 2 * 2);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int fit = 0;
  PCV_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&fit, kernel, &cfg));
  PCV_REQUIRE(fit >= 1, PCV_ERR_UNSUPPORTED, "the CTA-pair kernel: no 2-CTA cluster fits on device %d", dev);
  *workers = std::min(sms / 2, fit);
  if (fit_out != nullptr) *fit_out = fit;
  cache[dev] = {*workers, fit};
  return PCV_OK;
}

// The returned shared_ptr keeps the host-side plan alive for the caller even if another thread evicts it; the
// device tables of an evicted plan are released only after a synchronize of their device, and eviction removes
// the least recently used half (never the entry being returned).
int get_plan(int B, int H, int N, int M, const Mode& mode, std::shared_ptr<Plan>* out) {
  int dev = 0;
  PCV_CHECK_CUDA(cudaGetDevice(&dev));
  int sms = 0;
  if (mode.pair) {
    const int rc = pair_workers(dev, &sms);  // workers are CTA pairs
    if (rc != PCV_OK) return rc;
  } else {
    PCV_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  std::lock_guard<std::mutex> lk(g_plan_mu);
  const int QB = (N + mode.rows_per_unit - 1) / mode.rows_per_unit;
  const int T = (M + kTileN - 1) / kTileN;
  const int last_ntile =
      (mode.rows_per_unit > mode.rows_per_tile && (N - (QB - 1) * mode.rows_per_unit) > mode.rows_per_tile) ? 2 : 1;
  const PlanKey key = std::make_tuple(dev, B, H, QB, last_ntile, T, sms, mode.rows_per_unit, mode.rows_per_tile);
  auto it = g_plans.find(key);
  if (it != g_plans.end()) {
    it->second->seq = ++g_plan_seq;
    *out = it->second;
    return PCV_OK;
  }
  auto pl = std::make_shared<Plan>();
  pl->dev = dev;
  pl->seq = ++g_plan_seq;
  build_plan(*pl, B, H, N, M, sms, mode.rows_per_unit, mode.rows_per_tile);
  PCV_CHECK_CUDA(cudaMalloc(&pl->d_segs, sizeof(Segment) * pl->segs.size()));
  PCV_CHECK_CUDA(cudaMalloc(&pl->d_cta, sizeof(int) * pl->cta_seg_begin.size()));
  PCV_CHECK_CUDA(cudaMemcpy(pl->d_segs, pl->segs.data(), sizeof(Segment) * pl->segs.size(), cudaMemcpyHostToDevice));
  PCV_CHECK_CUDA(cudaMemcpy(pl->d_cta, pl->cta_seg_begin.data(), sizeof(int) * pl->cta_seg_begin.size(),
                            cudaMemcpyHostToDevice));
  if (!pl->units.empty()) {
    PCV_CHECK_CUDA(cudaMalloc(&pl->d_units, sizeof(UnitRec) * pl->units.size()));
    PCV_CHECK_CUDA(cudaMemcpy(pl->d_units, pl->units.data(), sizeof(UnitRec) * pl->units.size(), cudaMemcpyHostToDevice));
  }
  if (g_plans.size() >= kMaxPlans) {
    std::vector<uint64_t> seqs;
    for (auto& kv : g_plans) seqs.push_back(kv.second->seq);
    std::nth_element(seqs.begin(), seqs.begin() + seqs.size() / 2, seqs.end());
    const uint64_t cut = seqs[seqs.size() / 2];
    for (auto jt = g_plans.begin(); jt != g_plans.end();) {
      if (jt->second->seq < cut) {
        free_plan_tables(*jt->second);
        jt = g_plans.erase(jt);
      } else {
        ++jt;
      }
    }
  }
  g_plans[key] = pl;
  *out = pl;
  return PCV_OK;
}

inline int pad64(int d) { return (d + 63) / 64 * 64; }

size_t slots_bytes(const Plan& pl, int DV, int slot_rows) {
  // [slot][row][DV] numerators, [slot][row] row max, [slot][row] denominators
  return sizeof(float) * (size_t)pl.num_slots * slot_rows * (DV + 2);
}
// The CTA-pair kernel takes a call only when it is asked for (impl = PCV_IMPL_TCGEN05_PAIR): at head dim 128 it is
// slower than the single-CTA kernel at every N measured (README).
Mode choose_mode(const pcv_attn_params& a) {
  if (a.impl == PCV_IMPL_TCGEN05_PAIR) return Mode{2 * kTileM, kTileM, 2 * kTileM, true};
  return Mode{kTileM, kTileM, kTileM, false};
}

int dv_pass_width(int dv) { return std::min(kMaxDvPass, pad64(dv)); }

template <int NQB, int NVB, bool BF16, bool PAIR, bool DROP, bool FP8 = false>
int launch_fwd(const Plan& pl, const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const TcParams& p,
               cudaStream_t stream) {
  prof_mark_begin(stream);
  // num_ctas counts CTA pairs in the pair mode
  int rc;
  if constexpr (FP8)
    rc = launch_kernel(attn_fwd_fp8_kernel<NQB, NVB, BF16>, dim3(pl.num_ctas), kThreads, FwdCfg<NQB, NVB>::kSmemBytes, 0,
                       stream, tq, tk, tv, p);
  else if constexpr (DROP)
    rc = launch_kernel(attn_fwd_drop_kernel<NQB, NVB, BF16>, dim3(pl.num_ctas), kThreads, FwdCfg<NQB, NVB>::kSmemBytes, 0,
                       stream, tq, tk, tv, p);
  else
    rc = launch_kernel(attn_fwd_kernel<NQB, NVB, BF16, PAIR>, dim3(PAIR ? 2 * pl.num_ctas : pl.num_ctas), kThreads,
                       FwdCfg<NQB, NVB>::kSmemBytes, PAIR ? 2 : 0, stream, tq, tk, tv, p);
  prof_mark_end(stream);
  if (rc != PCV_OK) return rc;
  if (pl.num_units > 0) {
    dim3 grid(pl.num_units, p.slot_rows / 8);
    if (NVB == 1)
      tc_combine_kernel<64, BF16><<<grid, 256, 0, stream>>>(pl.d_units, p);
    else
      tc_combine_kernel<128, BF16><<<grid, 256, 0, stream>>>(pl.d_units, p);
    PCV_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  return PCV_OK;
}

template <int NQB, bool BF16, bool DROP>
int launch_nqb(int nvb, bool pair, const Plan& pl, const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
               const TcParams& p, cudaStream_t stream) {
  if constexpr (NQB <= 2 && !DROP) {
    if (pair)
      return nvb == 1 ? launch_fwd<NQB, 1, BF16, true, false>(pl, tq, tk, tv, p, stream)
                      : launch_fwd<NQB, 2, BF16, true, false>(pl, tq, tk, tv, p, stream);
  }
  return nvb == 1 ? launch_fwd<NQB, 1, BF16, false, DROP>(pl, tq, tk, tv, p, stream)
                  : launch_fwd<NQB, 2, BF16, false, DROP>(pl, tq, tk, tv, p, stream);
}

template <bool BF16, bool DROP>
int launch_dispatch(int nqb, int nvb, bool pair, const Plan& pl, const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                    const TcParams& p, cudaStream_t stream) {
  switch (nqb) {
    case 1: return launch_nqb<1, BF16, DROP>(nvb, pair, pl, tq, tk, tv, p, stream);
    case 2: return launch_nqb<2, BF16, DROP>(nvb, pair, pl, tq, tk, tv, p, stream);
    case 3: return launch_nqb<3, BF16, DROP>(nvb, pair, pl, tq, tk, tv, p, stream);
    case 4: return launch_nqb<4, BF16, DROP>(nvb, pair, pl, tq, tk, tv, p, stream);
    case 5: return launch_nqb<5, BF16, DROP>(nvb, pair, pl, tq, tk, tv, p, stream);
    case 6: return launch_nqb<6, BF16, DROP>(nvb, pair, pl, tq, tk, tv, p, stream);
    case 7: return launch_nqb<7, BF16, DROP>(nvb, pair, pl, tq, tk, tv, p, stream);
    case 8: return launch_nqb<8, BF16, DROP>(nvb, pair, pl, tq, tk, tv, p, stream);
  }
  set_error("tensor-core attention: qk head dim needs %d 64-channel boxes (at most 8)", nqb);
  return PCV_ERR_UNSUPPORTED;
}

template <bool BF16>
int launch_dispatch_fp8(int nqb, int nvb, const Plan& pl, const CUtensorMap& tq, const CUtensorMap& tk,
                        const CUtensorMap& tv, const TcParams& p, cudaStream_t stream) {
  if (nqb == 1)
    return nvb == 1 ? launch_fwd<1, 1, BF16, false, false, true>(pl, tq, tk, tv, p, stream)
                    : launch_fwd<1, 2, BF16, false, false, true>(pl, tq, tk, tv, p, stream);
  return nvb == 1 ? launch_fwd<2, 1, BF16, false, false, true>(pl, tq, tk, tv, p, stream)
                  : launch_fwd<2, 2, BF16, false, false, true>(pl, tq, tk, tv, p, stream);
}

// The checks attn_tc_supported and attn_tc_fp8_supported end with: the output, the sequence lengths and the device
// (an FP8 call has passed dv % 16 == 0 before, so the dv % 4 of the partial state never refuses it).
bool tc_output_supported(const pcv_attn_params& p, const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (!p.write_partial) {
    if (!al16(p.out) || (p.o_stride_n % 8) || (p.o_stride_h % 8) || (p.o_stride_b % 8))
      return fail("output must be 16-byte aligned with strides in multiples of 8 elements");
  } else {
    if (!al16(p.part_o) || (p.dv % 4)) return fail("partial output alignment");
  }
  if ((int64_t)p.N > (1 << 24) || (int64_t)p.M > (1 << 30)) return fail("sequence too long");
  if (const char* w = device_problem()) return fail(w);
  return true;
}

// What the 16-bit and the FP8 launches share, after their own checks: the plan and the workspace checks (error
// messages prefixed with `what`), the TcParams core, the workspace slots, the packed pad mask and the Q / K tensor maps
// (K boxes of `k_box_rows` keys).  The caller adds its own fields to `p` and launches one pass per V slice.
int tc_setup(const pcv_attn_params& a, const Mode& mode, const char* what, int k_box_rows, cudaStream_t stream,
             std::shared_ptr<Plan>* plan, TcParams* tp, CUtensorMap* tq, CUtensorMap* tk) {
  int rc = attach_wait_diag(&g_wait_diag);
  if (rc != PCV_OK) return rc;
  rc = get_plan(a.B, a.H, a.N, a.M, mode, plan);
  if (rc != PCV_OK) return rc;
  const Plan& pl = **plan;
  size_t need = 0;
  rc = attn_tc_workspace_bytes(a, &need);
  if (rc != PCV_OK) return rc;
  PCV_REQUIRE(need == 0 || (a.workspace != nullptr && a.workspace_bytes >= need), PCV_ERR_WORKSPACE,
              "%s: workspace of %zu bytes required, %zu given", what, need, a.workspace_bytes);
  PCV_REQUIRE(need == 0 || (reinterpret_cast<uintptr_t>(a.workspace) & 15) == 0, PCV_ERR_WORKSPACE,
              "%s: workspace must be 16-byte aligned", what);

  TcParams& p = *tp;
  p = TcParams{};
  p.segs = pl.d_segs;
  p.cta_seg_begin = pl.d_cta;
  p.B = a.B; p.H = a.H; p.N = a.N; p.M = a.M; p.dv = a.dv;
  p.scale_log2 = a.scale * kLog2e;
  p.causal = a.causal;
  p.causal_shift = (a.m_total - a.N) - a.m_offset;
  p.q_bcast = (a.q_stride_b == 0) ? 1 : 0;
  p.out = a.out; p.osb = a.o_stride_b; p.osn = a.o_stride_n; p.osh = a.o_stride_h;
  p.write_partial = a.write_partial;
  p.rows_per_unit = mode.rows_per_unit;
  p.slot_rows = mode.slot_rows;
  p.fin_o = a.part_o; p.fin_m = a.part_m; p.fin_l = a.part_l;
  const int slot_dv = dv_pass_width(a.dv);
  char* ws = reinterpret_cast<char*>(a.workspace);
  const size_t nrows = (size_t)pl.num_slots * mode.slot_rows;
  p.slot_o = reinterpret_cast<float*>(ws);
  p.slot_m = p.slot_o + nrows * slot_dv;
  p.slot_l = p.slot_m + nrows;
  if (a.pad_mask != nullptr) {
    size_t off = (slots_bytes(pl, slot_dv, mode.slot_rows) + 255) / 256 * 256;
    uint32_t* bits = reinterpret_cast<uint32_t*>(ws + off);
    p.pad_bits = bits;
    p.pad_wpr = pad_words_per_row(a.M);
    rc = launch_pack_pad(a.pad_mask, a.pad_stride_b, a.B, a.M, bits, stream);
    if (rc != PCV_OK) return rc;
  }

  const int Bq = a.q_stride_b == 0 ? 1 : a.B;
  rc = make_tmap_4d(tq, a.q, a.dtype, a.dqk, a.N, a.H, Bq, a.q_stride_n, a.q_stride_h, a.q_stride_b, kTileM);
  if (rc != PCV_OK) return rc;
  return make_tmap_4d(tk, a.k, a.dtype, a.dqk, a.M, a.H, a.B, a.k_stride_m, a.k_stride_h, a.k_stride_b, k_box_rows);
}

}  // namespace

// Host-only (no CUDA call): the work plan of the tensor-core kernel for a problem, one record of 8 ints per segment
// {cta, b, h, q0, ntile, t0, t1, slot}; tests/test_plan_cpu.py checks its invariants on the CPU.
int debug_plan(int B, int H, int N, int M, int workers, int rows_per_unit, int rows_per_tile, int32_t* segs,
               int max_segs, int32_t* counts) {
  Plan pl;
  build_plan(pl, B, H, N, M, workers, rows_per_unit, rows_per_tile);
  counts[0] = (int32_t)pl.segs.size();
  counts[1] = pl.num_ctas;
  counts[2] = pl.num_slots;
  counts[3] = pl.num_units;
  if ((int)pl.segs.size() > max_segs) return PCV_ERR_WORKSPACE;
  for (int c = 0; c < pl.num_ctas; ++c)
    for (int s = pl.cta_seg_begin[c]; s < pl.cta_seg_begin[c + 1]; ++s) {
      const Segment& g = pl.segs[s];
      int32_t* r = segs + 8 * s;
      r[0] = c; r[1] = g.b; r[2] = g.h; r[3] = g.q0; r[4] = g.ntile; r[5] = g.t0; r[6] = g.t1; r[7] = g.slot;
    }
  return PCV_OK;
}

int debug_pair_workers(int32_t* workers, int32_t* clusters_fit) {
  int dev = 0, w = 0, fit = 0;
  PCV_CHECK_CUDA(cudaGetDevice(&dev));
  const int rc = pair_workers(dev, &w, &fit);
  if (rc != PCV_OK) return rc;
  *workers = w;
  *clusters_fit = fit;
  return PCV_OK;
}

bool attn_tc_supported(const pcv_attn_params& p, const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (p.dqk > 512) return fail("qk head dim > 512");
  if (p.dv > 512) return fail("v head dim > 512");
  if ((p.dqk % 8) || (p.dv % 8)) return fail("head dims must be multiples of 8 (16-byte TMA strides)");
  if (!(p.scale > 0.f)) return fail("scale must be positive");
  if (!al16(p.q) || !al16(p.k) || !al16(p.v)) return fail("q/k/v base pointers must be 16-byte aligned");
  if ((p.q_stride_n % 8) || (p.k_stride_m % 8) || (p.v_stride_m % 8) || (p.q_stride_h % 8) || (p.k_stride_h % 8) ||
      (p.v_stride_h % 8) || (p.q_stride_b % 8) || (p.k_stride_b % 8) || (p.v_stride_b % 8))
    return fail("q/k/v strides must be multiples of 8 elements");
  return tc_output_supported(p, why);
}

int attn_tc_workspace_bytes(const pcv_attn_params& p, size_t* bytes) {
  std::shared_ptr<Plan> pl;
  const Mode mode = choose_mode(p);
  int rc = get_plan(p.B, p.H, p.N, p.M, mode, &pl);
  if (rc != PCV_OK) return rc;
  size_t b = slots_bytes(*pl, dv_pass_width(p.dv), mode.slot_rows);
  b = (b + 255) / 256 * 256;
  if (p.pad_mask != nullptr) b += sizeof(uint32_t) * (size_t)p.B * pad_words_per_row(p.M);
  *bytes = b;
  return PCV_OK;
}

bool attn_tc_fuse_supported(const pcv_attn_params& a, const char** why) {
  if (!attn_tc_supported(a, why)) return false;
  if (a.dv % 4) {
    *why = "fused merge needs v head dim % 4 == 0";
    return false;
  }
  return true;
}

int launch_attn_tc(const pcv_attn_params& a, cudaStream_t stream, const pcv_shard_fuse* fuse, const DropoutRule* drop) {
  {
    const char* why = "";
    PCV_REQUIRE(attn_tc_supported(a, &why), PCV_ERR_UNSUPPORTED, "tensor-core attention: %s", why);
  }
  PCV_REQUIRE(drop == nullptr || (fuse == nullptr && a.write_partial && a.impl != PCV_IMPL_TCGEN05_PAIR &&
                                  a.m_offset % 2 == 0 && drop->thresh > 0),
              PCV_ERR_UNSUPPORTED,
              "tensor-core attention: dropout needs a partial-state call starting at an even key, no CTA pair");
  if (fuse != nullptr) {
    const char* why = "";
    PCV_REQUIRE(attn_tc_fuse_supported(a, &why), PCV_ERR_UNSUPPORTED, "fused merge: %s", why);
    PCV_REQUIRE(a.write_partial, PCV_ERR_INVALID, "fused merge: the launch must write the partial state (write_partial = 1)");
  }
  const Mode mode = choose_mode(a);
  if (mode.pair) {
    int dev = 0, sms = 0;
    PCV_CHECK_CUDA(cudaGetDevice(&dev));
    PCV_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PCV_REQUIRE(pad64(a.dqk) <= 128 && pad64(a.dv) <= 128 && sms >= 2, PCV_ERR_UNSUPPORTED,
                "the CTA-pair kernel needs qk and v head dims <= 128 and at least two SMs");
  }
  std::shared_ptr<Plan> pl;
  TcParams p;
  CUtensorMap tq, tk, tv;
  const int kv_box_rows = mode.pair ? kTileN / 2 : kTileN;  // a pair loads 64-key halves of every K / V tile
  int rc = tc_setup(a, mode, "tensor-core attention", kv_box_rows, stream, &pl, &p, &tq, &tk);
  if (rc != PCV_OK) return rc;
  if (drop != nullptr) {
    p.drop = *drop;
    p.drop_key_base = a.m_offset;
  }
  if (fuse != nullptr) {
    PeerTail& t = p.tail;
    t.enabled = 1;
    t.num_peers = fuse->num_peers;
    t.rank = fuse->rank;
    t.epoch = fuse->epoch;
    const int64_t R = (int64_t)a.B * a.H * a.N;
    for (int g = 0; g < fuse->num_peers; ++g) {
      const float* base = reinterpret_cast<const float*>(fuse->part[g]);
      t.part_o[g] = base;
      t.part_m[g] = base + R * a.dv;
      t.part_l[g] = base + R * a.dv + R;
      t.out[g] = fuse->out[g];
      t.flags[g] = fuse->flags[g];
    }
    t.osb = fuse->o_stride_b; t.osn = fuse->o_stride_n; t.osh = fuse->o_stride_h;
    t.row_begin = R * fuse->rank / fuse->num_peers;
    t.row_end = R * (fuse->rank + 1) / fuse->num_peers;
    // the local partial state IS this rank's symmetric buffer
    p.fin_o = const_cast<float*>(t.part_o[fuse->rank]);
    p.fin_m = const_cast<float*>(t.part_m[fuse->rank]);
    p.fin_l = const_cast<float*>(t.part_l[fuse->rank]);
  }
  const bool bf = a.dtype == PCV_BF16;
  const int nqb = pad64(a.dqk) / 64;
  // one launch per slice of at most 128 V channels (the scores are recomputed per slice)
  for (int off = 0; off < a.dv; off += kMaxDvPass) {
    p.dv_off = off;
    p.dv_pass = std::min(kMaxDvPass, a.dv - off);
    const int nvb = (p.dv_pass + 63) / 64;
    const char* vbase = reinterpret_cast<const char*>(a.v) + 2 * (size_t)off;
    rc = make_tmap_4d(&tv, vbase, a.dtype, p.dv_pass, a.M, a.H, a.B, a.v_stride_m, a.v_stride_h, a.v_stride_b, kv_box_rows);
    if (rc != PCV_OK) return rc;
    if (drop != nullptr)
      rc = bf ? launch_dispatch<true, true>(nqb, nvb, false, *pl, tq, tk, tv, p, stream)
              : launch_dispatch<false, true>(nqb, nvb, false, *pl, tq, tk, tv, p, stream);
    else
      rc = bf ? launch_dispatch<true, false>(nqb, nvb, mode.pair, *pl, tq, tk, tv, p, stream)
              : launch_dispatch<false, false>(nqb, nvb, mode.pair, *pl, tq, tk, tv, p, stream);
    if (rc != PCV_OK) return rc;
  }
  if (p.tail.enabled) {
    int dev = 0, sms = 0;
    PCV_CHECK_CUDA(cudaGetDevice(&dev));
    PCV_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (bf)
      peer_tail_kernel<true><<<sms, kTailThreads, 0, stream>>>(p);
    else
      peer_tail_kernel<false><<<sms, kTailThreads, 0, stream>>>(p);
    PCV_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  return PCV_OK;
}

// Host-only (no CUDA call except the device check at the end).
bool attn_tc_fp8_supported(const pcv_attn_params& p, const pcv_fp8_attn& f, const char** why) {
  auto fail = [&](const char* w) {
    *why = w;
    return false;
  };
  if (p.dtype != PCV_E4M3) return fail("q / k / v^T must be e4m3 (dtype PCV_E4M3)");
  if (f.out_dtype != PCV_BF16 && f.out_dtype != PCV_F16) return fail("out_dtype must be bf16 or fp16");
  if (p.impl != PCV_IMPL_AUTO && p.impl != PCV_IMPL_TCGEN05)
    return fail("FP8 runs on the single-CTA tensor-core kernel only (no CTA pair, SIMT or decode kernel)");
  if (p.dqk > 256) return fail("qk head dim > 256");
  if (p.dv > 512) return fail("v head dim > 512");
  if ((p.dqk % 16) || (p.dv % 16)) return fail("head dims must be multiples of 16");
  if (!(p.scale > 0.f)) return fail("scale must be positive");
  if (f.q_descale == nullptr || f.k_descale == nullptr || f.v_descale == nullptr) return fail("a descale pointer is NULL");
  if (!al16(p.q) || !al16(p.k) || !al16(p.v)) return fail("q / k / v^T base pointers must be 16-byte aligned");
  if ((p.q_stride_n % 16) || (p.k_stride_m % 16) || (p.q_stride_h % 16) || (p.k_stride_h % 16) || (p.q_stride_b % 16) ||
      (p.k_stride_b % 16) || (f.vt_stride_b % 16) || (f.vt_stride_h % 16) || (f.vt_stride_c % 16))
    return fail("q / k / v^T strides must be multiples of 16 elements");
  if (f.vt_stride_c < p.M) return fail("v^T channel stride must cover the M keys");
  if (p.B > 1 && (p.k_stride_b == 0 || f.vt_stride_b == 0))
    return fail("k and v^T need a non-zero batch stride when B > 1 (only q broadcasts over the batch)");
  return tc_output_supported(p, why);
}

int launch_attn_tc_fp8(const pcv_attn_params& a, const pcv_fp8_attn& f, cudaStream_t stream) {
  {
    const char* why = "";
    PCV_REQUIRE(attn_tc_fp8_supported(a, f, &why), PCV_ERR_UNSUPPORTED, "FP8 tensor-core attention: %s", why);
  }
  // a.dtype is PCV_E4M3 (checked above): the Q / K boxes hold 128 e4m3 channels
  std::shared_ptr<Plan> pl;
  TcParams p;
  CUtensorMap tq, tk, tv;
  int rc = tc_setup(a, choose_mode(a), "FP8 tensor-core attention", kTileN, stream, &pl, &p, &tq, &tk);
  if (rc != PCV_OK) return rc;
  p.q_descale = f.q_descale; p.k_descale = f.k_descale; p.v_descale = f.v_descale;
  p.v_descale_stride = a.dv;
  const bool bf = f.out_dtype == PCV_BF16;
  const int nqb = (a.dqk + 127) / 128;
  // one launch per slice of at most 128 V channels; V^T is viewed as (keys M, channels of the slice, H, B), so keys
  // past M and channels past the slice read as zero
  for (int off = 0; off < a.dv; off += kMaxDvPass) {
    p.dv_off = off;
    p.dv_pass = std::min(kMaxDvPass, a.dv - off);
    const int nvb = (p.dv_pass + 63) / 64;
    const char* vbase = reinterpret_cast<const char*>(a.v) + (size_t)off * f.vt_stride_c;
    rc = make_tmap_4d(&tv, vbase, PCV_E4M3, a.M, p.dv_pass, a.H, a.B, f.vt_stride_c, f.vt_stride_h, f.vt_stride_b, kMaxDvPass);
    if (rc != PCV_OK) return rc;
    rc = bf ? launch_dispatch_fp8<true>(nqb, nvb, *pl, tq, tk, tv, p, stream)
            : launch_dispatch_fp8<false>(nqb, nvb, *pl, tq, tk, tv, p, stream);
    if (rc != PCV_OK) return rc;
  }
  return PCV_OK;
}

}  // namespace pcv
