// Tensor-core kernels of the path (Hopper wgmma tf32, fp32 accumulators in registers):
//
//  * K2 / K6  dist_tc_kernel: query x centroid (coarse quantiser, gamma_index_ivfflat.cc:568 /
//    gamma_index_ivfpq.cc:595) and point x centroid (k-means assign, faiss Clustering via
//    gamma_index_ivfflat.cc:407 / gamma_index_ivfpq.cc:372).  faiss itself evaluates this
//    contraction as sgemm + norms (IndexFlat, >= 20 queries).
//  * K2 fused  coarse_topk_kernel: the coarse quantiser's top-nprobe without a score matrix (TMA-fed, the
//    same MMAs as dist_tc_kernel, per-query key sets kept by selection warpgroups beside the MMA warpgroup).
//  * K3 list-major: when many queries of a batch probe the same list the IVF-Flat scan
//    (gamma_index_ivfflat.cc:579-787) IS a dense contraction.  The (query, probe) pairs are grouped by
//    list on the device (lm_count / lmk_scan / lmk_assign / lmk_items); a work item multiplies a group
//    of <= 128 pairs by the 128-row tiles of a row segment of the list, so the list is read once per
//    128 queries instead of once per query, and tombstones / bitmaps / score window / top-k are
//    applied as scan_codes does (gamma_index_ivfflat.h:63-91).  Three kernels, one algorithm:
//      ivf_listmajor_tma_kernel   operands arrive by cp.async.bulk from the pre-tiled mirror (k <= 32, d > 16)
//      ivf_listmajor_pipe_kernel  warp-specialised, operands staged through registers (no mirror, d <= 16 or k <= 64)
//      ivf_listmajor_tc_kernel + seg_select_kernel   dense scores + segment select (k > 64)
//
// Precision: every operand is split x = hi + lo, hi = the TF32-representable head (low 13 mantissa
// bits cleared), and three MMAs accumulate hi*hi + hi*lo + lo*hi in fp32 (error-compensated
// "3xTF32", relative error ~2^-21).  Integer-valued operands below 2^11 have lo == 0 and every
// product and partial sum is exact, so on the SIFT-shaped parity data scores are bit-equal to the
// exact fp32 kernels.  L2 uses |x|^2 + |y|^2 - 2 x.y with both norms accumulated in-kernel from the
// staged operands (faiss clamps the expanded form at 0; so do we).  The K3 kernels stage x - s_l and y - s_l
// under L2, s_l the shift of the probed list (launch_list_shifts), so that rounding scales with the residuals.
//
// Operand layout: canonical no-swizzle K-major tiles (8-row x 16-byte core matrices; LBO = stride
// between the two K core matrices of one MMA, SBO = stride between 8-row groups).  One warpgroup
// (warps 0-3) issues the MMAs of a 128 x 128 tile as two m64n128k8 halves and owns the accumulator;
// thread t of it is pair / row t of the tile, and receives its accumulator row through the slab
// exchange of tc_common.cuh.  Register-staged kernels: global loads -> hi/lo split -> st.shared,
// fence.proxy.async, barrier, wgmma; thread t stages row t of both operands, so it also owns |x_t|^2
// and |y_t|^2.  TMA kernel: the same tiles already exist in global memory (tc_mirror_build_kernel,
// lm_stage_queries_kernel) and arrive as 16 KiB bulk copies.
#include <float.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"

namespace gb {

namespace {

constexpr int TC_M = 128, TC_N = 128, TC_BK = 16, TC_NT = 128, TC_STAGES = 2;
constexpr int TC_TILE_BYTES = TC_M * TC_BK * 4;          // 8 KiB per operand part (hi or lo) per stage
constexpr int TC_STAGE_BYTES = 4 * TC_TILE_BYTES;        // a_hi, a_lo, b_hi, b_lo
constexpr int TC_SMEM = TC_STAGES * TC_STAGE_BYTES;      // 64 KiB
static_assert(kSlabBytes <= TC_SMEM / 2, "the accumulator slabs reuse the first operand stage");
static_assert(TC_M * 16 == 2048, "lt_desc assumes LBO = 2048");

__device__ __forceinline__ float4 f4_sub(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }

// The 3xTF32 MMAs of one K = 16 chunk whose four 128 x 16 tiles sit at a_hi, a_lo, b_hi, b_lo.
// Issued by every thread of warpgroup 0; the caller fences before and commits after.
__device__ __forceinline__ void tc_chunk_mma(float (&acc)[2][64], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                             uint32_t b_lo, bool first) {
#pragma unroll
  for (int ks = 0; ks < TC_BK / 8; ks++) {  // one MMA consumes K = 8 (two 4-wide core matrices)
    const uint64_t koff = (uint64_t)((ks * 2 * TC_M * 16) >> 4);
    const uint64_t dbh = lt_desc(b_hi) + koff, dbl = lt_desc(b_lo) + koff;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const uint64_t dah = lt_desc(a_hi) + koff + h * kDescHalfM, dal = lt_desc(a_lo) + koff + h * kDescHalfM;
      wg_mma_tf32(acc[h], dah, dbh, (first && ks == 0) ? 0u : 1u);
      wg_mma_tf32(acc[h], dah, dbl, 1u);
      wg_mma_tf32(acc[h], dal, dbh, 1u);
    }
  }
}

// One 128 x 128 tile: D[i][j] = <A_i, B_j> over d columns.  arow / brow: row pointers of THIS
// thread's row of A and B (nullptr => all zeros).  On return the accumulator sits in `acc` (wgmma
// fragments), thread t holds |A_t|^2 in *an and sh->cn[t] = |B_t|^2, and the operand stages are
// free.  Caller: one warpgroup of 128 threads, TC_SMEM bytes of dynamic smem at `smem`.
//
// Pipeline: two smem stages of K = 16.  While the tensor core works on stage s (asynchronously,
// one wgmma commit group per chunk) the threads already hold the NEXT chunks in registers (global
// loads issued two chunks ahead) and write them into the other stage, so neither the global-load
// latency nor the MMA latency sits on the critical path.
struct TcShared {
  alignas(16) float cn[TC_N];  // |y|^2 of the tile's rows (aligned: the epilogues' reads vectorise)
};

// shift: nullptr, or a row subtracted from both operands' rows before the split (the list shift of K3; see
// tc_split_row)
__device__ __forceinline__ void tc_tile_run(unsigned char* smem, TcShared* sh, const float* __restrict__ arow,
                                            const float* __restrict__ brow, const float* __restrict__ shift, int d,
                                            float (&acc)[2][64], float* an) {
  const int tid = threadIdx.x;
  // canonical layout: element (r, k) of a 128 x 16 tile lives at (k/4)*(128*16) + (r/8)*128 + (r%8)*16 + (k%4)*4
  const uint32_t LBO = TC_M * 16, SBO = 128;
  const uint32_t row_off = (uint32_t)(tid >> 3) * SBO + (uint32_t)(tid & 7) * 16;
  constexpr int NV = TC_BK / 4;  // float4 per operand row per chunk

  float an_acc = 0.f, bn_acc = 0.f;
  const int nk = (d + TC_BK - 1) / TC_BK;
  float4 pa0[NV], pb0[NV], pa1[NV], pb1[NV];
  auto prefetch = [&](int kc, float4 (&pa)[NV], float4 (&pb)[NV]) {
#pragma unroll
    for (int kb = 0; kb < NV; kb++) {
      const int gk = kc * TC_BK + kb * 4;
      pa[kb] = make_float4(0.f, 0.f, 0.f, 0.f);
      pb[kb] = pa[kb];
      if (arow && gk < d) pa[kb] = __ldg(reinterpret_cast<const float4*>(arow + gk));
      if (brow && gk < d) pb[kb] = __ldg(reinterpret_cast<const float4*>(brow + gk));
      if (shift && gk < d) {
        const float4 s4 = __ldg(reinterpret_cast<const float4*>(shift + gk));
        if (arow) pa[kb] = f4_sub(pa[kb], s4);
        if (brow) pb[kb] = f4_sub(pb[kb], s4);
      }
    }
  };
  auto chunk = [&](int kc, float4 (&pa)[NV], float4 (&pb)[NV]) {
    const int s = kc & 1;
    unsigned char* a_hi = smem + (size_t)s * TC_STAGE_BYTES;
    unsigned char* a_lo = a_hi + TC_TILE_BYTES;
    unsigned char* b_hi = a_hi + 2 * TC_TILE_BYTES;
    unsigned char* b_lo = a_hi + 3 * TC_TILE_BYTES;
    if (kc >= TC_STAGES) {  // the MMAs of chunk kc-2 read this stage: done in every warp
      wg_wait<1>();
      __syncthreads();
    }
#pragma unroll
    for (int kb = 0; kb < NV; kb++) {
      const uint32_t off = (uint32_t)kb * LBO + row_off;  // consecutive threads -> consecutive rows: conflict-free
      const float4 va = pa[kb], vb = pb[kb];
      an_acc = fmaf(va.x, va.x, an_acc), an_acc = fmaf(va.y, va.y, an_acc);
      an_acc = fmaf(va.z, va.z, an_acc), an_acc = fmaf(va.w, va.w, an_acc);
      bn_acc = fmaf(vb.x, vb.x, bn_acc), bn_acc = fmaf(vb.y, vb.y, bn_acc);
      bn_acc = fmaf(vb.z, vb.z, bn_acc), bn_acc = fmaf(vb.w, vb.w, bn_acc);
      auto split = [](float v, float& hi, float& lo) {
        hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
        lo = v - hi;
      };
      float4 ah, al, bh, bl;
      split(va.x, ah.x, al.x), split(va.y, ah.y, al.y), split(va.z, ah.z, al.z), split(va.w, ah.w, al.w);
      split(vb.x, bh.x, bl.x), split(vb.y, bh.y, bl.y), split(vb.z, bh.z, bl.z), split(vb.w, bh.w, bl.w);
      *reinterpret_cast<float4*>(a_hi + off) = ah;
      *reinterpret_cast<float4*>(a_lo + off) = al;
      *reinterpret_cast<float4*>(b_hi + off) = bh;
      *reinterpret_cast<float4*>(b_lo + off) = bl;
    }
    if (kc + 2 < nk) prefetch(kc + 2, pa, pb);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> async (tensor) proxy
    __syncthreads();
    wg_fence();
    tc_chunk_mma(acc, smem_u32(a_hi), smem_u32(a_lo), smem_u32(b_hi), smem_u32(b_lo), kc == 0);
    wg_commit();
  };
  prefetch(0, pa0, pb0);
  if (nk > 1) prefetch(1, pa1, pb1);
  for (int kc = 0; kc < nk; kc += 2) {
    chunk(kc, pa0, pb0);
    if (kc + 1 < nk) chunk(kc + 1, pa1, pb1);
  }
  wg_wait<0>();
  wg_fence_acc(acc);
  sh->cn[tid] = bn_acc;
  __syncthreads();  // every warp's MMAs are complete: the stages are free, cn is visible
  *an = an_acc;
}

// the unclamped score: the expanded L2 form, or the dot
template <int METRIC>
__device__ __forceinline__ float tc_raw(float dot, float xn, float cn) {
  return METRIC == kMetricL2 ? fmaf(-2.0f, dot, xn + cn) : dot;
}
template <int METRIC>
__device__ __forceinline__ float tc_score(float dot, float xn, float cn) {
  // faiss IndexFlat clamps the expanded L2 form at 0 (SURVEY Appendix A)
  return METRIC == kMetricL2 ? fmaxf(0.f, tc_raw<METRIC>(dot, xn, cn)) : dot;
}

// ---- K2 / K6: dense score tile or fused row arg-min ----------------------------------------
template <int METRIC, int EPI_ARGMIN>
__global__ void __launch_bounds__(TC_NT)
    dist_tc_kernel(const float* __restrict__ X, int64_t ldx, int n, const float* __restrict__ C, int64_t ldc, int m,
                   int d, float* __restrict__ out, int64_t ldo, unsigned long long* __restrict__ best) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ TcShared sh;
  const int tid = threadIdx.x;
  const int row0 = blockIdx.y * TC_M, col0 = blockIdx.x * TC_N;
  const float* arow = row0 + tid < n ? X + (int64_t)(row0 + tid) * ldx : nullptr;
  const float* brow = col0 + tid < m ? C + (int64_t)(col0 + tid) * ldc : nullptr;
  float acc[2][64];
  float xn;
  tc_tile_run(smem, &sh, arow, brow, nullptr, d, acc, &xn);
  float* slabs = reinterpret_cast<float*>(smem);

  const int gr = row0 + tid;
  unsigned long long kbest = kKeySentinel;
#pragma unroll
  for (int c0 = 0; c0 < TC_N; c0 += 32) {
    uint32_t v[32];
    acc_cols(acc, c0, slabs, v);
#pragma unroll
    for (int j = 0; j < 32; j++) {
      const int gc = col0 + c0 + j;
      const float raw = tc_raw<METRIC>(__uint_as_float(v[j]), xn, sh.cn[c0 + j]);
      const float s = METRIC == kMetricL2 ? fmaxf(0.f, raw) : raw;
      if (gr < n && gc < m) {
        if (EPI_ARGMIN) {
          // a NaN before L2's clamp at 0 (a NaN or infinite operand: the split of inf is NaN) stays NaN for the key
          unsigned long long key = make_key(argmin_ord<METRIC>(raw != raw ? raw : s), (uint32_t)gc);
          kbest = key < kbest ? key : kbest;
        } else {
          out[(int64_t)gr * ldo + gc] = s;
        }
      }
    }
  }
  if (EPI_ARGMIN && gr < n && kbest != kKeySentinel) atomicMin(best + gr, kbest);
}

// ---- K3 list-major: one (list, 128-pair group, 128-row tile) work item per CTA --------------
template <int METRIC>
__global__ void __launch_bounds__(TC_NT)
    ivf_listmajor_tc_kernel(const float* __restrict__ xq, int64_t ldq, int d, const LmTile* __restrict__ tiles,
                            const int32_t* __restrict__ pair_q, const int64_t* __restrict__ pair_off,
                            ListDirectory dir, const float* __restrict__ shifts, float* __restrict__ scores) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ TcShared sh;
  const int tid = threadIdx.x;
  const LmTile t = tiles[blockIdx.x];
  const float* arow = nullptr;
  int64_t obase = 0;
  if (tid < t.npairs) {
    arow = xq + (int64_t)pair_q[t.pair0 + tid] * ldq;
    obase = pair_off[t.pair0 + tid] + t.row0;
  }
  const float* brow = tid < t.nrows ? dir.vecs[t.list] + (int64_t)(t.row0 + tid) * d : nullptr;
  float acc[2][64];
  float xn;
  tc_tile_run(smem, &sh, arow, brow, shifts ? shifts + (int64_t)t.list * ldq : nullptr, d, acc, &xn);
  float* slabs = reinterpret_cast<float*>(smem);
  // Epilogue.  Thread t owns accumulator row t, but its row lands in a score segment far away from
  // its neighbours' rows, so writing straight from registers would touch 32 different cache lines
  // per store.  Each warp therefore transposes its 32 x 32 block through shared memory (behind the
  // slabs; row stride 33 floats => conflict-free both ways) and writes every row as one contiguous
  // 128-byte run.
  float* stile = reinterpret_cast<float*>(smem + kSlabBytes) + (size_t)(tid >> 5) * 32 * 33;
  const int lane = tid & 31, wrow0 = (tid >> 5) * 32;
#pragma unroll
  for (int c0 = 0; c0 < TC_N; c0 += 32) {
    uint32_t v[32];
    acc_cols(acc, c0, slabs, v);
#pragma unroll
    for (int j = 0; j < 32; j++) stile[lane * 33 + j] = tc_score<METRIC>(__uint_as_float(v[j]), xn, sh.cn[c0 + j]);
    __syncwarp();
    const bool colok = c0 + lane < t.nrows;
#pragma unroll 4
    for (int rr = 0; rr < 32; rr++) {
      const long long ob = __shfl_sync(0xffffffffu, (long long)obase, rr);
      if (wrow0 + rr < t.npairs && colok) scores[ob + c0 + lane] = stile[rr * 33 + lane];
    }
    __syncwarp();
  }
}

// ---- K3 list-major, fused top-k epilogue -----------------------------------------------------
// Thread t of the CTA owns pair t of the item for the whole row segment: accumulator row t, a k-slot
// key set in shared memory (slot-major, thread-minor: conflict-free) and a register bound tau.  The
// hot loop is  score -> one float compare against the bound;  everything else (row validity, score
// window, tombstone, bitmaps, exact 64-bit key compare, set update) sits behind that compare in a
// non-inlined function, as rare as in the query-major kernels (expected k ln(n/k) hits per query).
// tau_g[q] carries the best bound any CTA has published for query q: a key is only dropped when it
// is >= the k-th best of k valid keys of the same query, so the union of the per-pair sets always
// contains the query's true top-k, whatever the CTA schedule.
struct LmkState {
  unsigned long long tau;  // admission bound (exclusive)
  int n;                   // keys held, <= k
};
constexpr uint32_t kLmkNoVid = 0xFFFFFFFFu;

template <int METRIC>
__device__ __noinline__ LmkState lmk_consider(unsigned long long* hk, int k, uint32_t vid, float sc, float min_score,
                                              float max_score, LmkState st) {
  if (vid == kLmkNoVid) return st;  // padding row, tombstone, deleted or filtered out
  if (!(sc <= max_score && sc >= min_score)) return st;
  const unsigned long long key = make_key(score2ord<METRIC>(sc), vid);
  if (key >= st.tau) return st;
  if (st.n < k) {
    hk[st.n * TC_NT] = key;
    if (++st.n < k) return st;
    unsigned long long mx = 0;
    for (int i = 0; i < k; i++) {
      const unsigned long long v = hk[i * TC_NT];
      mx = v > mx ? v : mx;
    }
    if (mx < st.tau) st.tau = mx;
    return st;
  }
  unsigned long long mx = 0, mx2 = 0;
  int pos = 0;
  for (int i = 0; i < k; i++) {
    const unsigned long long v = hk[i * TC_NT];
    if (v > mx) {
      mx2 = mx, mx = v, pos = i;
    } else if (v > mx2) {
      mx2 = v;
    }
  }
  unsigned long long nm = mx;
  if (key < mx) {
    hk[pos * TC_NT] = key;
    nm = key > mx2 ? key : mx2;
  }
  if (nm < st.tau) st.tau = nm;
  return st;
}

// 32 accumulator columns of one pair (thread): turn them into scores in place and collect, branch-free, one
// bit per column that beats the bound the block started with; only then visit the hits (the rare path
// re-checks every hit against the live bound).  cn32 / vid32: the columns' |y|^2 (16-byte aligned) and row ids.
template <int METRIC>
__device__ __forceinline__ void lmk_scan_block(uint32_t (&v)[32], float xn, const float* cn32, const uint32_t* vid32,
                                               unsigned long long* hk, int k, float min_score, float max_score,
                                               LmkState& st, float& bound) {
  uint32_t hit = 0;
#pragma unroll
  for (int j4 = 0; j4 < 32; j4 += 4) {
    const float4 c4 = *reinterpret_cast<const float4*>(cn32 + j4);
    const float cc[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const float sc = tc_score<METRIC>(__uint_as_float(v[j4 + u]), xn, cc[u]);
      v[j4 + u] = __float_as_uint(sc);
      hit |= (METRIC == kMetricL2 ? sc <= bound : sc >= bound) ? (1u << (j4 + u)) : 0u;
    }
  }
  if (hit) {
#pragma unroll
    for (int jj = 0; jj < 32; jj++) {
      if (hit & (1u << jj)) st = lmk_consider<METRIC>(hk, k, vid32[jj], __uint_as_float(v[jj]), min_score, max_score, st);
    }
    bound = key_bound<METRIC>(st.tau);
  }
}

// MMAs of one 128 x 128 tile from a ring of operand stages (warpgroup 0).  Chunk n of the CTA's
// sequence sits in stage n % NST once full[s] completes its phase; every thread arrives on empty[s]
// once its warp's MMAs of that chunk are done (one commit group stays in flight).
template <int NST, int STAGE>
__device__ __forceinline__ void ring_tile_mma(float (&acc)[2][64], uint32_t r_base, uint64_t* full, uint64_t* empty,
                                              int n0, int nk, int a_lo, int b_hi, int b_lo) {
  int prev = 0;
  for (int kc = 0; kc < nk; kc++) {
    const int n = n0 + kc, s = n % NST;
    mbar_wait(&full[s], (uint32_t)((n / NST) & 1));
    const uint32_t a = r_base + (uint32_t)s * STAGE;
    wg_fence();
    tc_chunk_mma(acc, a, a + a_lo, a + b_hi, a + b_lo, kc == 0);
    wg_commit();
    if (kc > 0) {
      wg_wait<1>();
      mbar_arrive(&empty[prev]);
    }
    prev = s;
  }
  wg_wait<0>();
  wg_fence_acc(acc);
  mbar_arrive(&empty[prev]);
}

// Thread 0: the mbarriers of a ring of nst stages.  A full phase completes after full_count arrivals (and, for a
// TMA-fed ring, the transaction bytes of the stage's copies); an empty phase once every MMA thread has arrived.
__device__ __forceinline__ void ring_init(uint64_t* full, uint64_t* empty, int nst, uint32_t full_count) {
  for (int s = 0; s < nst; s++) {
    mbar_init(&full[s], full_count);
    mbar_init(&empty[s], TC_M);
  }
  mbar_fence_init();
}

// After a tile: exchange bounds with the other CTAs working on the same query (tau_q = its slot of tau_g) --
// adopt a tighter published bound, or publish this thread's own.
template <int METRIC>
__device__ __forceinline__ void lmk_exchange_bound(unsigned long long* tau_q, LmkState& st, float& bound) {
  const unsigned long long tg = __ldcg(tau_q);
  if (tg < st.tau) {
    st.tau = tg;
    bound = key_bound<METRIC>(st.tau);
  } else if (st.tau < tg) {
    atomicMin(tau_q, st.tau);
  }
}

// the thread's key set (n keys, slot-major in shared memory) -> o[0, k), sentinel padded
__device__ __forceinline__ void lmk_write_keys(unsigned long long* o, const unsigned long long* hk, int k, int n) {
  for (int i = 0; i < k; i++) o[i] = i < n ? hk[i * TC_NT] : kKeySentinel;
}

// ---- K3 list-major, register-staged pipeline ---------------------------------------------------
// The fused top-k kernel that needs no mirror.  Staging runs concurrently with the MMAs and the
// epilogue, synchronised by mbarriers only:
//   warps 4-7  producers: thread p stages row p of the query group and of the list tile, one K = 16
//              chunk at a time, into a ring of LW_STAGES operand stages (hi/lo TF32 split, canonical
//              K-major layout), two chunks of global loads in flight per thread;
//   warps 0-3  one warpgroup: wgmma over the chunks of tile i as soon as their stages are full
//              (each released as its MMAs complete), then the bound test / key-set update of tile i
//              while the producers fill the ring with tile i + 1.
constexpr int LW_STAGES = 3;
constexpr int LW_NT = 256;
constexpr int LW_RING = LW_STAGES * TC_STAGE_BYTES;

struct LwShared {
  alignas(16) float cn[2][TC_N];  // |y|^2 of the tile's rows (read as float4)
  uint32_t vid[2][TC_N];          // ids of the tile's rows, kLmkNoVid = can never be returned
  float xn[TC_M];                 // |x|^2 of the group's queries
  uint64_t full[LW_STAGES], empty[LW_STAGES], acc_empty[2];
};


template <int METRIC>
__global__ void __launch_bounds__(LW_NT, 1)
    ivf_listmajor_pipe_kernel(const float* __restrict__ xq, int64_t ldq, int d, const LmTile* __restrict__ items,
                              const int64_t* __restrict__ totals, const int64_t* __restrict__ pair_j, int nprobe,
                              ListDirectory dir, const float* __restrict__ shifts, int k, int nseg_max, FilterArgs f,
                              unsigned long long* tau_g, unsigned long long* __restrict__ out) {
  extern __shared__ __align__(1024) unsigned char smem[];  // [ring][slabs][key sets: k * 1 KiB]
  __shared__ LwShared sh;
  if ((int64_t)blockIdx.x >= totals[1]) return;
  if (cta_cancelled(f.cancel, kCsListmajorPipe)) return;
  const int tid = threadIdx.x, warp = tid >> 5;
  const LmTile t = items[blockIdx.x];
  const int row_end = t.row0 + t.nrows;
  const int ntiles = (t.nrows + TC_N - 1) / TC_N;
  // at least two K chunks per tile, which the ring's phase arithmetic assumes (d <= 16: the loads zero-fill
  // columns >= d, so the second chunk adds exact zeros)
  const int nk = max(2, (d + TC_BK - 1) / TC_BK);

  if (tid == 0) {
    for (int b = 0; b < 2; b++) mbar_init(&sh.acc_empty[b], TC_M);  // every epilogue thread arrives
    ring_init(sh.full, sh.empty, LW_STAGES, TC_M);                   // every producer thread arrives
  }
  __syncthreads();
  const uint32_t LBO = TC_M * 16, SBO = 128;

  if (warp < 4) {
    // ======================= MMA + epilogue =======================
    unsigned long long* hk = reinterpret_cast<unsigned long long*>(smem + LW_RING + kSlabBytes) + tid;
    float* slabs = reinterpret_cast<float*>(smem + LW_RING);
    const bool valid = tid < t.npairs;
    int64_t j = 0;
    int q = 0;
    LmkState st{0ull, 0};
    if (valid) {
      j = pair_j[t.pair0 + tid];
      q = (int)(j / nprobe);
      st.tau = __ldcg(tau_g + q);
    }
    float bound = key_bound<METRIC>(st.tau);
    float xn = 0.f;
    float acc[2][64];
    for (int i = 0; i < ntiles; i++) {
      const int b = i & 1;
      ring_tile_mma<LW_STAGES, TC_STAGE_BYTES>(acc, smem_u32(smem), sh.full, sh.empty, i * nk, nk, TC_TILE_BYTES,
                                               2 * TC_TILE_BYTES, 3 * TC_TILE_BYTES);
      if (i == 0) xn = sh.xn[tid];
#pragma unroll
      for (int c0 = 0; c0 < TC_N; c0 += 32) {
        uint32_t v[32];
        acc_cols(acc, c0, slabs, v);
        lmk_scan_block<METRIC>(v, xn, &sh.cn[b][c0], &sh.vid[b][c0], hk, k, f.min_score, f.max_score, st, bound);
      }
      mbar_arrive(&sh.acc_empty[b]);  // cn[b], vid[b] may be overwritten
      if (valid) lmk_exchange_bound<METRIC>(tau_g + q, st, bound);
    }
    if (valid) lmk_write_keys(out + ((int64_t)j * nseg_max + t.seg) * k, hk, k, st.n);
  } else {
    // ======================= producers =======================
    const int p = tid - TC_M;
    const float* arow = nullptr;
    if (p < t.npairs) arow = xq + (pair_j[t.pair0 + p] / nprobe) * ldq;
    const float* lvecs = dir.vecs[t.list];
    const float* shift = shifts ? shifts + (int64_t)t.list * ldq : nullptr;
    const int64_t* __restrict__ lids = dir.ids[t.list];
    const uint32_t row_off = (uint32_t)(p >> 3) * SBO + (uint32_t)(p & 7) * 16;
    constexpr int NV = TC_BK / 4;
    const int T = ntiles * nk;
    float an_acc = 0.f, bn_acc = 0.f;
    uint32_t myvid = kLmkNoVid;
    float4 pa0[NV], pb0[NV], pa1[NV], pb1[NV];
    auto prefetch = [&](int n, float4 (&pa)[NV], float4 (&pb)[NV]) {
      const int i = n / nk, kc = n - i * nk;
      const int row = t.row0 + i * TC_N + p;
      const float* brow = row < row_end ? lvecs + (int64_t)row * d : nullptr;
#pragma unroll
      for (int kb = 0; kb < NV; kb++) {
        const int gk = kc * TC_BK + kb * 4;
        pa[kb] = make_float4(0.f, 0.f, 0.f, 0.f);
        pb[kb] = pa[kb];
        if (arow && gk < d) pa[kb] = __ldg(reinterpret_cast<const float4*>(arow + gk));
        if (brow && gk < d) pb[kb] = __ldg(reinterpret_cast<const float4*>(brow + gk));
        if (shift && gk < d) {
          const float4 s4 = __ldg(reinterpret_cast<const float4*>(shift + gk));
          if (arow) pa[kb] = f4_sub(pa[kb], s4);
          if (brow) pb[kb] = f4_sub(pb[kb], s4);
        }
      }
    };
    auto chunk = [&](int n, float4 (&pa)[NV], float4 (&pb)[NV]) {
      const int i = n / nk, kc = n - i * nk;
      const int s = n % LW_STAGES;
      if (kc == 0) {  // new tile: row validity is resolved while the tile's chunks stream through
        bn_acc = 0.f;
        myvid = kLmkNoVid;
        const int row = t.row0 + i * TC_N + p;
        if (row < row_end) {
          const int64_t raw = lids[row];  // tombstone: gamma_index_ivfflat.h:72
          if (raw >= 0 && ctx_is_valid(f.del_bits, f.filter_bits, (uint32_t)raw)) myvid = (uint32_t)raw;
        }
      }
      mbar_wait(&sh.empty[s], (uint32_t)(((n / LW_STAGES) & 1) ^ 1));
      unsigned char* a_hi = smem + (size_t)s * TC_STAGE_BYTES;
      unsigned char* a_lo = a_hi + TC_TILE_BYTES;
      unsigned char* b_hi = a_hi + 2 * TC_TILE_BYTES;
      unsigned char* b_lo = a_hi + 3 * TC_TILE_BYTES;
#pragma unroll
      for (int kb = 0; kb < NV; kb++) {
        const uint32_t off = (uint32_t)kb * LBO + row_off;
        const float4 va = pa[kb], vb = pb[kb];
        an_acc = fmaf(va.x, va.x, an_acc), an_acc = fmaf(va.y, va.y, an_acc);
        an_acc = fmaf(va.z, va.z, an_acc), an_acc = fmaf(va.w, va.w, an_acc);
        bn_acc = fmaf(vb.x, vb.x, bn_acc), bn_acc = fmaf(vb.y, vb.y, bn_acc);
        bn_acc = fmaf(vb.z, vb.z, bn_acc), bn_acc = fmaf(vb.w, vb.w, bn_acc);
        auto split = [](float v, float& hi, float& lo) {
          hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
          lo = v - hi;
        };
        float4 ah, al, bh, bl;
        split(va.x, ah.x, al.x), split(va.y, ah.y, al.y), split(va.z, ah.z, al.z), split(va.w, ah.w, al.w);
        split(vb.x, bh.x, bl.x), split(vb.y, bh.y, bl.y), split(vb.z, bh.z, bl.z), split(vb.w, bh.w, bl.w);
        *reinterpret_cast<float4*>(a_hi + off) = ah;
        *reinterpret_cast<float4*>(a_lo + off) = al;
        *reinterpret_cast<float4*>(b_hi + off) = bh;
        *reinterpret_cast<float4*>(b_lo + off) = bl;
      }
      if (kc == nk - 1) {  // tile complete: publish its per-row scalars for the epilogue
        const int b = i & 1;
        mbar_wait(&sh.acc_empty[b], (uint32_t)(((i >> 1) & 1) ^ 1));  // epilogue of tile i-2 is done with them
        sh.cn[b][p] = bn_acc;
        sh.vid[b][p] = myvid;
        if (i == 0) sh.xn[p] = an_acc;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> tensor-core proxy
      mbar_arrive(&sh.full[s]);
      // after the arrive: a release-arrive waits for the thread's outstanding loads
      if (n + 2 < T) prefetch(n + 2, pa, pb);
    };
    if (T > 0) prefetch(0, pa0, pb0);
    if (T > 1) prefetch(1, pa1, pb1);
    for (int n = 0; n < T; n += 2) {
      chunk(n, pa0, pb0);
      if (n + 1 < T) chunk(n + 1, pa1, pb1);
    }
  }
}

// ---- K3 list-major, TMA-fed pipeline over the pre-tiled mirror ---------------------------------
// Same work items, same epilogue and the same results as ivf_listmajor_pipe_kernel; what changes is
// who feeds the tensor core.  Both operands already sit in global memory in the canonical operand
// layout (lists: the mirror built by tc_mirror_build_kernel; queries: staged per pair group by
// lm_stage_queries_kernel), so one thread issues two 16 KiB cp.async.bulk copies per K chunk into
// a ring of stages and the copies complete on the stage's mbarrier (complete_tx).  No producer warps, no
// registers or scoreboards tied up by loads, as many chunks in flight as the ring is deep.
//   warps 0-3  one warpgroup: fetch the tile's row ids / norms, wgmma, bound test (thread = pair)
//   warp  4    TMA producer (one elected lane issues)
constexpr int LT_STAGES = 3;  // 32 KiB stages (query chunk + list chunk)
constexpr int LT_NT = 160;
constexpr int LT_RING = LT_STAGES * TC_STAGE_BYTES;
constexpr int LT_HALF = TC_STAGE_BYTES / 2;  // one operand's chunk: hi + lo tile, 16 KiB

struct LtShared {
  alignas(16) float cn[2][TC_N];
  uint32_t vid[2][TC_N];
  uint64_t full[LT_STAGES], empty[LT_STAGES];
};

// TMA producer of an LT_STAGES ring (the whole warp loops, one elected lane issues): for each of ntiles tiles and
// each of its nk K chunks, chunk kc of the A operand (a_chunks, the same for every tile) and chunk (tile, kc) of the
// B operand (b_chunks), 16 KiB each, into the next stage
__device__ __forceinline__ void ring_tma_produce(unsigned char* ring, uint64_t* full, uint64_t* empty, const char* a_chunks,
                                                 const char* b_chunks, int ntiles, int nk) {
  int n = 0;
  for (int i = 0; i < ntiles; i++) {
    for (int kc = 0; kc < nk; kc++, n++) {
      const int s = n % LT_STAGES;
      mbar_wait(&empty[s], (uint32_t)(((n / LT_STAGES) & 1) ^ 1));
      if (elect_one()) {
        unsigned char* stage = ring + (size_t)s * TC_STAGE_BYTES;
        mbar_arrive_expect_tx(&full[s], TC_STAGE_BYTES);
        bulk_g2s(stage, a_chunks + (int64_t)kc * LT_HALF, LT_HALF, &full[s]);
        bulk_g2s(stage + LT_HALF, b_chunks + ((int64_t)i * nk + kc) * LT_HALF, LT_HALF, &full[s]);
      }
      __syncwarp();
    }
  }
}



template <int METRIC>
__global__ void __launch_bounds__(LT_NT, 1)
    ivf_listmajor_tma_kernel(const float* __restrict__ a_scratch, const float* __restrict__ a_norms, TcMirrorView mv,
                             const LmTile* __restrict__ items, const int64_t* __restrict__ totals,
                             const int64_t* __restrict__ pair_j, int nprobe, ListDirectory dir, int k, int nseg_max,
                             FilterArgs f, unsigned long long* tau_g, unsigned long long* __restrict__ out) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ LtShared sh;
  if ((int64_t)blockIdx.x >= totals[1]) return;
  if (cta_cancelled(f.cancel, kCsListmajorTma)) return;
  constexpr int NST = LT_STAGES;
  constexpr int STAGE = TC_STAGE_BYTES;
  const int tid = threadIdx.x, warp = tid >> 5;
  const LmTile t = items[blockIdx.x];
  const int row_end = t.row0 + t.nrows;
  const int ntiles = (t.nrows + TC_N - 1) / TC_N;
  const int nk = mv.k16 / TC_BK;
  unsigned char* ring = smem;  // [ring: NST * STAGE] [slabs] [key sets: k * 1 KiB]

  if (tid == 0) ring_init(sh.full, sh.empty, NST, 1);  // the producer's arrive.expect_tx; the copies complete the phase
  __syncthreads();
  const int64_t tile_floats = (int64_t)TC_N * mv.k16 * 2;
  const int64_t ltile0 = mv.tile0[t.list] + t.row0 / TC_N;  // first mirror tile of this item

  if (warp < 4) {
    // ======================= MMA + epilogue =======================
    unsigned long long* hk = reinterpret_cast<unsigned long long*>(ring + (size_t)NST * STAGE + kSlabBytes) + tid;
    float* slabs = reinterpret_cast<float*>(ring + (size_t)NST * STAGE);
    const bool valid = tid < t.npairs;
    int64_t j = 0;
    int q = 0;
    LmkState st{0ull, 0};
    if (valid) {
      j = pair_j[t.pair0 + tid];
      q = (int)(j / nprobe);
      st.tau = __ldcg(tau_g + q);
    }
    float bound = key_bound<METRIC>(st.tau);
    const float xn = a_norms[(int64_t)t.grp * TC_M + tid];
    const int64_t* __restrict__ lids = dir.ids[t.list];
    float acc[2][64];
    for (int i = 0; i < ntiles; i++) {
      const int b = i & 1;
      // this tile's per-row scalars: loads issued before the MMAs, stored after them
      const int row = t.row0 + i * TC_N + tid;
      int64_t raw = -1;
      float cn = 0.f;
      if (row < row_end) {
        raw = lids[row];
        cn = mv.norms[(ltile0 + i) * TC_N + tid];
      }
      ring_tile_mma<NST, STAGE>(acc, smem_u32(ring), sh.full, sh.empty, i * nk, nk, TC_TILE_BYTES, LT_HALF,
                                LT_HALF + TC_TILE_BYTES);
      uint32_t myvid = kLmkNoVid;
      if (raw >= 0 && ctx_is_valid(f.del_bits, f.filter_bits, (uint32_t)raw)) myvid = (uint32_t)raw;  // tombstone: gamma_index_ivfflat.h:72
      sh.cn[b][tid] = cn;  // buffer b was last read in tile i - 2, before tile i - 1's exchange barriers
      sh.vid[b][tid] = myvid;  // visible after the first exchange's barrier
#pragma unroll
      for (int c0 = 0; c0 < TC_N; c0 += 32) {
        uint32_t v[32];
        acc_cols(acc, c0, slabs, v);
        lmk_scan_block<METRIC>(v, xn, &sh.cn[b][c0], &sh.vid[b][c0], hk, k, f.min_score, f.max_score, st, bound);
      }
      if (valid) lmk_exchange_bound<METRIC>(tau_g + q, st, bound);
    }
    if (valid) lmk_write_keys(out + ((int64_t)j * nseg_max + t.seg) * k, hk, k, st.n);
  } else {
    // ======================= TMA producer =======================
    ring_tma_produce(ring, sh.full, sh.empty, reinterpret_cast<const char*>(a_scratch) + (int64_t)t.grp * nk * LT_HALF,
                     reinterpret_cast<const char*>(mv.base + ltile0 * tile_floats), ntiles, nk);
  }
}


// one operand row -> its 16-byte units of every K chunk, TF32 head and fp32 remainder, canonical
// K-major layout; returns |row|^2 accumulated in index order (the order the staging loops use).
// shift: nullptr, or a row subtracted first (the K3 list shift: src - s_l; a missing row stays zero)
__device__ __forceinline__ float tc_split_row(const float* __restrict__ src, const float* __restrict__ shift, int d, int k16,
                                              int r, float* tile) {
  float nrm = 0.f;
  for (int kc = 0; kc < k16 / TC_BK; kc++) {
    float* hi = tile + (int64_t)kc * (TC_STAGE_BYTES / 8);  // 16 KiB per chunk = 4096 floats: hi then lo
    float* lo = hi + TC_TILE_BYTES / 4;
#pragma unroll
    for (int k4 = 0; k4 < 4; k4++) {
      const int gk = kc * TC_BK + k4 * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (src && gk < d) v = __ldg(reinterpret_cast<const float4*>(src + gk));
      if (src && shift && gk < d) v = f4_sub(v, __ldg(reinterpret_cast<const float4*>(shift + gk)));
      nrm = fmaf(v.x, v.x, nrm), nrm = fmaf(v.y, v.y, nrm), nrm = fmaf(v.z, v.z, nrm), nrm = fmaf(v.w, v.w, nrm);
      float4 h, l;
      h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u), l.x = v.x - h.x;
      h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u), l.y = v.y - h.y;
      h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u), l.z = v.z - h.z;
      h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u), l.w = v.w - h.w;
      const int off = k4 * (TC_M * 4) + r * 4;  // unit (r, k4): k4 * LBO + r * 16 bytes
      *reinterpret_cast<float4*>(hi + off) = h;
      *reinterpret_cast<float4*>(lo + off) = l;
    }
  }
  return nrm;
}

__global__ void __launch_bounds__(TC_N)
    tc_mirror_build_kernel(ListDirectory dir, int d, int k16, const int64_t* __restrict__ tile0,
                           const float* __restrict__ shifts, float* __restrict__ mirror, float* __restrict__ norms) {
  const int64_t gt = blockIdx.x;
  int lo = 0, hi = dir.nlist;  // last list whose first tile is <= gt
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tile0[mid] <= gt) lo = mid; else hi = mid;
  }
  const int l = lo, r = threadIdx.x;
  const int row = (int)(gt - tile0[l]) * TC_N + r;
  const float* src = row < dir.len[l] ? dir.vecs[l] + (int64_t)row * d : nullptr;
  norms[gt * TC_N + r] = tc_split_row(src, shifts ? shifts + (int64_t)l * d : nullptr, d, k16, r,
                                      mirror + gt * ((int64_t)TC_N * k16 * 2));
}

// The K3 list shifts (one block per list l): rho = half the distance from c_l to its nearest other centroid (fp64,
// direct form), g = the largest power of two <= rho / sqrt(d), s_l = round(c_l / g) * g; s_l = c_l when rho = 0.
// The grid keeps integer data integer: an integer centroid, or any g >= 1, gives an integer shift.
__global__ void __launch_bounds__(256)
    list_shift_kernel(const float* __restrict__ cent, int64_t ldc, int nlist, int d, float* __restrict__ shifts) {
  __shared__ double red[8];
  const int l = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* cl = cent + (int64_t)l * ldc;
  double best = INFINITY;
  for (int j = warp; j < nlist; j += 8) {
    if (j == l) continue;
    const float* cj = cent + (int64_t)j * ldc;
    double acc = 0.0;
    for (int c = lane; c < d; c += 32) {
      const double t = (double)cl[c] - (double)cj[c];
      acc = fma(t, t, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    best = fmin(best, acc);
  }
  if (lane == 0) red[warp] = best;
  __syncthreads();
  double r2 = red[0];  // squared distance to the nearest other centroid (inf if nlist == 1)
  for (int w = 1; w < 8; w++) r2 = fmin(r2, red[w]);
  const double t = r2 / 4.0 / (double)d;  // (rho / sqrt(d))^2
  const bool exact = !(t > 0.0) || isinf(t);
  double g = 0.0;
  if (!exact) {
    int e;
    frexp(t, &e);  // t in [2^(e-1), 2^e): g^2 <= t for g = 2^p iff 2p <= e - 1
    const int E = e - 1;
    g = ldexp(1.0, E >= 0 ? E / 2 : -((1 - E) / 2));
  }
  for (int c = tid; c < ldc; c += blockDim.x) {
    const float v = cl[c];
    shifts[(int64_t)l * ldc + c] = exact ? v : (float)(rint((double)v / g) * g);
  }
}

__global__ void tc_mirror_append_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d, int k16,
                                        const int32_t* __restrict__ list, const int32_t* __restrict__ pos,
                                        const int64_t* __restrict__ tile0, const float* __restrict__ shifts,
                                        float* __restrict__ mirror, float* __restrict__ norms) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = list[i];
  if (l < 0) return;
  const int p = pos[i];
  const int64_t gt = tile0[l] + p / TC_N;
  norms[gt * TC_N + p % TC_N] = tc_split_row(x + i * ldx, shifts ? shifts + (int64_t)l * d : nullptr, d, k16, p % TC_N,
                                             mirror + gt * ((int64_t)TC_N * k16 * 2));
}

// Stages 128-row operand tiles (canonical layout, hi + lo per K chunk) and their row norms.  With items: tile = pair
// group, row r = the query of the group's pair r.  Without (items == nullptr): tile b = rows [128 b, 128 b + 128) of
// x, rows past nrows zero (the coarse quantiser's query tiles and the centroid copy).
__global__ void __launch_bounds__(TC_M)
    lm_stage_queries_kernel(const float* __restrict__ xq, int64_t ldq, int d, int k16, const LmTile* __restrict__ items,
                            const int64_t* __restrict__ totals, const int64_t* __restrict__ pair_j, int nprobe, int64_t nrows,
                            const float* __restrict__ shifts, float* __restrict__ a_scratch, float* __restrict__ a_norms) {
  const int r = threadIdx.x;
  int64_t grp = blockIdx.x;
  const float* src = nullptr;
  const float* shift = nullptr;
  if (items) {
    if ((int64_t)blockIdx.x >= totals[1]) return;
    const LmTile t = items[blockIdx.x];
    if (t.seg != 0) return;  // one staging per pair group: the first item of the group owns the slot
    grp = t.grp;
    if (r < t.npairs) src = xq + (pair_j[t.pair0 + r] / nprobe) * ldq;
    if (shifts) shift = shifts + (int64_t)t.list * ldq;
  } else if (grp * TC_M + r < nrows) {
    src = xq + (grp * TC_M + r) * ldq;
  }
  a_norms[grp * TC_M + r] = tc_split_row(src, shift, d, k16, r, a_scratch + grp * ((int64_t)TC_M * k16 * 2));
}

// ---- K2 fused: the coarse quantiser's top-nprobe on the tensor cores ----------------------------
// Warp roles (ck_nt<TPQ>() threads, one CTA per SM):
//   warps 0-3           one warpgroup: the wgmma sequence of dist_tc_kernel (the same chunks, MMAs and order, so every
//                       score is bit-equal to the matrix that kernel writes) for tile i + 1 while the selection warps
//                       scan tile i; then the accumulator goes to the score buffer (four slabs, acc_to_slab layout).
//                       Thread 0 refills each ring stage by TMA once every warp's MMAs of it are complete: a
//                       producer warp of its own would lower every thread's register budget below the 128 registers
//                       the accumulator alone takes.
//   next 128 * TPQ      selection: TPQ threads per query, thread (r, h) scans columns [h, h + 1) * 128 / TPQ of query
//                       r's row of every tile and keeps its own key set of k keys
// The score buffer is single (full / empty mbarriers); the accumulator registers are the second buffer.
//
// Work split: the nqt x ntc (query tile, centroid tile) pairs, query-tile-major, are cut into gridDim.x equal
// contiguous ranges, one per CTA.  A query tile shared by several CTAs gets one partial key set per CTA and thread;
// the CTA that completes it last (a per-tile counter) merges them, sorts and writes the tile's keys.  Every key set
// of a query holds only keys below a bound that is the k-th best of k of its valid keys (tau_g shares the bounds of
// one query across threads and CTAs), so their union holds the query's true top k; the merge runs without that bound.
constexpr int CK_NST = LT_STAGES;
constexpr int CK_SCORE_BYTES = 4 * kSlabFloats * 4;  // the 128 x 128 dot products of one tile: 64 KiB
constexpr int CK_MIN_TILES = 4;                      // fewest tile pairs per CTA (bounds the partial sets a merge reads)

// threads per query: as many as fit their key sets (k keys of 8 bytes each) in 64 KiB, at most two
__host__ __device__ constexpr int ck_tpq(int k) { return k <= 32 ? 2 : 1; }
template <int TPQ>
__host__ __device__ constexpr int ck_nt() {
  return TC_M * (1 + TPQ);
}
// the CTA whose range holds tile pair w, for W pairs cut into G ranges [b W / G, (b + 1) W / G)
__host__ __device__ __forceinline__ int ck_owner(int64_t w, int64_t W, int G) { return (int)(((w + 1) * G - 1) / W); }

struct CkShared {
  alignas(16) float cn[TC_N];  // |y|^2 of the buffered tile's centroids
  uint64_t full[CK_NST], sfull, sempty;
  int last;
};

// named barrier of the selection threads (barrier 1 is wg0_sync's)
template <int NSEL>
__device__ __forceinline__ void ck_sel_sync() {
  asm volatile("bar.sync 2, %0;" ::"n"(NSEL) : "memory");
}

// A key set: slot i of selection thread s at hk[i * S].  Once it holds k keys they form a max-heap, so a replacement
// costs one sift-down (log2 k levels of two independent shared loads) instead of a scan of all k slots.
template <int S>
__device__ __forceinline__ void ck_sift_down(unsigned long long* hk, int n, int i, unsigned long long key) {
  for (;;) {
    const int l = 2 * i + 1;
    if (l >= n) break;
    const unsigned long long vl = hk[l * S], vr = l + 1 < n ? hk[(l + 1) * S] : 0ull;
    const int c = vr > vl ? l + 1 : l;
    const unsigned long long vc = vr > vl ? vr : vl;
    if (vc <= key) break;
    hk[i * S] = vc;
    i = c;
  }
  hk[i * S] = key;
}

// the admission rule of lmk_consider: key < st.tau enters; k keys kept
template <int S>
__device__ __noinline__ LmkState ck_insert(unsigned long long* hk, int k, unsigned long long key, LmkState st) {
  if (key >= st.tau) return st;
  if (st.n < k) {
    hk[st.n * S] = key;
    if (++st.n < k) return st;
    for (int i = k / 2 - 1; i >= 0; i--) ck_sift_down<S>(hk, k, i, hk[i * S]);  // the set is full: heapify
  } else {
    ck_sift_down<S>(hk, k, 0, key);  // key < st.tau <= the largest key: it replaces the top
  }
  const unsigned long long mx = hk[0];
  if (mx < st.tau) st.tau = mx;
  return st;
}

template <int METRIC, int S>
__device__ __forceinline__ LmkState ck_consider(unsigned long long* hk, int k, uint32_t vid, float sc, LmkState st) {
  // the score window of select_rows_kernel: non-finite scores never enter
  if (vid == kLmkNoVid || !(sc <= FLT_MAX && sc >= -FLT_MAX)) return st;
  return ck_insert<S>(hk, k, make_key(score2ord<METRIC>(sc), vid), st);
}

// keys of a partial set -> this thread's set, eight loads in flight
template <int S>
__device__ __forceinline__ LmkState ck_absorb(unsigned long long* hk, int k, const unsigned long long* src, int64_t stride,
                                              LmkState st) {
  for (int i0 = 0; i0 < k; i0 += 8) {
    unsigned long long v[8];
#pragma unroll
    for (int u = 0; u < 8; u++) v[u] = i0 + u < k ? __ldcg(src + (int64_t)(i0 + u) * stride) : kKeySentinel;
#pragma unroll
    for (int u = 0; u < 8; u++)
      if (v[u] < st.tau) st = ck_insert<S>(hk, k, v[u], st);
  }
  return st;
}

template <int METRIC, int TPQ>
__global__ void __launch_bounds__(ck_nt<TPQ>(), 1)
    coarse_topk_kernel(const float* __restrict__ a_tiles, const float* __restrict__ a_norms, int nq,
                       const float* __restrict__ c_tiles, const float* __restrict__ c_norms, int nlist, int k16, int k,
                       int nparts, unsigned long long* tau_g, unsigned int* cnt, unsigned long long* part,
                       unsigned long long* __restrict__ out) {
  extern __shared__ __align__(1024) unsigned char smem[];  // [ring: NST * STAGE] [score buffer] [key sets: k * NSEL * 8]
  __shared__ CkShared sh;
  constexpr int NST = CK_NST, STAGE = TC_STAGE_BYTES, NSEL = TC_M * TPQ, SLICE = TC_N / TPQ;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int nk = k16 / TC_BK, ntc = (nlist + TC_N - 1) / TC_N;
  const int64_t W = (int64_t)((nq + TC_M - 1) / TC_M) * ntc;
  const int G = gridDim.x, b = blockIdx.x;
  const int64_t w0 = b * W / G, w1 = (b + 1) * W / G;
  unsigned char* ring = smem;
  float* scores = reinterpret_cast<float*>(smem + (size_t)NST * STAGE);

  if (tid == 0) {
    for (int s = 0; s < NST; s++) mbar_init(&sh.full[s], 1);  // thread 0's arrive.expect_tx; the copies complete the phase
    mbar_init(&sh.sfull, TC_M);
    mbar_init(&sh.sempty, NSEL);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ======================= MMA =======================
    // chunk n of this CTA's sequence: K chunk n % nk of tile pair w0 + n / nk, in ring stage n % NST
    const int64_t nchunks = (w1 - w0) * nk;
    auto issue = [&](int64_t n) {
      const int64_t w = w0 + n / nk;
      const int kc = (int)(n % nk), qt = (int)(w / ntc), ct = (int)(w % ntc);
      unsigned char* stage = ring + (size_t)(n % NST) * STAGE;
      uint64_t* full = &sh.full[n % NST];
      mbar_arrive_expect_tx(full, STAGE);
      bulk_g2s(stage, reinterpret_cast<const char*>(a_tiles) + ((int64_t)qt * nk + kc) * LT_HALF, LT_HALF, full);
      bulk_g2s(stage + LT_HALF, reinterpret_cast<const char*>(c_tiles) + ((int64_t)ct * nk + kc) * LT_HALF, LT_HALF, full);
    };
    // the stage of chunk m has been read by every warp's MMAs (their wgmma groups are complete): chunk m + NST
    auto refill = [&](int64_t m) {
      wg0_sync();
      if (tid == 0 && m + NST < nchunks) issue(m + NST);
    };
    if (tid == 0)
      for (int64_t n = 0; n < NST && n < nchunks; n++) issue(n);
    float acc[2][64];
    int64_t n = 0;
    int i = 0;
    for (int64_t w = w0; w < w1; w++, i++) {
      const int ct = (int)(w % ntc);
      const float cn = c_norms[ct * TC_N + tid];  // issued before the MMAs, stored after them
      for (int kc = 0; kc < nk; kc++, n++) {
        mbar_wait(&sh.full[n % NST], (uint32_t)((n / NST) & 1));
        const uint32_t a = smem_u32(ring) + (uint32_t)(n % NST) * STAGE;
        wg_fence();
        tc_chunk_mma(acc, a, a + TC_TILE_BYTES, a + LT_HALF, a + LT_HALF + TC_TILE_BYTES, kc == 0);
        wg_commit();
        if (kc > 0) {
          wg_wait<1>();
          refill(n - 1);
        }
      }
      wg_wait<0>();
      wg_fence_acc(acc);
      refill(n - 1);
      mbar_wait(&sh.sempty, (uint32_t)((i & 1) ^ 1));  // the selection threads are done with tile i - 1
#pragma unroll
      for (int c0 = 0; c0 < TC_N; c0 += 32) acc_to_slab(acc, c0, scores + (c0 >> 5) * kSlabFloats);
      sh.cn[tid] = cn;
      mbar_arrive(&sh.sfull);
    }
  } else {
    // ======================= selection =======================
    const int sid = tid - TC_M, r = sid & (TC_M - 1), h = sid / TC_M;
    unsigned long long* hk = reinterpret_cast<unsigned long long*>(scores + 4 * kSlabFloats) + sid;
    LmkState st{0ull, 0};
    float bound = 0.f, xn = 0.f;
    int q = 0;
    bool valid = false;
    int i = 0;
    for (int64_t w = w0; w < w1; w++, i++) {
      const int qt = (int)(w / ntc), ct = (int)(w - (int64_t)qt * ntc);
      if (ct == 0 || w == w0) {  // this CTA's first tile of query tile qt: a fresh key set
        q = qt * TC_M + r;
        valid = q < nq;
        st = LmkState{valid ? __ldcg(tau_g + q) : 0ull, 0};  // bound 0: padding rows admit nothing
        bound = key_bound<METRIC>(st.tau);
        xn = a_norms[q];
      }
      mbar_wait(&sh.sfull, (uint32_t)(i & 1));
#pragma unroll
      for (int c0 = h * SLICE; c0 < (h + 1) * SLICE; c0 += 32) {
        const float* slab = scores + (c0 >> 5) * kSlabFloats;
        uint32_t v[32];
        slab_row(slab, v);
        uint32_t hit = 0;
#pragma unroll
        for (int j4 = 0; j4 < 32; j4 += 4) {
          const float4 c4 = *reinterpret_cast<const float4*>(&sh.cn[c0 + j4]);
          const float cc[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
          for (int u = 0; u < 4; u++) {
            const float sc = tc_score<METRIC>(__uint_as_float(v[j4 + u]), xn, cc[u]);
            hit |= (METRIC == kMetricL2 ? sc <= bound : sc >= bound) ? (1u << (j4 + u)) : 0u;
          }
        }
        // Each lane walks its OWN hits, re-reading the dot product from the slab, so a warp iterates as often as
        // its busiest lane and not once per column that any lane hit.
        const float* srow = slab + r * 32;  // this thread's row (acc_to_slab layout)
        while (hit) {
          const int jj = __ffs(hit) - 1;
          hit &= hit - 1;
          const float sc = tc_score<METRIC>(srow[(((jj >> 2) ^ (r & 7)) << 2) | (jj & 3)], xn, sh.cn[c0 + jj]);
          const int col = ct * TC_N + c0 + jj;
          st = ck_consider<METRIC, NSEL>(hk, k, col < nlist ? (uint32_t)col : kLmkNoVid, sc, st);
        }
        bound = key_bound<METRIC>(st.tau);
      }
      mbar_arrive(&sh.sempty);
      if (valid) lmk_exchange_bound<METRIC>(tau_g + q, st, bound);  // with the query's other threads and CTAs
      if (ct != ntc - 1 && w != w1 - 1) continue;

      // ---- this CTA is done with query tile qt ----
      for (int j = st.n; j < k; j++) hk[j * NSEL] = kKeySentinel;  // a set of fewer than k keys reads as k
      const int first = ck_owner((int64_t)qt * ntc, W, G);
      const int nown = ck_owner((int64_t)qt * ntc + ntc - 1, W, G) - first + 1;
      const int slot = b - first;
      // partial set (query tile, slot, h): k keys, key i of row r at [i][r]
      auto part_at = [&](int s, int hh) { return part + (((int64_t)qt * nparts + s) * TPQ + hh) * k * TC_M + r; };
      bool merge = true;
      if (nown > 1) {
        if (valid) {
          unsigned long long* o = part_at(slot, h);
          for (int j = 0; j < k; j++) o[(int64_t)j * TC_M] = hk[j * NSEL];
        }
        __threadfence();
        ck_sel_sync<NSEL>();
        if (sid == 0) sh.last = atomicAdd(cnt + qt, 1u) == (unsigned)(nown - 1);
        ck_sel_sync<NSEL>();
        merge = sh.last;  // the other CTAs of this tile have published theirs
        if (merge) __threadfence();
      }
      if (!merge) continue;
      // exact union of the sets: no borrowed bound from here on
      st.tau = st.n == k ? hk[0] : kKeySentinel;
      if (valid)
        for (int s = 0; s < nown; s++)
          if (s != slot) st = ck_absorb<NSEL>(hk, k, part_at(s, h), TC_M, st);
      for (int j = st.n; j < k; j++) hk[j * NSEL] = kKeySentinel;
      if (TPQ > 1) ck_sel_sync<NSEL>();  // the partner's set is complete
      if (h == 0 && valid) {
        for (int hh = 1; hh < TPQ; hh++)
          for (int j = 0; j < k; j++) st = ck_insert<NSEL>(hk, k, hk[(j * NSEL) + hh * TC_M], st);
        // ascending order: a set of k keys is a max-heap; a smaller one is heapified first
        const int n = st.n;
        if (n < k)
          for (int j = n / 2 - 1; j >= 0; j--) ck_sift_down<NSEL>(hk, n, j, hk[j * NSEL]);
        for (int m = n - 1; m > 0; m--) {
          const unsigned long long top = hk[0];
          ck_sift_down<NSEL>(hk, m, 0, hk[m * NSEL]);
          hk[m * NSEL] = top;
        }
        unsigned long long* o = out + (int64_t)q * k;
        for (int j = 0; j < k; j++) o[j] = j < n ? hk[j * NSEL] : kKeySentinel;
      }
      if (TPQ > 1) ck_sel_sync<NSEL>();  // the partner's set is read before its next tile refills it
    }
  }
}

__global__ void coarse_init_kernel(unsigned long long* __restrict__ tau_g, int nq, unsigned int* __restrict__ cnt, int nqt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nq) tau_g[i] = kKeySentinel;
  if (i < nqt) cnt[i] = 0;
}

// ---- grouping for the fused kernel: histogram (lm_count_kernel) -> scan -> slots -> items ----
__device__ __forceinline__ int lmk_nseg(int len, int nseg_max) {
  int n = (len + kLmkSegRows - 1) / kLmkSegRows;
  return n < 1 ? 1 : (n > nseg_max ? nseg_max : n);
}

__global__ void __launch_bounds__(1024)
    lmk_scan_kernel(const int32_t* __restrict__ cnt, ListDirectory dir, int nseg_max, int gsize, int32_t* __restrict__ start,
                    int32_t* __restrict__ item_start, int32_t* __restrict__ grp_start, int64_t* __restrict__ totals) {
  __shared__ long long s_pairs[1024], s_items[1024], s_grps[1024];
  __shared__ long long carry[3];
  const int tid = threadIdx.x;
  if (tid == 0) carry[0] = carry[1] = carry[2] = 0;
  __syncthreads();
  for (int base = 0; base < dir.nlist; base += 1024) {
    const int l = base + tid;
    long long c = 0, it = 0, g = 0;
    if (l < dir.nlist) {
      c = cnt[l];
      const int len = dir.len[l];
      if (c > 0 && len > 0) {
        g = (c + gsize - 1) / gsize;
        it = g * lmk_nseg(len, nseg_max);
      }
    }
    s_pairs[tid] = c, s_items[tid] = it, s_grps[tid] = g;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      long long a = 0, b = 0, e = 0;
      if (tid >= off) a = s_pairs[tid - off], b = s_items[tid - off], e = s_grps[tid - off];
      __syncthreads();
      s_pairs[tid] += a, s_items[tid] += b, s_grps[tid] += e;
      __syncthreads();
    }
    if (l < dir.nlist) {
      start[l] = (int32_t)(carry[0] + s_pairs[tid] - c);
      item_start[l] = (int32_t)(carry[1] + s_items[tid] - it);
      grp_start[l] = (int32_t)(carry[2] + s_grps[tid] - g);
    }
    __syncthreads();
    if (tid == 1023) carry[0] += s_pairs[1023], carry[1] += s_items[1023], carry[2] += s_grps[1023];
    __syncthreads();
  }
  if (tid == 0) totals[0] = carry[2], totals[1] = carry[1], totals[2] = carry[0];  // groups, items, pairs
}

__global__ void lmk_assign_kernel(const int32_t* __restrict__ probe_ids, int64_t npairs, ListDirectory dir,
                                  const int32_t* __restrict__ start, int32_t* __restrict__ cursor,
                                  int64_t* __restrict__ pair_j) {
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= npairs) return;
  const int l = probe_ids[j];
  if (l < 0 || l >= dir.nlist || dir.len[l] <= 0) return;
  pair_j[start[l] + atomicAdd(cursor + l, 1)] = j;  // slot order inside a list does not affect results
}

__global__ void lmk_items_kernel(const int32_t* __restrict__ cnt, const int32_t* __restrict__ start,
                                 const int32_t* __restrict__ item_start, const int32_t* __restrict__ grp_start,
                                 ListDirectory dir, int nseg_max, int gsize, LmTile* __restrict__ items) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= dir.nlist) return;
  const int c = cnt[l], len = dir.len[l];
  if (c <= 0 || len <= 0) return;
  const int nseg = lmk_nseg(len, nseg_max);
  const int seglen = (((len + nseg - 1) / nseg) + TC_N - 1) / TC_N * TC_N;
  // the list's pairs are split evenly over its ceil(c / gsize) groups: no group is a mostly empty remainder
  const int ng = (c + gsize - 1) / gsize;
  int it = item_start[l];
  for (int g = 0; g < ng; g++) {
    const int p0 = (int)((int64_t)g * c / ng), p1 = (int)((int64_t)(g + 1) * c / ng);
    for (int sg = 0; sg < nseg; sg++) {
      LmTile tl;
      tl.list = l, tl.pair0 = start[l] + p0, tl.npairs = p1 - p0;
      tl.row0 = sg * seglen, tl.nrows = max(0, min(seglen, len - tl.row0)), tl.seg = sg;
      tl.grp = grp_start[l] + g;
      items[it++] = tl;
    }
  }
}

// ---- segment select: per query, stream its P score segments, filter, keep the top-k ---------
constexpr int SEG_NT = 256;
constexpr int SEG_ITEMS = 4;

template <int METRIC>
__global__ void __launch_bounds__(SEG_NT)
    seg_select_kernel(const float* __restrict__ scores, const int64_t* __restrict__ seg_off,
                      const int32_t* __restrict__ probe_ids, int nprobe, ListDirectory dir, int k, int KP, int SORTN,
                      FilterArgs f, unsigned long long* __restrict__ out_keys) {
  if (cta_cancelled(f.cancel, kCsSegSelect)) return;
  extern __shared__ __align__(16) unsigned char sel_smem[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(sel_smem);
  __shared__ int s_cnt;
  __shared__ unsigned long long s_tau;
  CandQueue cq{buf, &s_cnt, &s_tau, k, KP, SORTN};
  cq.init();
  const int q = blockIdx.x;
  int est = 0;
  const int flush_at = max(SEG_NT * SEG_ITEMS - KP, 4 * KP);
  for (int p = 0; p < nprobe; p++) {
    const int list = probe_ids[(int64_t)q * nprobe + p];
    const int64_t off = seg_off[(int64_t)q * nprobe + p];
    if (list < 0 || list >= dir.nlist || off < 0) continue;  // CTA-uniform
    const int len = dir.len[list];
    const float* __restrict__ seg = scores + off;
    const int64_t* __restrict__ lids = dir.ids[list];
    for (int base = 0; base < len; base += SEG_NT * SEG_ITEMS) {
      const unsigned long long tau = s_tau;
      float sv[SEG_ITEMS];
#pragma unroll
      for (int u = 0; u < SEG_ITEMS; u++) {
        const int j = base + u * SEG_NT + threadIdx.x;
        sv[u] = j < len ? seg[j] : 0.f;
      }
      int pushed = 0;
#pragma unroll
      for (int u = 0; u < SEG_ITEMS; u++) {
        const int j = base + u * SEG_NT + threadIdx.x;
        const float sc = sv[u];
        bool pred = j < len && sc <= f.max_score && sc >= f.min_score;
        unsigned long long key = kKeySentinel;
        const uint32_t ord = score2ord<METRIC>(sc);
        pred = pred && ord <= (uint32_t)(tau >> 32);
        if (pred) {
          const int64_t raw = lids[j];
          pred = raw >= 0;  // tombstone (gamma_index_ivfflat.h:72)
          const uint32_t vid = (uint32_t)raw;
          if (pred) pred = ctx_is_valid(f.del_bits, f.filter_bits, vid);
          key = make_key(ord, vid);
          pred = pred && key < tau;
        }
        cq.push_warp(pred, key);
        pushed |= pred ? 1 : 0;
      }
      // exact fill after a barrier pair (one more barrier than an upper bound, but flushes -- block
      // bitonic sorts -- are what this kernel spends its instructions on): flush early so tau
      // tightens after the first ~1k candidates, and whenever the next round might overflow
      (void)pushed;
      __syncthreads();
      est = s_cnt;
      __syncthreads();
      if (est >= flush_at || est + SEG_NT * SEG_ITEMS > cq.cap()) cq.flush();
    }
  }
  __syncthreads();
  cq.flush(true);
  for (int i = threadIdx.x; i < k; i += SEG_NT) out_keys[(int64_t)q * k + i] = buf[i];
}

// ---- list-major grouping on device: histogram -> scan -> slot assignment -> tile table ------
__global__ void lm_count_kernel(const int32_t* __restrict__ probe_ids, int64_t npairs, ListDirectory dir,
                                int32_t* __restrict__ cnt) {
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= npairs) return;
  int l = probe_ids[j];
  if (l >= 0 && l < dir.nlist && dir.len[l] > 0) atomicAdd(cnt + l, 1);
}

// single CTA: exclusive scans over the lists of (pairs, score floats, tiles); totals[0] = floats,
// totals[1] = tiles, totals[2] = valid pairs
__global__ void __launch_bounds__(1024)
    lm_scan_kernel(const int32_t* __restrict__ cnt, ListDirectory dir, int32_t* __restrict__ start,
                   int64_t* __restrict__ base_off, int32_t* __restrict__ tile_start, int64_t* __restrict__ totals) {
  __shared__ long long s_pairs[1024], s_floats[1024], s_tiles[1024];
  __shared__ long long carry[3];
  const int tid = threadIdx.x;
  if (tid == 0) carry[0] = carry[1] = carry[2] = 0;
  __syncthreads();
  for (int base = 0; base < dir.nlist; base += 1024) {
    const int l = base + tid;
    long long c = 0, fl = 0, tl = 0;
    if (l < dir.nlist) {
      c = cnt[l];
      const long long len = dir.len[l];
      fl = c * len;
      tl = ((c + 127) / 128) * ((len + 127) / 128);
    }
    s_pairs[tid] = c, s_floats[tid] = fl, s_tiles[tid] = tl;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {  // Hillis-Steele inclusive scan
      long long a = 0, b = 0, e = 0;
      if (tid >= off) a = s_pairs[tid - off], b = s_floats[tid - off], e = s_tiles[tid - off];
      __syncthreads();
      s_pairs[tid] += a, s_floats[tid] += b, s_tiles[tid] += e;
      __syncthreads();
    }
    if (l < dir.nlist) {
      start[l] = (int32_t)(carry[0] + s_pairs[tid] - c);
      base_off[l] = carry[1] + s_floats[tid] - fl;
      tile_start[l] = (int32_t)(carry[2] + s_tiles[tid] - tl);
    }
    __syncthreads();
    if (tid == 1023) carry[0] += s_pairs[1023], carry[1] += s_floats[1023], carry[2] += s_tiles[1023];
    __syncthreads();
  }
  if (tid == 0) totals[0] = carry[1], totals[1] = carry[2], totals[2] = carry[0];
}

__global__ void lm_assign_kernel(const int32_t* __restrict__ probe_ids, int64_t npairs, int nprobe, ListDirectory dir,
                                 const int32_t* __restrict__ start, int32_t* __restrict__ cursor,
                                 const int64_t* __restrict__ base_off, int32_t* __restrict__ pair_q,
                                 int64_t* __restrict__ pair_off, int64_t* __restrict__ seg_off) {
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= npairs) return;
  int l = probe_ids[j];
  if (l < 0 || l >= dir.nlist || dir.len[l] <= 0) {
    seg_off[j] = -1;
    return;
  }
  const int within = atomicAdd(cursor + l, 1);  // slot order inside a list does not affect results
  const int slot = start[l] + within;
  const int64_t off = base_off[l] + (int64_t)within * dir.len[l];
  pair_q[slot] = (int32_t)(j / nprobe);
  pair_off[slot] = off;
  seg_off[j] = off;
}

__global__ void lm_tiles_kernel(const int32_t* __restrict__ cnt, const int32_t* __restrict__ start,
                                const int32_t* __restrict__ tile_start, ListDirectory dir, LmTile* __restrict__ tiles) {
  int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= dir.nlist) return;
  const int c = cnt[l], len = dir.len[l];
  if (c <= 0 || len <= 0) return;
  int t = tile_start[l];
  for (int p0 = 0; p0 < c; p0 += 128)
    for (int r0 = 0; r0 < len; r0 += 128) {
      LmTile tl;
      tl.list = l, tl.pair0 = start[l] + p0, tl.npairs = min(128, c - p0), tl.row0 = r0, tl.nrows = min(128, len - r0), tl.seg = 0, tl.grp = 0;
      tiles[t++] = tl;
    }
}

template <int METRIC, int EPI>
cudaError_t launch_tc(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d, float* out,
                      int64_t ldo, unsigned long long* best, cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(dist_tc_kernel<METRIC, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM);
  if (e != cudaSuccess) return e;
  const int max_rows = 65535 * TC_M;
  for (int r0 = 0; r0 < n; r0 += max_rows) {
    int nr = n - r0 < max_rows ? n - r0 : max_rows;
    dim3 grid((m + TC_N - 1) / TC_N, (nr + TC_M - 1) / TC_M);
    dist_tc_kernel<METRIC, EPI><<<grid, TC_NT, TC_SMEM, st>>>(X + (int64_t)r0 * ldx, ldx, nr, C, ldc, m, d,
                                                             out ? out + (int64_t)r0 * ldo : nullptr, ldo,
                                                             best ? best + r0 : nullptr);
    note_launch();
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace

cudaError_t launch_dist_matrix_tc(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d,
                                  int metric, float* out, int64_t ldo, cudaStream_t st) {
  if ((d & 3) || (ldx & 3) || (ldc & 3)) return cudaErrorInvalidValue;
  if (n <= 0 || m <= 0) return cudaSuccess;
  return metric == kMetricL2 ? launch_tc<kMetricL2, 0>(X, ldx, n, C, ldc, m, d, out, ldo, nullptr, st)
                             : launch_tc<kMetricIP, 0>(X, ldx, n, C, ldc, m, d, out, ldo, nullptr, st);
}

cudaError_t launch_dist_argmin_tc(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d,
                                  int metric, unsigned long long* best, cudaStream_t st) {
  if ((d & 3) || (ldx & 3) || (ldc & 3)) return cudaErrorInvalidValue;
  if (n <= 0 || m <= 0) return cudaSuccess;
  return metric == kMetricL2 ? launch_tc<kMetricL2, 1>(X, ldx, n, C, ldc, m, d, nullptr, 0, best, st)
                             : launch_tc<kMetricIP, 1>(X, ldx, n, C, ldc, m, d, nullptr, 0, best, st);
}

cudaError_t launch_ivf_listmajor_tc(const float* xq, int64_t ldq, int d, const LmTile* tiles, int ntiles,
                                    const int32_t* pair_q, const int64_t* pair_off, ListDirectory dir,
                                    const float* shifts, int metric, float* scores, cudaStream_t st) {
  if ((d & 3) || (ldq & 3)) return cudaErrorInvalidValue;
  if (ntiles <= 0) return cudaSuccess;
  cudaError_t e;
  if (metric == kMetricL2) {
    e = cudaFuncSetAttribute(ivf_listmajor_tc_kernel<kMetricL2>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM);
    if (e != cudaSuccess) return e;
    ivf_listmajor_tc_kernel<kMetricL2><<<ntiles, TC_NT, TC_SMEM, st>>>(xq, ldq, d, tiles, pair_q, pair_off, dir, shifts,
                                                                      scores);
  } else {
    e = cudaFuncSetAttribute(ivf_listmajor_tc_kernel<kMetricIP>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM);
    if (e != cudaSuccess) return e;
    ivf_listmajor_tc_kernel<kMetricIP><<<ntiles, TC_NT, TC_SMEM, st>>>(xq, ldq, d, tiles, pair_q, pair_off, dir, shifts,
                                                                      scores);
  }
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_lm_count_scan(const int32_t* probe_ids, int64_t npairs, ListDirectory dir, int32_t* cnt,
                                 int32_t* start, int64_t* base_off, int32_t* tile_start, int64_t* totals,
                                 cudaStream_t st) {
  if (npairs <= 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(cnt, 0, sizeof(int32_t) * dir.nlist, st);
  if (e != cudaSuccess) return e;
  lm_count_kernel<<<(unsigned)((npairs + 255) / 256), 256, 0, st>>>(probe_ids, npairs, dir, cnt);
  note_launch();
  lm_scan_kernel<<<1, 1024, 0, st>>>(cnt, dir, start, base_off, tile_start, totals);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_lm_assign_tiles(const int32_t* probe_ids, int64_t npairs, int nprobe, ListDirectory dir,
                                   const int32_t* cnt, const int32_t* start, int32_t* cursor, const int64_t* base_off,
                                   const int32_t* tile_start, int32_t* pair_q, int64_t* pair_off, int64_t* seg_off,
                                   LmTile* tiles, cudaStream_t st) {
  if (npairs <= 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(cursor, 0, sizeof(int32_t) * dir.nlist, st);
  if (e != cudaSuccess) return e;
  lm_assign_kernel<<<(unsigned)((npairs + 255) / 256), 256, 0, st>>>(probe_ids, npairs, nprobe, dir, start, cursor, base_off,
                                                                    pair_q, pair_off, seg_off);
  note_launch();
  lm_tiles_kernel<<<(dir.nlist + 255) / 256, 256, 0, st>>>(cnt, start, tile_start, dir, tiles);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_lmk_group(const int32_t* probe_ids, int64_t npairs, ListDirectory dir, int nseg_max, int gsize, int32_t* cnt,
                             int32_t* start, int32_t* cursor, int32_t* item_start, int32_t* grp_start, int64_t* totals,
                             int64_t* pair_j, LmTile* items, cudaStream_t st) {
  if (npairs <= 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(cnt, 0, sizeof(int32_t) * dir.nlist, st);
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(cursor, 0, sizeof(int32_t) * dir.nlist, st);
  if (e != cudaSuccess) return e;
  const unsigned nb = (unsigned)((npairs + 255) / 256);
  lm_count_kernel<<<nb, 256, 0, st>>>(probe_ids, npairs, dir, cnt);
  note_launch();
  lmk_scan_kernel<<<1, 1024, 0, st>>>(cnt, dir, nseg_max, gsize, start, item_start, grp_start, totals);
  note_launch();
  lmk_assign_kernel<<<nb, 256, 0, st>>>(probe_ids, npairs, dir, start, cursor, pair_j);
  note_launch();
  lmk_items_kernel<<<(dir.nlist + 255) / 256, 256, 0, st>>>(cnt, start, item_start, grp_start, dir, nseg_max, gsize, items);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_list_shifts(const float* cent, int64_t ldc, int nlist, int d, float* shifts, cudaStream_t st) {
  if (nlist <= 0) return cudaSuccess;
  if (d <= 0 || ldc < d) return cudaErrorInvalidValue;
  list_shift_kernel<<<nlist, 256, 0, st>>>(cent, ldc, nlist, d, shifts);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_tc_mirror_build(ListDirectory dir, int d, int k16, const int64_t* tile0, int64_t total_tiles,
                                   const float* shifts, float* mirror, float* norms, cudaStream_t st) {
  if (total_tiles <= 0) return cudaSuccess;
  if (total_tiles > INT32_MAX || (d & 3) || (k16 % TC_BK)) return cudaErrorInvalidValue;
  tc_mirror_build_kernel<<<(unsigned)total_tiles, TC_N, 0, st>>>(dir, d, k16, tile0, shifts, mirror, norms);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_tc_mirror_append(const float* x, int64_t ldx, int64_t n, int d, int k16, const int32_t* list,
                                    const int32_t* pos, const int64_t* tile0, const float* shifts, float* mirror,
                                    float* norms, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  tc_mirror_append_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(x, ldx, n, d, k16, list, pos, tile0, shifts, mirror,
                                                                       norms);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_lm_stage_queries(const float* xq, int64_t ldq, int d, int k16, const LmTile* items, int max_items,
                                    const int64_t* totals, const int64_t* pair_j, int nprobe, const float* shifts,
                                    float* a_scratch, float* a_norms, cudaStream_t st) {
  if (max_items <= 0) return cudaSuccess;
  lm_stage_queries_kernel<<<max_items, TC_M, 0, st>>>(xq, ldq, d, k16, items, totals, pair_j, nprobe, 0, shifts, a_scratch,
                                                      a_norms);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_tc_stage_rows(const float* x, int64_t ldx, int64_t n, int d, int k16, float* tiles, float* norms,
                                 cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  if ((d & 3) || (ldx & 3) || (k16 % TC_BK) || k16 < d) return cudaErrorInvalidValue;
  lm_stage_queries_kernel<<<(unsigned)((n + TC_M - 1) / TC_M), TC_M, 0, st>>>(x, ldx, d, k16, nullptr, nullptr, nullptr, 1, n,
                                                                              nullptr, tiles, norms);
  note_launch();
  return cudaGetLastError();
}

// the fused coarse quantiser's split: G CTAs (one per SM, at least CK_MIN_TILES tile pairs each) and the most CTAs
// that share one query tile (its partial sets)
struct CkGeometry {
  int nqt, ntc, G, nparts;
  int64_t W;
};
static CkGeometry ck_geometry(int nq, int nlist, int nsm) {
  CkGeometry g;
  g.nqt = (nq + TC_M - 1) / TC_M;
  g.ntc = (nlist + TC_N - 1) / TC_N;
  g.W = (int64_t)g.nqt * g.ntc;
  g.G = (int)std::max<int64_t>(1, std::min<int64_t>(nsm, g.W / CK_MIN_TILES));
  g.nparts = 1;
  for (int qt = 0; qt < g.nqt; qt++) {
    const int64_t w = (int64_t)qt * g.ntc;
    g.nparts = std::max(g.nparts, ck_owner(w + g.ntc - 1, g.W, g.G) - ck_owner(w, g.W, g.G) + 1);
  }
  return g;
}

// workspace: tau_g[nq], the partial sets, cnt[nqt]
static size_t ck_part_keys(const CkGeometry& g, int k) { return (size_t)g.nqt * g.nparts * ck_tpq(k) * k * TC_M; }

size_t coarse_topk_workspace_bytes(int nq, int nlist, int k, int nsm) {
  if (nq <= 0 || nlist <= 0 || k <= 0) return 0;
  const CkGeometry g = ck_geometry(nq, nlist, nsm);
  return ((size_t)nq + ck_part_keys(g, k)) * 8 + (size_t)g.nqt * 4;
}

template <int METRIC, int TPQ>
static cudaError_t launch_coarse_topk_t(const float* a_tiles, const float* a_norms, int nq, const float* c_tiles,
                                        const float* c_norms, int nlist, int k16, int k, const CkGeometry& g, void* ws,
                                        unsigned long long* out, cudaStream_t st) {
  unsigned long long* tau_g = static_cast<unsigned long long*>(ws);
  unsigned long long* part = tau_g + nq;
  unsigned int* cnt = reinterpret_cast<unsigned int*>(part + ck_part_keys(g, k));
  const int n = std::max(nq, g.nqt);
  coarse_init_kernel<<<(n + 255) / 256, 256, 0, st>>>(tau_g, nq, cnt, g.nqt);
  note_launch();
  const size_t smem = (size_t)CK_NST * TC_STAGE_BYTES + CK_SCORE_BYTES + (size_t)k * TC_M * TPQ * 8;
  cudaError_t e = cudaFuncSetAttribute(coarse_topk_kernel<METRIC, TPQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  coarse_topk_kernel<METRIC, TPQ><<<g.G, ck_nt<TPQ>(), smem, st>>>(a_tiles, a_norms, nq, c_tiles, c_norms, nlist, k16, k,
                                                                   g.nparts, tau_g, cnt, part, out);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_coarse_topk(const float* a_tiles, const float* a_norms, int nq, const float* c_tiles, const float* c_norms,
                               int nlist, int k16, int metric, int k, int nsm, void* ws, unsigned long long* out,
                               cudaStream_t st) {
  if (k <= 0 || k > kCoarseMaxK || k16 <= TC_BK || (k16 % TC_BK) || nsm <= 0) return cudaErrorInvalidValue;
  if (nq <= 0 || nlist <= 0) return cudaSuccess;
  const CkGeometry g = ck_geometry(nq, nlist, nsm);
  if (ck_tpq(k) == 2)
    return metric == kMetricL2
               ? launch_coarse_topk_t<kMetricL2, 2>(a_tiles, a_norms, nq, c_tiles, c_norms, nlist, k16, k, g, ws, out, st)
               : launch_coarse_topk_t<kMetricIP, 2>(a_tiles, a_norms, nq, c_tiles, c_norms, nlist, k16, k, g, ws, out, st);
  return metric == kMetricL2
             ? launch_coarse_topk_t<kMetricL2, 1>(a_tiles, a_norms, nq, c_tiles, c_norms, nlist, k16, k, g, ws, out, st)
             : launch_coarse_topk_t<kMetricIP, 1>(a_tiles, a_norms, nq, c_tiles, c_norms, nlist, k16, k, g, ws, out, st);
}

template <int METRIC>
static cudaError_t launch_tma_t(const float* a_scratch, const float* a_norms, TcMirrorView mv, const LmTile* items,
                                int max_items, const int64_t* totals, const int64_t* pair_j, int nprobe, ListDirectory dir,
                                int k, int nseg_max, FilterArgs f, unsigned long long* tau_g, unsigned long long* out,
                                cudaStream_t st) {
  const size_t smem = (size_t)LT_RING + kSlabBytes + (size_t)k * TC_NT * 8;
  cudaError_t e = cudaFuncSetAttribute(ivf_listmajor_tma_kernel<METRIC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
  ivf_listmajor_tma_kernel<METRIC><<<max_items, LT_NT, smem, st>>>(a_scratch, a_norms, mv, items, totals, pair_j, nprobe, dir,
                                                                  k, nseg_max, f, tau_g, out);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_ivf_listmajor_tma(const float* a_scratch, const float* a_norms, TcMirrorView mv, const LmTile* items,
                                     int max_items, const int64_t* totals, const int64_t* pair_j, int nprobe,
                                     ListDirectory dir, int k, int nseg_max, int metric, FilterArgs f,
                                     unsigned long long* tau_g, unsigned long long* out, cudaStream_t st) {
  if (k <= 0 || k > kLmkMaxK || mv.k16 <= TC_BK || (mv.k16 % TC_BK)) return cudaErrorInvalidValue;
  if (max_items <= 0) return cudaSuccess;
  if (metric == kMetricL2)
    return launch_tma_t<kMetricL2>(a_scratch, a_norms, mv, items, max_items, totals, pair_j, nprobe, dir, k, nseg_max, f,
                                   tau_g, out, st);
  return launch_tma_t<kMetricIP>(a_scratch, a_norms, mv, items, max_items, totals, pair_j, nprobe, dir, k, nseg_max, f, tau_g,
                                 out, st);
}

cudaError_t launch_ivf_listmajor_pipe(const float* xq, int64_t ldq, int d, const LmTile* items, int max_items,
                                      const int64_t* totals, const int64_t* pair_j, int nprobe, ListDirectory dir,
                                      const float* shifts, int k, int nseg_max, int metric, FilterArgs f,
                                      unsigned long long* tau_g, unsigned long long* out, cudaStream_t st) {
  if ((d & 3) || (ldq & 3) || k <= 0 || k > kLmkMaxK) return cudaErrorInvalidValue;
  if (max_items <= 0) return cudaSuccess;
  const size_t smem = (size_t)LW_RING + kSlabBytes + (size_t)k * TC_NT * 8;
  cudaError_t e;
  if (metric == kMetricL2) {
    e = cudaFuncSetAttribute(ivf_listmajor_pipe_kernel<kMetricL2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    ivf_listmajor_pipe_kernel<kMetricL2><<<max_items, LW_NT, smem, st>>>(xq, ldq, d, items, totals, pair_j, nprobe, dir,
                                                                        shifts, k, nseg_max, f, tau_g, out);
  } else {
    e = cudaFuncSetAttribute(ivf_listmajor_pipe_kernel<kMetricIP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    ivf_listmajor_pipe_kernel<kMetricIP><<<max_items, LW_NT, smem, st>>>(xq, ldq, d, items, totals, pair_j, nprobe, dir,
                                                                        shifts, k, nseg_max, f, tau_g, out);
  }
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_seg_select(const float* scores, const int64_t* seg_off, const int32_t* probe_ids, int nq, int nprobe,
                              ListDirectory dir, int k, int metric, FilterArgs f, unsigned long long* out_keys,
                              cudaStream_t st) {
  if (nq <= 0) return cudaSuccess;
  if (k <= 0 || k > 4096) return cudaErrorInvalidValue;
  const int KP = next_pow2(k < 16 ? 16 : k);
  const int SORTN = next_pow2(KP + 2 * SEG_NT * SEG_ITEMS);
  const size_t smem = (size_t)SORTN * 8;
  cudaError_t e;
  if (metric == kMetricL2) {
    e = cudaFuncSetAttribute(seg_select_kernel<kMetricL2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    seg_select_kernel<kMetricL2><<<nq, SEG_NT, smem, st>>>(scores, seg_off, probe_ids, nprobe, dir, k, KP, SORTN, f, out_keys);
  } else {
    e = cudaFuncSetAttribute(seg_select_kernel<kMetricIP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    seg_select_kernel<kMetricIP><<<nq, SEG_NT, smem, st>>>(scores, seg_off, probe_ids, nprobe, dir, k, KP, SORTN, f, out_keys);
  }
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
