// K5, list-major: the IVF-PQ ADC scan of a large query batch as a filtered tensor-core contraction.
//
// Reference semantics: GammaIVFPQScanner::scan_list_with_table (index/impl/gamma_index_ivfpq.h:923-953)
// driven by search_preassigned (gamma_index_ivfpq.cc:730-947): per (query, probed list, entry)
//     dis = dis0 + sum_m tab[m][code[m]],   tab = T[list] - 2 ip[query]   (L2, precomputed-table form)
//     dis = <x, centroid> + sum_m ip[query][m][code[m]]                    (inner product)
// and the k' best (k' = recall_num or k) survive.  The query-major list scan (list_scan.cuh) evaluates that
// sum literally, 16 shared-memory gathers per (query, entry): it is bound by instruction issue and
// LDS wavefronts, not by HBM.  When every list is probed by dozens of queries of the same batch the
// same numbers are a dense contraction:
//     sum_m tab[m][code[m]] = |r_e|^2 - 2 <x - c_list, r_e>,   r_e = the entry's PQ reconstruction,
// i.e. (query, list) pairs x decoded entries.  This file computes THAT with wgmma on int8 operands (exact s32 sums) and uses it
// only as a FILTER; every number that leaves the pipeline is recomputed with the reference's own
// arithmetic, so results stay bit-identical to the LUT kernel and to the oracle:
//
//   phase A  the exact LUT kernel scans each query's leading probes in full (the fewest whose lists hold
//            >= 4 k' entries, pqtc_plan_phase_a_kernel) and yields k' exact keys, unordered, the largest --
//            B_q, an upper bound of the query's final k'-th score -- in slot k' - 1;
//   phase B  (this file) for the remaining probes: pairs grouped by list (lmk_group), per group an
//            int8 operand tile of rn((x - c_list) / sa) rows staged once (pq_stage_pairs_kernel), then a
//            persistent warp-specialised kernel (pqtc_scan_kernel) decodes 128 entries at a time
//            from their codes into the second operand (int8 codebook rn(pq / sb) in shared memory),
//            multiplies up to 256 pairs x 128 entries x d on the tensor core (two consumer warpgroups of 128
//            pairs share each decoded tile) and compares
//            |r_e|^2 - 2 sa sb acc against  B_q - dis0 + eps(pair).  eps bounds |approximate - reference fp32|
//            rigorously (int8 quantisation of both operands, Cauchy-Schwarz over the quantisation errors; fp32
//            noise of both evaluations), so every entry whose reference score is <= B_q passes.  |r_e|^2 comes from a per-entry cache
//            in HBM (pq_entry_norms_kernel), streamed with the codes.  Passing entries (a few per query)
//            go through a shared-memory queue to a drain warp that appends (probe, position) to the
//            query's candidate list, so no global atomic sits in the epilogue;
//   phase C  pq_rescore_kernel re-evaluates the candidates with the reference arithmetic (same
//            fmaf / add order as the LUT kernel), merges them with phase A's keys and keeps k'.
//   A query whose candidate list overflows (no usable bound, adversarial data) is redone by the
//   exact kernel over all its probes (flag-gated launch), so the result never depends on the filter.
//
// Operand layout: canonical no-swizzle K-major tiles of int8 (8-row x 16-byte core matrices,
// LBO 2048 = next core matrix along K, SBO 128 = next 8 rows).  A centroid is dsub bytes: with dsub = 8
// two sub-quantisers fill one 16-byte core-matrix row (2 x LDS.64 from the codebook, one STS.128 into
// the tile), conflict-free on the store side (consecutive entries -> consecutive rows).
//
// Algorithmic bytes: (M + 8) per scanned entry per 256-pair group instead of per pair.
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"

namespace gb {

namespace {

constexpr int PT_M = 128;          // pairs per warpgroup (MMA M: two m64 halves) = rows of one A operand tile
constexpr int PT_G = 2 * PT_M;     // pairs per group: two consumer warpgroups share each decoded B tile
constexpr int PT_N = 128;          // entries per tile (MMA N, accumulator columns)
// warpgroups 0-1 MMA + epilogue (pairs 0-127 / 128-255 of the group), 2 decode, 3: warp 12 TMA producer,
// warp 13 candidate drain, warps 14-15 idle (setmaxnreg works per warpgroup)
constexpr int PT_NT = 512;
constexpr int PT_REG_MMA = 192, PT_REG_OTHER = 64;  // 2 x 128 x (192 + 64) = the 64 K registers of the SM
constexpr int PT_RQ = 512;         // records of the CTA's candidate queue (shared memory)
constexpr unsigned long long kRecEmpty = ~0ull;
constexpr int PT_CS = 4;           // code stages
constexpr int PT_KSUB = 256;

struct PtShared {
  uint64_t code_full[PT_CS], code_empty[PT_CS];
  uint64_t b_full[2], b_empty[2], a_full[2], a_empty[2], acc_empty[2];
  alignas(16) float ne[2][PT_N];  // |r_e|^2 of the tile's entries, +inf = can never be returned
  alignas(16) float ne_min[2][PT_N / 32];  // min of ne over each decode warp's 32 entries (columns 32 g .. 32 g + 31)
  // candidate queue: the epilogue warps append (query, probe, position) records with shared-memory atomics and move on;
  // the drain warp turns them into the global per-query lists.  A global atomicAdd-with-return costs ~1 us of latency:
  // issued from the epilogue it stalled the whole pipeline as soon as a loose bound let a percent of the entries through.
  unsigned int q_head, q_tail;
  int q_done;
  unsigned long long q_rec[PT_RQ];  // (q << 48 | p << 32 | pos), kRecEmpty = free slot
};

// ---- tables derived from the PQ codebook ---------------------------------------------------------
// sb = max |pq| / 127 (one scale for the whole codebook); cb[m][c][0..dsub) = int8 rn(pq[m][c][.] / sb);
// nrm[m][c] = |pq[m][c]|^2 (fp32, L2 only); rmax2[0] = R^2 = sum_m max_c |pq[m][c]|^2, rmax2[1] = sb (0 when the codebook
// is all zero or not finite: no filter), rmax2[2] = D = sqrt(sum_m max_c |pq[m][c] - sb cb[m][c]|^2), the largest
// quantisation error of a reconstruction   (single CTA of 256 threads)
__global__ void __launch_bounds__(256)
    pqtc_tables_kernel(const float* __restrict__ pq, int M, int dsub, int8_t* __restrict__ cb, float* __restrict__ nrm,
                       float* __restrict__ rmax2) {
  __shared__ float s_max[256], s_err[256];
  const int c = threadIdx.x;
  float mx = 0.f;
  for (int i = c; i < M * PT_KSUB * dsub; i += 256) mx = fmaxf(mx, fabsf(pq[i]));
  s_max[c] = mx;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (c < off) s_max[c] = fmaxf(s_max[c], s_max[c + off]);
    __syncthreads();
  }
  const float cbmax = s_max[0];
  const bool ok = cbmax > 0.f && cbmax < INFINITY;
  const float sb = ok ? cbmax / 127.f : 0.f, inv = ok ? 127.f / cbmax : 0.f;
  __syncthreads();
  float total = 0.f, err = 0.f;
  for (int m = 0; m < M; m++) {
    const float* p = pq + ((int64_t)m * PT_KSUB + c) * dsub;
    float n2 = 0.f, e2 = 0.f;
    for (int j = 0; j < dsub; j++) {
      const float v = p[j];
      n2 = fmaf(v, v, n2);
      const int qv = max(-127, min(127, __float2int_rn(v * inv)));
      const float dv = v - sb * (float)qv;
      e2 = fmaf(dv, dv, e2);
      cb[((int64_t)m * PT_KSUB + c) * dsub + j] = (int8_t)qv;
    }
    nrm[m * PT_KSUB + c] = n2;
    s_max[c] = n2, s_err[c] = e2;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
      if (c < off) s_max[c] = fmaxf(s_max[c], s_max[c + off]), s_err[c] = fmaxf(s_err[c], s_err[c + off]);
      __syncthreads();
    }
    total += s_max[0], err += s_err[0];
    __syncthreads();
  }
  if (threadIdx.x == 0) rmax2[0] = total, rmax2[1] = sb, rmax2[2] = sqrtf(err);
}

// ---- phase A's plan ---------------------------------------------------------------------------------------------------
// Query q's phase A scans its first P_q probes IN FULL: the fewest whose lists hold >= target entries together, at most
// pa_max.  probes_a / probes_b = probe_ids with the other phase's probes set to -1 ("no list", skipped by both scans);
// row_limit[q][p] = rows of probe p phase A scores exactly (the whole list, or 0).  A tight bound matters far more than
// a cheap phase A: bounding from a PREFIX of the nearest list instead of the whole list multiplies the candidates and
// slows the filter kernel (DESIGN.md section 3).
__global__ void pqtc_plan_phase_a_kernel(const int32_t* __restrict__ probe_ids, int64_t npairs, int nprobe, int pa_max,
                                         long long target, const int* __restrict__ list_len, int32_t* __restrict__ probes_a,
                                         int32_t* __restrict__ probes_b, int* __restrict__ row_limit) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= npairs) return;
  const int64_t q = j / nprobe;
  const int p = (int)(j - q * nprobe);
  const int32_t* row = probe_ids + q * nprobe;
  int P = pa_max;
  long long cum = 0;
  for (int i = 0; i < pa_max; i++) {
    const int l = row[i];
    if (l >= 0) cum += list_len[l];
    if (cum >= target) {
      P = i + 1;
      break;
    }
  }
  const int32_t id = row[p];
  const bool in_a = p < P;
  probes_a[j] = in_a ? id : -1;
  probes_b[j] = in_a ? -1 : id;
  row_limit[j] = in_a && id >= 0 ? list_len[id] : 0;
}

// ---- per pair group: the A operand tile and the pairs' thresholds ---------------------------------
// The accumulator of pair (query, list) and entry e is the exact integer acc = <qa, qr_e>, biased by kAccBias: its bits
// read as a float are 12582912 + acc exactly (|acc| <= 127^2 d < 2^22).  The filter evaluates v = ne * c - (bias + acc)
// = (ne - f s acc) / (f s) - bias with one fma, f = 2 (L2) / 1 (IP), s = sa sb; v <= thr passes.
constexpr uint32_t kAccBias = 0x4B400000u;  // 1.5 * 2^23: floats in [2^23, 2^24) step by 1 per unit of their bits
constexpr double kAccBiasF = 12582912.0;

struct PairMeta {
  float thr;  // candidate  <=>  v = fma(ne, c, -(bias + acc)) <= thr
  float lo;   // ... and v >= lo  (the other side of the score window, checked on the rare path)
  float c;    // 1 / (f sa sb): accumulator units per score unit
  int q, p;
  int lim;    // rows [0, lim) of this pair's list were scored exactly by phase A: never candidates
};

// What the threshold of a pair needs besides the bound B_q, in double: eps (the error margin in score units) and fs = f s
// (score units per accumulator unit).  fs = 0: the pair has no filter test (an empty row, or one already sent to the
// exact kernel while staging).  A filtered pair has fs > 0: a_ok and sb > 0, and a subnormal sa would make the row tiny.
struct PairBound {
  double eps, fs;
};

// A group of up to PT_G pairs is staged as two stacked 128-row tiles, one per consumer warpgroup; its pairs are split
// evenly over the two (the first ceil(n / 2) in tile 0), so neither runs a mostly empty remainder.  Thread r = row r % 128
// of tile r / 128; meta[grp * PT_G + r] is that row's pair.  Nothing here reads phase A's keys, so the staging runs
// beside phase A; pq_bind_bounds_kernel sets thr from B_q afterwards (thr = -inf until then).
template <int METRIC>
__global__ void __launch_bounds__(PT_G)
    pq_stage_pairs_kernel(const float* __restrict__ xq, int64_t ldq, int d, const float* __restrict__ coarse, int64_t ldc,
                          const LmTile* __restrict__ items, const int64_t* __restrict__ totals,
                          const int64_t* __restrict__ pair_j, int nprobe, const float* __restrict__ coarse_dis,
                          const float* __restrict__ rmax2, float min_score, float max_score,
                          unsigned char* __restrict__ a_scratch, PairMeta* __restrict__ meta,
                          PairBound* __restrict__ bounds, int* __restrict__ cand_cnt, int cap,
                          const int* __restrict__ row_limit) {
  if ((int64_t)blockIdx.x >= totals[1]) return;
  const LmTile t = items[blockIdx.x];
  if (t.seg != 0) return;  // one staging per pair group: the first item of the group owns the slot
  const int h = threadIdx.x / PT_M, r = threadIdx.x % PT_M;
  const int n0 = (t.npairs + 1) / 2;  // pairs of tile 0
  const int kc_n = d / 16;
  unsigned char* tile = a_scratch + ((int64_t)t.grp * 2 + h) * ((int64_t)kc_n * 2048);
  PairMeta pm{-INFINITY, INFINITY, 1.0f, -1, 0, 0};
  const float* x = nullptr;
  const float* c = nullptr;
  if (r < (h ? t.npairs - n0 : n0)) {
    const int64_t j = pair_j[t.pair0 + h * n0 + r];
    pm.q = (int)(j / nprobe);
    pm.p = (int)(j - (int64_t)pm.q * nprobe);
    x = xq + (int64_t)pm.q * ldq;
    c = coarse + (int64_t)t.list * ldc;
  }
  // the row a = x - c (L2) / x (IP), 16 components (one core-matrix row of int8) at a time
  auto load16 = [&](int kc, float (&a)[16]) {
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + kc * 16 + 4 * u));
      a[4 * u] = v.x, a[4 * u + 1] = v.y, a[4 * u + 2] = v.z, a[4 * u + 3] = v.w;
    }
  };
  // pass 1: norms and the largest component of a
  float na2 = 0.f, nx2 = 0.f, nc2 = 0.f, amax = 0.f;
  if (x) {
    for (int kc = 0; kc < kc_n; kc++) {
      float a[16];
      load16(kc, a);
      if (METRIC == kMetricL2) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const float4 cv = __ldg(reinterpret_cast<const float4*>(c + kc * 16 + 4 * u));
          const float cc[4] = {cv.x, cv.y, cv.z, cv.w};
#pragma unroll
          for (int v = 0; v < 4; v++) {
            nx2 = fmaf(a[4 * u + v], a[4 * u + v], nx2);
            nc2 = fmaf(cc[v], cc[v], nc2);
            a[4 * u + v] -= cc[v];
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 16; u++) na2 = fmaf(a[u], a[u], na2), amax = fmaxf(amax, fabsf(a[u]));
    }
  }
  // pass 2: qa = rn(a / sa), sa = amax / 127, as int8 in the canonical K-major operand layout; da2 = |a - sa qa|^2
  const bool a_ok = amax > 0.f && amax < INFINITY;
  const float sa = a_ok ? amax / 127.f : 0.f, inv = a_ok ? 127.f / amax : 0.f;
  float da2 = 0.f;
  for (int kc = 0; kc < kc_n; kc++) {
    uint32_t wv[4] = {0u, 0u, 0u, 0u};
    if (x) {
      float a[16];
      load16(kc, a);
      if (METRIC == kMetricL2) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const float4 cv = __ldg(reinterpret_cast<const float4*>(c + kc * 16 + 4 * u));
          a[4 * u] -= cv.x, a[4 * u + 1] -= cv.y, a[4 * u + 2] -= cv.z, a[4 * u + 3] -= cv.w;
        }
      }
#pragma unroll
      for (int u = 0; u < 16; u++) {
        const int qv = max(-127, min(127, __float2int_rn(a[u] * inv)));
        const float dv = a[u] - sa * (float)qv;
        da2 = fmaf(dv, dv, da2);
        wv[u >> 2] |= ((uint32_t)qv & 0xFFu) << (8 * (u & 3));
      }
    }
    *reinterpret_cast<uint4*>(tile + (int64_t)kc * 2048 + r * 16) = make_uint4(wv[0], wv[1], wv[2], wv[3]);
  }
  PairBound pb{0.0, 0.0};
  if (x) {
    const float dis0 = coarse_dis[(int64_t)pm.q * nprobe + pm.p];
    pm.lim = row_limit ? row_limit[(int64_t)pm.q * nprobe + pm.p] : 0;
    const float R2 = rmax2[0], R = sqrtf(R2), sb = rmax2[1], Dq = rmax2[2];
    // eps below has relative terms only.  Near fp32's subnormal range (|a|^2 or the codebook's largest |r|^2 below
    // 2^-96) the roundings of the exact table evaluation are absolute (2^-149 each) and can exceed it: no filter there.
    // A zero or non-finite row or codebook has no int8 scale: no filter either
    const bool tiny = (amax > 0.f && na2 < 0x1p-96f) || (R2 > 0.f && R2 < 0x1p-96f);
    if (tiny || !a_ok || !(sb > 0.f && sb < INFINITY)) {
      // the bound would not hold -> the exact kernel redoes this query
      atomicMax(cand_cnt + pm.q, cap + 1);
    } else {
      // |<a, r> - s <qa, qr>| = |<da, r> + <sa qa, dr>| <= |da| R + (|a| + |da|) D   (Cauchy-Schwarz; da = a - sa qa,
      //   dr = r - sb qr, |r| <= R and |dr| <= D for every entry, s = sa sb, the products s <qa, qr> are exact integers
      //   times s); the 5 % slack covers the fp32 roundings of |a|, |da|, R and D.  Scores scale it by f = 2 (L2) / 1 (IP).
      // + fp32 noise of the reference evaluation, bounded by 2^-17 of the magnitudes that enter it
      // + the filter's own fp32: v = fma(ne, c, -(bias + acc)) rounds once at magnitude < 2^24 + ne c (<= 1 unit of
      //   1 / (f s), i.e. f s in score units, plus 2^-24 ne) and c = fl(1 / (f s)) is off by 2^-24 relative (2^-24 ne)
      const double na = sqrt((double)na2), da = sqrt((double)da2), s = (double)sa * (double)sb;
      const double f = METRIC == kMetricL2 ? 2.0 : 1.0;
      const double quant = f * 1.05 * (da * R + (na + da) * Dq);
      double eps, lo;
      if (METRIC == kMetricL2) {
        const double Z = fabs((double)dis0) + R2 + 2.0 * (sqrt((double)nx2) + sqrt((double)nc2)) * R;
        eps = quant + 0x1p-17 * Z + f * s + 0x1p-22 * R2;
        lo = (double)min_score - dis0 - eps;
      } else {
        // score = dis0 + s acc; better = larger, so the test runs on -s acc
        const double Z = fabs((double)dis0) + na * R;
        eps = quant + 0x1p-17 * Z + f * s;
        lo = (double)dis0 - max_score - eps;
      }
      // in accumulator units, rounded outwards (thr: pq_bind_bounds_kernel)
      const double fs = f * s;
      pm.c = (float)(1.0 / fs);
      pm.lo = __double2float_rd(lo / fs - kAccBiasF);
      pb = {eps, fs};
    }
  }
  const int64_t slot = (int64_t)t.grp * PT_G + threadIdx.x;
  meta[slot] = pm;
  bounds[slot] = pb;
}

// One thread per pair slot, after phase A: thr from the query's bound B_q = the k'-th key of phase A (slot k' - 1).
// A query whose phase A found fewer than k' entries has no bound: its pairs get no filter test and the exact kernel
// redoes it.  Same double expressions and roundings as the staging kernel's lo, so the thresholds are exact functions
// of (B_q, dis0, eps, fs).
template <int METRIC>
__global__ void __launch_bounds__(256)
    pq_bind_bounds_kernel(const int64_t* __restrict__ totals, int64_t max_slots, int nprobe,
                          const float* __restrict__ coarse_dis, const unsigned long long* __restrict__ bound_keys,
                          int64_t bound_stride, int kprime, float min_score, float max_score,
                          const PairBound* __restrict__ bounds, PairMeta* __restrict__ meta, int* __restrict__ cand_cnt,
                          int cap) {
  const int64_t slot = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= max_slots || slot / PT_G >= totals[0]) return;  // totals[0] = pair groups staged
  const PairBound pb = bounds[slot];
  if (!(pb.fs > 0.0)) return;
  PairMeta* pm = meta + slot;
  const int q = pm->q, p = pm->p;
  const unsigned long long bk = bound_keys[(int64_t)q * bound_stride + kprime - 1];
  if (bk == kKeySentinel) {
    atomicMax(cand_cnt + q, cap + 1);
    pm->lo = INFINITY;
    pm->c = 1.0f;
    return;
  }
  const float dis0 = coarse_dis[(int64_t)q * nprobe + p];
  const float B = ord2score((uint32_t)(bk >> 32), METRIC);
  double thr;
  if (METRIC == kMetricL2)
    thr = (double)fminf(B, max_score) - dis0 + pb.eps;
  else
    thr = (double)dis0 - fmaxf(B, min_score) + pb.eps;
  // FLT_MAX keeps masked entries (ne = +inf) out
  pm->thr = fminf(__double2float_ru(thr / pb.fs - kAccBiasF), FLT_MAX);
}

// ---- the scan ---------------------------------------------------------------------------------------
// Accumulator fragments of a consumer thread: fragment index 4 j + 2 r8 + e of half u = row 64 u + 16 w + l / 4 + 8 r8,
// column 8 j + 2 (l % 4) + e (w = warp of the warpgroup, l = lane).  Its four rows f4 = 2 u + r8:
__device__ __forceinline__ int pt_frag_row(int f4, int t) { return (f4 >> 1) * 64 + (t >> 5) * 16 + ((t & 31) >> 2) + (f4 & 1) * 8; }

// rare path of the epilogue, called by a whole warp when one of its lanes has a candidate in the tile: each lane tests
// its own fragments again (the same fmaf as the fast path, now with the score window's lower side and the phase-A row
// limit) and the warp appends the hits to the CTA's queue with one shared-memory atomic.  Inlined: the fragments are
// registers, and handing them over by reference would force a local-memory copy of the accumulator in the hot loop.
__device__ __forceinline__ void pt_push_frag_hits(const uint32_t (&acc)[2][64], const float* ne, const float (&fthr)[4],
                                                  const float (&fc)[4], const PairMeta* gm, uint32_t pos0,
                                                  PtShared* sh) {
  const int t = threadIdx.x & 127, lane = t & 31;
  float lo[4];
  int lim[4];
  uint32_t mask[4];
#pragma unroll
  for (int f4 = 0; f4 < 4; f4++) {
    const PairMeta* m = gm + pt_frag_row(f4, t);
    lo[f4] = __ldg(&m->lo);
    lim[f4] = __ldg(&m->lim);
    mask[f4] = 0;
  }
  // column-outer: each |r_e|^2 is loaded once for the four rows, so only the accumulator stays live in registers
#pragma unroll
  for (int j = 0; j < PT_N / 8; j++) {
    const float2 n2 = *reinterpret_cast<const float2*>(&ne[8 * j + 2 * (lane & 3)]);
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int col = 8 * j + 2 * (lane & 3) + e;
#pragma unroll
      for (int f4 = 0; f4 < 4; f4++) {
        // ns = -v exactly (fma rounds symmetrically).  Written as the fast path's fmaf, ptxas would keep all 128 sums of
        // the fast path alive for this rarely taken path and spill them
        const float ns = fmaf(-(e ? n2.y : n2.x), fc[f4], __uint_as_float(acc[f4 >> 1][4 * j + 2 * (f4 & 1) + e]));
        // rows phase A has scored exactly stay out
        if (ns >= -fthr[f4] && ns <= -lo[f4] && (int)(pos0 + col) >= lim[f4]) mask[f4] |= 1u << (2 * j + e);
      }
    }
  }
  const int n = __popc(mask[0]) + __popc(mask[1]) + __popc(mask[2]) + __popc(mask[3]);
  int incl = n;  // warp-inclusive prefix sum of the hit counts
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  unsigned int base = 0;
  if (lane == 31 && total) base = atomicAdd(&sh->q_head, (unsigned int)total);
  unsigned int idx = __shfl_sync(0xffffffffu, base, 31) + (unsigned int)(incl - n);
#pragma unroll
  for (int f4 = 0; f4 < 4; f4++) {
    uint32_t mk = mask[f4];
    if (!mk) continue;
    const PairMeta* m = gm + pt_frag_row(f4, t);
    const unsigned long long hi = ((unsigned long long)(uint32_t)__ldg(&m->q) << 48) | ((unsigned long long)(uint32_t)__ldg(&m->p) << 32);
    while (mk) {
      const int b = __ffs(mk) - 1;
      mk &= mk - 1;
      const uint32_t col = 8 * (b >> 1) + 2 * (lane & 3) + (b & 1);
      // the slot's previous occupant (idx - PT_RQ) has been consumed once the tail has passed it
      while (idx - *reinterpret_cast<volatile unsigned int*>(&sh->q_tail) >= (unsigned int)PT_RQ) __nanosleep(32);
      *reinterpret_cast<volatile unsigned long long*>(&sh->q_rec[idx % PT_RQ]) = hi | (unsigned long long)(pos0 + col);
      idx++;
    }
  }
  __syncwarp();
}

__device__ __forceinline__ void bar_sync_256(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void bar_arrive_256(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// EAGER: tombstones and the docid predicate are resolved in the decode warps (one id + bitmap lookup per entry per
// 256 pairs) -- needed when a deletion / filter bitmap is present, because the bound B_q was taken over valid entries
// only and a selective filter would otherwise flood the candidate lists.  Without bitmaps the ids are not touched
// here at all (their DRAM latency sits on the decode warps' critical path);
// tombstoned entries that pass the filter are dropped by pq_rescore_kernel, which reads the id anyway.
template <int M, int DSUB, bool HAS_NORM, bool EAGER>
__global__ void __launch_bounds__(PT_NT, 1)
    pqtc_scan_kernel(const unsigned char* __restrict__ a_scratch, const PairMeta* __restrict__ meta,
                     const int8_t* __restrict__ cb_g, const float* __restrict__ pqnorm,
                     const int64_t* __restrict__ pqnorm_off, const LmTile* __restrict__ items,
                     const int64_t* __restrict__ totals, ListDirectory dir, FilterArgs f, int* __restrict__ cand_cnt,
                     unsigned long long* __restrict__ cand, int cap) {
  constexpr int D = M * DSUB;
  constexpr int KC = D / 16;               // core matrices (16 int8 wide) along K
  constexpr int TILE = KC * 2048;          // one 128-row operand tile, bytes
  constexpr int CB_BYTES = M * PT_KSUB * DSUB;
  // |r_e|^2 of every list entry is cached in HBM beside the lists (IVFPQIndex::ensure_pq_norms) and arrives with the
  // codes: 512 bytes per tile by TMA instead of 16 table gathers per entry in the decode warps
  constexpr int NRM_BYTES = HAS_NORM ? PT_CS * PT_N * 4 : 0;
  constexpr int CODE_STAGE = PT_N * M;
  constexpr int UNIT = DSUB;               // bytes of one centroid in the int8 codebook
  // K = 32 per MMA; |acc| <= 127^2 D < 2^22 keeps the biased accumulator exact
  static_assert(D % 32 == 0 && D <= 256 && M % 4 == 0 && (UNIT % 16 == 0 || 16 % UNIT == 0), "shape");
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ PtShared sh;
  unsigned char* cb = smem;
  float* nstage = reinterpret_cast<float*>(smem + CB_BYTES);  // [PT_CS][PT_N] norms of the staged tiles
  // [codebook][norms][A tiles: 2 items x 2 warpgroups][B tiles x 2][code stages]; the operand tiles start on 4 KiB
  // boundaries.  The A tiles are double-buffered: the producer loads item i + 1's pairs while item i's tiles run
  unsigned char* a_buf = smem + CB_BYTES + NRM_BYTES;
  a_buf += (4096u - (smem_u32(a_buf) & 4095u)) & 4095u;
  unsigned char* b_buf = a_buf + 4 * TILE;
  unsigned char* code_buf = b_buf + 2 * TILE;

  // once per CTA, before the barriers and the warp roles: the roles walk the items on their own, so none may leave
  // the schedule part way
  if (cta_cancelled(f.cancel, kCsPqtcScan)) return;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int64_t n_items = totals[1];

  if (tid == 0) {
    for (int s = 0; s < PT_CS; s++) {
      mbar_init(&sh.code_full[s], 1);       // producer's arrive.expect_tx; the bulk copy completes the phase
      mbar_init(&sh.code_empty[s], PT_N);   // every decode thread has read its code
    }
    for (int b = 0; b < 2; b++) {
      mbar_init(&sh.b_full[b], PT_N);       // every decode thread has written its row
      mbar_init(&sh.b_empty[b], PT_G);      // every MMA thread of both warpgroups, once its MMAs are complete
      mbar_init(&sh.acc_empty[b], PT_G);    // every epilogue thread of both warpgroups
    }
    for (int b = 0; b < 2; b++) {
      mbar_init(&sh.a_full[b], 1);          // bulk copies
      mbar_init(&sh.a_empty[b], PT_G);      // every MMA thread, after the item's last tile
    }
    mbar_fence_init();
    sh.q_head = 0, sh.q_tail = 0, sh.q_done = 0;
  }
  for (int i = tid; i < PT_RQ; i += PT_NT) sh.q_rec[i] = kRecEmpty;
  // codebook (int8): resident for the CTA's lifetime
  for (int i = tid; i < CB_BYTES / 16; i += PT_NT)
    reinterpret_cast<uint4*>(cb)[i] = __ldg(reinterpret_cast<const uint4*>(cb_g) + i);
  __syncthreads();

  if (warp < 8) {
    // ======================= MMA + epilogue: warpgroup h = pairs [128 h, 128 h + 128) of the group =======================
    // Both warpgroups multiply the same B tile and take turns on the tensor pipe (named barriers 2 and 3): warpgroup 1
    // issues tile i while warpgroup 0 tests tile i, warpgroup 0 issues tile i + 1 while warpgroup 1 tests tile i.
    setmaxnreg_inc<PT_REG_MMA>();
    const int h = warp >> 2, t = tid & 127;
    const uint32_t a_base = smem_u32(a_buf) + (uint32_t)(h * TILE), b_base = smem_u32(b_buf);
    uint32_t an = 0, bn = 0;
    bool turns = false;  // warpgroup 0 has issued a tile: from then on it waits for warpgroup 1's turn
    uint32_t acc[2][64];
    for (int64_t it = blockIdx.x; it < n_items; it += gridDim.x) {
      const LmTile tl = items[it];
      if (tl.nrows <= 0) continue;  // every role skips empty segments the same way
      const PairMeta* gm = meta + (int64_t)tl.grp * PT_G + h * PT_M;
      // thresholds of the four pairs (rows) whose accumulator fragments this thread holds
      float fthr[4], fc[4];
#pragma unroll
      for (int f4 = 0; f4 < 4; f4++) {
        const PairMeta* m = gm + pt_frag_row(f4, t);
        fthr[f4] = __ldg(&m->thr), fc[f4] = __ldg(&m->c);
      }
      const int ab = an & 1;
      mbar_wait(&sh.a_full[ab], (an >> 1) & 1);
      const int ntiles = (tl.nrows + PT_N - 1) / PT_N;
      for (int i = 0; i < ntiles; i++, bn++) {
        const int b = bn & 1;
        mbar_wait(&sh.b_full[b], (bn >> 1) & 1);
        if (h) bar_sync_256(3);
        else if (turns) bar_sync_256(2);
        // every warpgroup runs both m64 halves of every tile, empty rows included (their thresholds are -inf): a
        // branch around the MMAs or the wait makes ptxas serialise every wgmma of the kernel
        const uint64_t da = lt_desc(a_base + (uint32_t)(ab * 2 * TILE)), db = lt_desc(b_base + (uint32_t)(b * TILE));
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < KC / 2; kk++) {  // K = 32 per instruction: two core matrices = 4096 bytes further
          const uint64_t adv = (uint64_t)((kk * 4096) >> 4);
          wg_mma_s8(acc[0], da + adv, db + adv, kk != 0);
          wg_mma_s8(acc[1], da + adv + kDescHalfM, db + adv, kk != 0);
        }
        wg_commit();
        bar_arrive_256(h ? 2 : 3);
        turns = true;
        wg_wait<0>();
        wg_fence_acc(acc);
        mbar_arrive(&sh.b_empty[b]);
        if (i == ntiles - 1) mbar_arrive(&sh.a_empty[ab]);
        // Group screen: per pair and group of 32 columns (one decode warp's entries), lb = c * min ne - (bias + max acc)
        // with the same fma as the per-entry test.  Its exact argument is <= every entry's (ne >= min ne, c > 0,
        // acc <= max acc, and the biased float grows with acc), and correctly rounded fma is monotone, so lb <= v for
        // every entry of the group: a pair with some v <= thr has lb <= thr.  One integer max per element instead of an
        // add, an fma and a min; the per-entry test below runs only in warps the screen did not clear.
        const float4 nm4 = *reinterpret_cast<const float4*>(sh.ne_min[b]);
        const float nmin[4] = {nm4.x, nm4.y, nm4.z, nm4.w};
        bool maybe = false;
#pragma unroll
        for (int f4 = 0; f4 < 4; f4++) {
          float lb = INFINITY;
#pragma unroll
          for (int g = 0; g < PT_N / 32; g++) {
            int mx = (int)acc[f4 >> 1][16 * g + 2 * (f4 & 1)];
#pragma unroll
            for (int j = 4 * g; j < 4 * g + 4; j++)
#pragma unroll
              for (int e = 0; e < 2; e++) mx = max(mx, (int)acc[f4 >> 1][4 * j + 2 * (f4 & 1) + e]);
            lb = fminf(lb, fmaf(nmin[g], fc[f4], -__uint_as_float((uint32_t)mx + kAccBias)));
          }
          maybe |= lb <= fthr[f4];
        }
        if (__any_sync(0xffffffffu, maybe)) {
          // biased, the accumulators' bits are floats without a conversion (PairMeta).  (Starting the MMAs from the bias
          // instead makes ptxas serialise every wgmma of the kernel, C7520.)
#pragma unroll
          for (int u = 0; u < 2; u++)
#pragma unroll
            for (int k = 0; k < 64; k++) acc[u][k] += kAccBias;
          // min over the tile of v = c * ne - (bias + acc) per pair, on the fragments themselves.  A warp where some pair
          // has a candidate redoes the test per entry and pushes the hits (pt_push_frag_hits).
          float mn[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
#pragma unroll
          for (int j = 0; j < PT_N / 8; j++) {
            const float2 n2 = *reinterpret_cast<const float2*>(&sh.ne[b][8 * j + 2 * (t & 3)]);
#pragma unroll
            for (int f4 = 0; f4 < 4; f4++) {
              const uint32_t* a2 = &acc[f4 >> 1][4 * j + 2 * (f4 & 1)];
              mn[f4] = fminf(mn[f4], fminf(fmaf(n2.x, fc[f4], -__uint_as_float(a2[0])), fmaf(n2.y, fc[f4], -__uint_as_float(a2[1]))));
            }
          }
          bool hit = false;
#pragma unroll
          for (int f4 = 0; f4 < 4; f4++) hit |= mn[f4] <= fthr[f4];
          if (__any_sync(0xffffffffu, hit)) pt_push_frag_hits(acc, sh.ne[b], fthr, fc, gm, (uint32_t)(tl.row0 + i * PT_N), &sh);
        }
        mbar_arrive(&sh.acc_empty[b]);
      }
      an++;
    }
    if (h == 0 && turns) bar_sync_256(2);  // warpgroup 1's arrival after its last tile
    __syncwarp();
    if ((tid & 31) == 0) {
      __threadfence_block();
      atomicAdd(&sh.q_done, 1);  // this warp's records are all in the queue
    }
  } else if (warp < 12) {
    // ======================= decode: thread = entry of the tile =======================
    setmaxnreg_dec<PT_REG_OTHER>();
    const int e = tid - 8 * 32;
    uint32_t cn = 0, bn = 0;
    for (int64_t it = blockIdx.x; it < n_items; it += gridDim.x) {
      const LmTile t = items[it];
      const int64_t* __restrict__ lids = dir.ids[t.list];
      const int row_end = t.row0 + t.nrows;
      const int ntiles = (t.nrows + PT_N - 1) / PT_N;
      for (int i = 0; i < ntiles; i++, cn++, bn++) {
        const int s = cn % PT_CS;
        mbar_wait(&sh.code_full[s], (cn / PT_CS) & 1);
        uint32_t w[M / 4];
        {
          const unsigned char* cp = code_buf + s * CODE_STAGE + e * M;
          if (M % 16 == 0) {
#pragma unroll
            for (int u = 0; u < M / 16; u++) {
              const uint4 q4 = reinterpret_cast<const uint4*>(cp)[u];
              w[4 * u] = q4.x, w[4 * u + 1] = q4.y, w[4 * u + 2] = q4.z, w[4 * u + 3] = q4.w;
            }
          } else if (M % 8 == 0) {
#pragma unroll
            for (int u = 0; u < M / 8; u++) {
              const uint2 q2 = reinterpret_cast<const uint2*>(cp)[u];
              w[2 * u] = q2.x, w[2 * u + 1] = q2.y;
            }
          } else {
#pragma unroll
            for (int u = 0; u < M / 4; u++) w[u] = reinterpret_cast<const uint32_t*>(cp)[u];
          }
        }
        const float nstaged = HAS_NORM ? nstage[s * PT_N + e] : 0.f;
        mbar_arrive(&sh.code_empty[s]);
        // entries past the end of the segment decode whatever bytes the stage holds: finite values,
        // masked by ne = +inf.  Tombstones (gamma_index_ivfpq.h:930) and the docid predicate
        // (IsValid, :934-939) are resolved here, once per entry per 256 pairs.
        const int row = t.row0 + i * PT_N + e;
        bool valid = row < row_end;
        if (EAGER && valid) {
          const int64_t raw = lids[row];
          valid = raw >= 0 && ctx_is_valid(f.del_bits, f.filter_bits, (uint32_t)raw);
        }
        const int b = bn & 1;
        mbar_wait(&sh.b_empty[b], ((bn >> 1) & 1) ^ 1);
        unsigned char* brow = b_buf + b * TILE + e * 16;
        const float nsum = nstaged;
        auto centroid = [&](int m) { return cb + (m * PT_KSUB + ((w[m >> 2] >> (8 * (m & 3))) & 0xFFu)) * UNIT; };
        // one 16-byte core-matrix row per step: 16 / UNIT centroids (UNIT = 4, 8) or a 16-byte piece of one (16, 32)
#pragma unroll
        for (int kc = 0; kc < KC; kc++) {
          uint4 val;
          if constexpr (UNIT >= 16) {
            val = reinterpret_cast<const uint4*>(centroid(kc / (UNIT / 16)))[kc % (UNIT / 16)];
          } else if constexpr (UNIT == 8) {
            const uint2 v0 = *reinterpret_cast<const uint2*>(centroid(2 * kc));
            const uint2 v1 = *reinterpret_cast<const uint2*>(centroid(2 * kc + 1));
            val = make_uint4(v0.x, v0.y, v1.x, v1.y);
          } else {
            val = make_uint4(*reinterpret_cast<const uint32_t*>(centroid(4 * kc)), *reinterpret_cast<const uint32_t*>(centroid(4 * kc + 1)),
                             *reinterpret_cast<const uint32_t*>(centroid(4 * kc + 2)), *reinterpret_cast<const uint32_t*>(centroid(4 * kc + 3)));
          }
          *reinterpret_cast<uint4*>(brow + kc * 2048) = val;
        }
        // ne[b] is read by the epilogue of tile bn - 2: wait until it has released the buffer
        mbar_wait(&sh.acc_empty[b], ((bn >> 1) & 1) ^ 1);
        const float ne_e = valid ? nsum : INFINITY;
        sh.ne[b][e] = ne_e;
        float nmin = ne_e;  // the group screen's min ne over this warp's 32 entries (fminf: a NaN never wins)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) nmin = fminf(nmin, __shfl_xor_sync(0xffffffffu, nmin, o));
        if ((e & 31) == 0) sh.ne_min[b][e >> 5] = nmin;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> tensor-core proxy
        mbar_arrive(&sh.b_full[b]);
      }
    }
  } else {
    setmaxnreg_dec<PT_REG_OTHER>();  // warpgroup 3: warps 14 and 15 have no role and exit here
    if (warp == 12) {
      // ======================= TMA producer (whole warp loops, one elected lane issues) =======================
      uint32_t an = 0, cn = 0;
      for (int64_t it = blockIdx.x; it < n_items; it += gridDim.x) {
        const LmTile t = items[it];
        if (t.nrows <= 0) continue;  // every role skips empty segments the same way
        const int ab = an & 1;
        mbar_wait(&sh.a_empty[ab], ((an >> 1) & 1) ^ 1);
        if (elect_one()) {
          mbar_arrive_expect_tx(&sh.a_full[ab], 2 * TILE);
          for (int h = 0; h < 2; h++)
            bulk_g2s(a_buf + (ab * 2 + h) * TILE, a_scratch + ((int64_t)t.grp * 2 + h) * TILE, TILE, &sh.a_full[ab]);
        }
        __syncwarp();
        const unsigned char* lcodes = dir.codes[t.list];
        const float* lnorms = HAS_NORM ? pqnorm + pqnorm_off[t.list] : nullptr;  // list segments start 128-byte aligned
        const int ntiles = (t.nrows + PT_N - 1) / PT_N;
        for (int i = 0; i < ntiles; i++, cn++) {
          const int s = cn % PT_CS;
          mbar_wait(&sh.code_empty[s], ((cn / PT_CS) & 1) ^ 1);
          if (elect_one()) {
            const int n_e = min(PT_N, t.nrows - i * PT_N);
            const uint32_t bytes = ((uint32_t)n_e * M + 15u) & ~15u;
            const uint32_t nbytes = HAS_NORM ? ((uint32_t)n_e * 4u + 15u) & ~15u : 0u;
            mbar_arrive_expect_tx(&sh.code_full[s], bytes + nbytes);
            bulk_g2s(code_buf + s * CODE_STAGE, lcodes + (int64_t)(t.row0 + i * PT_N) * M, bytes, &sh.code_full[s]);
            if (HAS_NORM) bulk_g2s(nstage + s * PT_N, lnorms + (t.row0 + i * PT_N), nbytes, &sh.code_full[s]);
          }
          __syncwarp();
        }
        an++;
      }
    } else if (warp == 13) {
      // ======================= candidate drain: shared queue -> global per-query lists =======================
      const int lane = tid & 31;
      unsigned int t = 0;
      for (;;) {
        unsigned long long r[4];
        int n = 0;
        bool open = true;
#pragma unroll
        for (int u = 0; u < 4; u++) {
          r[u] = *reinterpret_cast<volatile unsigned long long*>(&sh.q_rec[(t + (unsigned)(lane + 32 * u)) % PT_RQ]);
          const unsigned int m = __ballot_sync(0xffffffffu, r[u] != kRecEmpty);
          if (open) {  // records are consumed as a contiguous prefix, so the tail stays a single counter
            if (m == 0xffffffffu) n += 32;
            else n += __ffs(~m) - 1, open = false;
          }
        }
        if (n == 0) {
          if (*reinterpret_cast<volatile int*>(&sh.q_done) == 8 && *reinterpret_cast<volatile unsigned int*>(&sh.q_head) == t) break;
          __nanosleep(64);
          continue;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
          if (lane + 32 * u < n) {
            const int q = (int)(r[u] >> 48), p = (int)((r[u] >> 32) & 0xFFFFu);
            const int slot = atomicAdd(cand_cnt + q, 1);  // a count above cap flags the query for the exact kernel
            if (slot < cap) cand[(int64_t)q * cap + slot] = ((unsigned long long)(uint32_t)p << 32) | (r[u] & 0xFFFFFFFFull);
            *reinterpret_cast<volatile unsigned long long*>(&sh.q_rec[(t + (unsigned)(lane + 32 * u)) % PT_RQ]) = kRecEmpty;
          }
        }
        __threadfence_block();
        __syncwarp();
        t += (unsigned int)n;
        if (lane == 0) *reinterpret_cast<volatile unsigned int*>(&sh.q_tail) = t;
      }
    }
  }
}

// ---- phase C: candidates -> reference arithmetic -> merge with phase A's keys ---------------------
constexpr int RS_NT = 256;

template <int METRIC>
__global__ void __launch_bounds__(RS_NT)
    pq_rescore_kernel(const float* __restrict__ ip_table, const int32_t* __restrict__ probe_ids,
                      const float* __restrict__ coarse_dis, int nprobe, ListDirectory dir, int M, const float* __restrict__ T,
                      const int* __restrict__ cand_cnt, const unsigned long long* __restrict__ cand, int cap,
                      const unsigned long long* __restrict__ keys_a, int64_t keys_a_stride, int kprime, int NP,
                      const int* __restrict__ row_limit, FilterArgs f, int sorted_out, unsigned long long* __restrict__ out) {
  if (cta_cancelled(f.cancel, kCsPqRescore)) return;
  extern __shared__ __align__(16) unsigned char rs_smem[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(rs_smem);  // [NP]
  float* ips = reinterpret_cast<float*>(buf + NP);                            // [M][256]
  const int q = blockIdx.x, tid = threadIdx.x;
  const int cnt = cand_cnt[q];
  if (cnt > cap) return;  // overflow: the exact kernel redoes this query (pq_fallback_merge_kernel writes out)
  if (cnt == 0 && !sorted_out) {  // nothing passed the filter: phase A's (unordered) keys are the answer -- the usual case
    for (int i = tid; i < kprime; i += RS_NT) out[(int64_t)q * kprime + i] = keys_a[(int64_t)q * keys_a_stride + i];
    return;
  }
  // a handful of candidates (the usual case) read the query's inner-product table straight from L2; staging the
  // 4 M bytes-per-sub-quantiser table in shared memory pays only for long candidate lists
  const float* ipq = ip_table + (int64_t)q * M * PT_KSUB;
  const bool staged = cnt > 64;
  if (staged) {
    const float4* ipq4 = reinterpret_cast<const float4*>(ipq);
    for (int i = tid; i < M * PT_KSUB / 4; i += RS_NT) reinterpret_cast<float4*>(ips)[i] = __ldg(ipq4 + i);
  }
  // CandQueue layout: buf[0, KP) = the current best (phase A's keys, sentinel padded), buf[KP, KP + cnt) = candidates;
  // its flush keeps the k' best -- a bitonic sort of the occupied prefix when short, an MSB radix select (linear in the
  // fill) when a loose bound let thousands of candidates through
  __shared__ int s_cnt;
  __shared__ unsigned long long s_tau;
  int KP = 16;
  while (KP < kprime) KP <<= 1;
  CandQueue cq{buf, &s_cnt, &s_tau, kprime, KP, NP};
  for (int i = tid; i < KP; i += RS_NT) buf[i] = i < kprime ? keys_a[(int64_t)q * keys_a_stride + i] : kKeySentinel;
  if (tid == 0) s_cnt = cnt, s_tau = kKeySentinel;
  __syncthreads();
  for (int i = tid; i < cnt; i += RS_NT) {
    const unsigned long long rec = cand[(int64_t)q * cap + i];
    const int p = (int)(rec >> 32);
    const uint32_t pos = (uint32_t)rec;
    const int l = probe_ids[(int64_t)q * nprobe + p];
    float dis = coarse_dis[(int64_t)q * nprobe + p];
    const unsigned char* code = dir.codes[l] + (int64_t)pos * M;
    const float* Tl = METRIC == kMetricL2 ? T + (int64_t)l * M * PT_KSUB : nullptr;
    // the reference's order: dis = dis0; dis += tab[m][code[m]], tab = T - 2 ip as the list scan's IVF-PQ codec builds it
    for (int m = 0; m < M; m++) {
      const int c = code[m];
      const float a = staged ? ips[m * PT_KSUB + c] : __ldg(ipq + m * PT_KSUB + c);
      dis += METRIC == kMetricL2 ? fmaf(-2.0f, a, __ldg(Tl + m * PT_KSUB + c)) : a;
    }
    const int64_t raw = dir.ids[l][pos];
    // positions below row_limit were scored exactly by phase A: they are in keys_a already (or lost there for good)
    const bool ok = (int)pos >= row_limit[(int64_t)q * nprobe + p] && raw >= 0 && ctx_is_valid(f.del_bits, f.filter_bits, (uint32_t)raw) && dis <= f.max_score && dis >= f.min_score;
    buf[KP + i] = ok ? make_key(score2ord<METRIC>(dis), (uint32_t)raw) : kKeySentinel;
  }
  __syncthreads();
  cq.flush(true);
  for (int i = tid; i < kprime; i += RS_NT) out[(int64_t)q * kprime + i] = buf[i];
}

// overflowed queries: the k' best of the exact kernel's per-group partials (ngroups runs of k') into out[q], streamed
// through a CandQueue in rounds of RS_NT * FM_ITEMS keys, so the shared memory depends on k' alone
constexpr int FM_ITEMS = 4;
__global__ void __launch_bounds__(RS_NT)
    pq_fallback_merge_kernel(const int* __restrict__ cand_cnt, int cap, const unsigned long long* __restrict__ partial,
                             int ngroups, int kprime, int KP, int SORTN, unsigned long long* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char rs_smem[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(rs_smem);
  __shared__ int s_cnt;
  __shared__ unsigned long long s_tau;
  const int q = blockIdx.x, tid = threadIdx.x;
  if (cand_cnt[q] <= cap) return;
  const int64_t n = (int64_t)ngroups * kprime;
  const unsigned long long* row = partial + (int64_t)q * n;
  CandQueue cq{buf, &s_cnt, &s_tau, kprime, KP, SORTN};
  cq.init();
  const int per_round = RS_NT * FM_ITEMS;
  for (int64_t base = 0; base < n; base += per_round) {
    const unsigned long long tau = s_tau;
#pragma unroll
    for (int u = 0; u < FM_ITEMS; u++) {
      const int64_t i = base + u * RS_NT + tid;
      const unsigned long long key = i < n ? row[i] : kKeySentinel;
      cq.push_warp(key < tau, key);
    }
    __syncthreads();
    const int c_now = s_cnt;
    __syncthreads();  // same snapshot in every thread before any warp pushes again
    if (base + per_round < n && c_now + per_round > cq.cap()) cq.flush();
  }
  cq.flush(true);
  for (int i = tid; i < kprime; i += RS_NT) out[(int64_t)q * kprime + i] = buf[i];
}

template <int M, int DSUB>
cudaError_t launch_scan_shape(const unsigned char* a_scratch, const PairMeta* meta, const int8_t* cb, const float* pqnorm,
                              const int64_t* pqnorm_off,
                              const LmTile* items, const int64_t* totals, ListDirectory dir, FilterArgs f, int metric,
                              int* cand_cnt, unsigned long long* cand, int cap, int grid, cudaStream_t st) {
  constexpr int TILE = (M * DSUB / 16) * 2048;
  const size_t base = (size_t)M * PT_KSUB * DSUB + 6 * (size_t)TILE + (size_t)PT_CS * PT_N * M + 4096;
  const bool l2 = metric == kMetricL2;
  const bool eager = f.del_bits != nullptr || f.filter_bits != nullptr;
  if (l2 && (!pqnorm || !pqnorm_off)) return cudaErrorInvalidValue;
  const size_t smem = base + (l2 ? (size_t)PT_CS * PT_N * 4 : 0);
  auto go = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, PT_NT, smem, st>>>(a_scratch, meta, cb, pqnorm, pqnorm_off, items, totals, dir, f, cand_cnt, cand, cap);
    note_launch();
    return cudaGetLastError();
  };
  if (l2) return eager ? go(pqtc_scan_kernel<M, DSUB, true, true>) : go(pqtc_scan_kernel<M, DSUB, true, false>);
  return eager ? go(pqtc_scan_kernel<M, DSUB, false, true>) : go(pqtc_scan_kernel<M, DSUB, false, false>);
}

}  // namespace

// ---- |r_e|^2 of every list entry (L2): out[off[l] + pos] = sum_m nrm[m][code[m]] ------------------------------------------
namespace {
__global__ void __launch_bounds__(256)
    pq_entry_norms_kernel(ListDirectory dir, int M, const float* __restrict__ nrm, const int64_t* __restrict__ off,
                          float* __restrict__ out) {
  extern __shared__ float s_nrm[];  // [M][256]
  const int l = blockIdx.y;
  const int len = dir.len[l];
  const int row0 = blockIdx.x * 1024;
  if (row0 >= len) return;
  for (int i = threadIdx.x; i < M * PT_KSUB; i += 256) s_nrm[i] = nrm[i];
  __syncthreads();
  const unsigned char* codes = dir.codes[l];
  float* dst = out + off[l];
  for (int r = row0 + threadIdx.x; r < min(len, row0 + 1024); r += 256) {
    const unsigned char* c = codes + (int64_t)r * M;
    float sum = 0.f;
    for (int m = 0; m < M; m++) sum += s_nrm[m * PT_KSUB + c[m]];
    dst[r] = sum;
  }
}
}  // namespace

cudaError_t launch_pq_entry_norms(ListDirectory dir, int nlist, int max_len, int M, const float* nrm, const int64_t* off,
                                  float* out, cudaStream_t st) {
  if (nlist <= 0 || max_len <= 0) return cudaSuccess;
  const size_t smem = (size_t)M * PT_KSUB * 4;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(pq_entry_norms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  dim3 grid((unsigned)((max_len + 1023) / 1024), (unsigned)nlist);
  pq_entry_norms_kernel<<<grid, 256, smem, st>>>(dir, M, nrm, off, out);
  note_launch();
  return cudaGetLastError();
}

bool pqtc_supported(int M, int dsub) {
  // power-of-two shapes only.  (M = 12, dsub = 8 -- 1536-byte code tiles, 24 KiB operand tiles -- compiled and ran, but
  // intermittently (about 1 search in 100, on some boxes more) lost the rows of one decode warp of a tile; the cause
  // was not found in the time available, so that shape stays on the LUT kernel.)
  return (M == 16 && dsub == 8) || (M == 8 && dsub == 16) || (M == 8 && dsub == 8) || (M == 16 && dsub == 4) ||
         (M == 4 && dsub == 16) || (M == 4 && dsub == 32) || (M == 4 && dsub == 8) || (M == 8 && dsub == 4);
}

size_t pqtc_pair_meta_bytes() { return sizeof(PairMeta) + sizeof(PairBound); }

cudaError_t launch_pqtc_tables(const float* pq, int M, int dsub, int8_t* cb, float* nrm, float* rmax2, cudaStream_t st) {
  pqtc_tables_kernel<<<1, 256, 0, st>>>(pq, M, dsub, cb, nrm, rmax2);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pqtc_plan_phase_a(const int32_t* probe_ids, int64_t npairs, int nprobe, int pa_max, long long target,
                                     const int* list_len, int32_t* probes_a, int32_t* probes_b, int* row_limit,
                                     cudaStream_t st) {
  if (npairs <= 0) return cudaSuccess;
  pqtc_plan_phase_a_kernel<<<(unsigned)((npairs + 255) / 256), 256, 0, st>>>(probe_ids, npairs, nprobe, pa_max, target,
                                                                            list_len, probes_a, probes_b, row_limit);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pq_stage_pairs(const float* xq, int64_t ldq, int d, const float* coarse, int64_t ldc, const LmTile* items,
                                  int max_items, const int64_t* totals, const int64_t* pair_j, int nprobe,
                                  const float* coarse_dis, const float* rmax2, FilterArgs f, int metric,
                                  unsigned char* a_scratch, void* meta, int64_t max_groups, int* cand_cnt, int cap,
                                  const int* row_limit, cudaStream_t st) {
  if (max_items <= 0) return cudaSuccess;
  if (d % 32) return cudaErrorInvalidValue;
  PairMeta* pm = static_cast<PairMeta*>(meta);
  PairBound* pb = reinterpret_cast<PairBound*>(pm + max_groups * PT_G);
  if (metric == kMetricL2)
    pq_stage_pairs_kernel<kMetricL2><<<max_items, PT_G, 0, st>>>(xq, ldq, d, coarse, ldc, items, totals, pair_j, nprobe,
                                                                coarse_dis, rmax2, f.min_score, f.max_score, a_scratch, pm,
                                                                pb, cand_cnt, cap, row_limit);
  else
    pq_stage_pairs_kernel<kMetricIP><<<max_items, PT_G, 0, st>>>(xq, ldq, d, coarse, ldc, items, totals, pair_j, nprobe,
                                                                coarse_dis, rmax2, f.min_score, f.max_score, a_scratch, pm,
                                                                pb, cand_cnt, cap, row_limit);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pq_bind_bounds(const int64_t* totals, int64_t max_groups, int nprobe, const float* coarse_dis,
                                  const unsigned long long* bound_keys, int64_t bound_stride, int kprime, FilterArgs f,
                                  int metric, void* meta, int* cand_cnt, int cap, cudaStream_t st) {
  if (max_groups <= 0) return cudaSuccess;
  PairMeta* pm = static_cast<PairMeta*>(meta);
  const PairBound* pb = reinterpret_cast<const PairBound*>(pm + max_groups * PT_G);
  const int64_t slots = max_groups * PT_G;
  const unsigned nb = (unsigned)((slots + 255) / 256);
  if (metric == kMetricL2)
    pq_bind_bounds_kernel<kMetricL2><<<nb, 256, 0, st>>>(totals, slots, nprobe, coarse_dis, bound_keys, bound_stride, kprime,
                                                        f.min_score, f.max_score, pb, pm, cand_cnt, cap);
  else
    pq_bind_bounds_kernel<kMetricIP><<<nb, 256, 0, st>>>(totals, slots, nprobe, coarse_dis, bound_keys, bound_stride, kprime,
                                                        f.min_score, f.max_score, pb, pm, cand_cnt, cap);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pqtc_scan(const unsigned char* a_scratch, const void* meta, const int8_t* cb, const float* pqnorm,
                             const int64_t* pqnorm_off,
                             const LmTile* items, int max_items, const int64_t* totals, ListDirectory dir, int M, int dsub,
                             FilterArgs f, int metric, int* cand_cnt, unsigned long long* cand, int cap, int num_sms,
                             cudaStream_t st) {
  if (max_items <= 0) return cudaSuccess;
  const int grid = max_items < num_sms ? max_items : num_sms;
  const PairMeta* pm = static_cast<const PairMeta*>(meta);
#define GB_PT(MM, DS) \
  if (M == MM && dsub == DS) return launch_scan_shape<MM, DS>(a_scratch, pm, cb, pqnorm, pqnorm_off, items, totals, dir, f, metric, cand_cnt, cand, cap, grid, st)
  GB_PT(16, 8);
  GB_PT(8, 16);
  GB_PT(8, 8);
  GB_PT(16, 4);
  GB_PT(4, 16);
  GB_PT(4, 32);
  GB_PT(4, 8);
  GB_PT(8, 4);
#undef GB_PT
  return cudaErrorInvalidValue;
}

cudaError_t launch_pq_rescore(const float* ip_table, int nq, const int32_t* probe_ids, const float* coarse_dis, int nprobe,
                              ListDirectory dir, int M, const float* T, const int* cand_cnt, const unsigned long long* cand,
                              int cap, const unsigned long long* keys_a, int64_t keys_a_stride, int kprime, int metric,
                              const int* row_limit, FilterArgs f, bool sorted_out, unsigned long long* out, cudaStream_t st) {
  if (nq <= 0) return cudaSuccess;
  const int NP = next_pow2(next_pow2(kprime < 16 ? 16 : kprime) + cap);  // CandQueue: KP best + cap candidates
  const size_t smem = (size_t)NP * 8 + (size_t)M * PT_KSUB * 4;
  if (smem > 200 * 1024) return cudaErrorInvalidValue;
  cudaError_t e;
  if (metric == kMetricL2) {
    e = cudaFuncSetAttribute(pq_rescore_kernel<kMetricL2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    pq_rescore_kernel<kMetricL2><<<nq, RS_NT, smem, st>>>(ip_table, probe_ids, coarse_dis, nprobe, dir, M, T, cand_cnt, cand,
                                                         cap, keys_a, keys_a_stride, kprime, NP, row_limit, f, sorted_out ? 1 : 0, out);
  } else {
    e = cudaFuncSetAttribute(pq_rescore_kernel<kMetricIP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    pq_rescore_kernel<kMetricIP><<<nq, RS_NT, smem, st>>>(ip_table, probe_ids, coarse_dis, nprobe, dir, M, T, cand_cnt, cand,
                                                         cap, keys_a, keys_a_stride, kprime, NP, row_limit, f, sorted_out ? 1 : 0, out);
  }
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pq_fallback_merge(const int* cand_cnt, int cap, int nq, const unsigned long long* partial, int ngroups,
                                     int kprime, unsigned long long* out, cudaStream_t st) {
  if (nq <= 0) return cudaSuccess;
  if (kprime <= 0 || kprime > 4096 || ngroups <= 0) return cudaErrorInvalidValue;
  const int KP = next_pow2(kprime < 16 ? 16 : kprime);
  const int SORTN = next_pow2(KP + RS_NT * FM_ITEMS);  // at most 64 KiB at k' = 4096
  const size_t smem = (size_t)SORTN * 8;
  cudaError_t e = cudaFuncSetAttribute(pq_fallback_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  pq_fallback_merge_kernel<<<nq, RS_NT, smem, st>>>(cand_cnt, cap, partial, ngroups, kprime, KP, SORTN, out);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
