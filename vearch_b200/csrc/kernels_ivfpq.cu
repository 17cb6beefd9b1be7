// K4 / K5 / K5r / K8(encode): IVF-PQ look-up tables, asymmetric-distance scan, exact re-rank,
// PQ encoding.
//
// Replaces, in the reference:
//   QueryTables::init_query_{L2,IP} / precompute_list_tables_{L2,IP}
//       (index/impl/gamma_index_ivfpq.h:154-175, 223-309)             -> pq_ip_table + in-CTA LUT
//   faiss IndexIVFPQ::precompute_table (called at gamma_index_ivfpq.cc:1099)  -> pq_precompute_table
//   GammaIVFPQScanner::scan_list_with_table (gamma_index_ivfpq.h:923-953),
//       scan_one_list / search_preassigned (gamma_index_ivfpq.cc:635-673, 730-947) -> ivfpq_scan
//   compute_dis exact re-rank (gamma_index_ivfpq.cc:675-726)            -> rerank
//   pq.compute_codes on residuals in GammaIVFPQIndex::Add (gamma_index_ivfpq.cc:478-494) -> pq_encode
//
// Arithmetic order is the reference's: tab = T[list] + (-2)*ip ; dis = dis0 ; dis += tab[m][code[m]]
// for m = 0..M-1 (one fp32 add at a time).  Table kernels use unfused mul/add so that tables are
// bit-identical to a scalar CPU evaluation; given the same (keys, coarse_dis) the ADC distances
// are bit-equal to the oracle's.
//
// Algorithmic bytes of the scan: (M + 8) per entry + M*256*4 per (query, list) for the T row.
//
// nbits_per_idx < 8 (ksub = 2^nbits): the table kernels and the encoder run over ksub centroids with the same
// arithmetic, the encoder's [n][M] codes are bit-packed by pq_pack_codes (faiss PQEncoderGeneric: code m at bits
// [m nbits, (m + 1) nbits) of the entry, LSB-first), and IvfpqPackedCodec scans them (code_size + 8 bytes per entry,
// M*ksub*4 per (query, list)).
#include <float.h>

#include "common.cuh"
#include "kernels.h"
#include "list_scan.cuh"

namespace gb {

namespace {

constexpr int KSUB = 256;  // ksub at nbits = 8, and the threads of the table kernels

// ---------------- per-query inner-product table ------------------------------------------
constexpr int IPT_QB = 32;

// one CTA per (sub-quantiser, IPT_QB queries); thread t computes centroid t % ksub of every (KSUB / ksub)-th query
__global__ void __launch_bounds__(KSUB)
    pq_ip_table_kernel(const float* __restrict__ xq, int64_t ldq, int nq, const float* __restrict__ pq, int M, int dsub,
                       int ksub, float* __restrict__ ip) {
  extern __shared__ float sm[];
  float* ps = sm;                // [dsub][ksub]
  float* xs = sm + dsub * ksub;  // [IPT_QB][dsub]
  const int m = blockIdx.x;
  const int q0 = blockIdx.y * IPT_QB;
  const int c = threadIdx.x % ksub, qstep = KSUB / ksub;
  for (int idx = threadIdx.x; idx < dsub * ksub; idx += KSUB) {
    int cc = idx / dsub, j = idx - cc * dsub;
    ps[j * ksub + cc] = pq[((int64_t)m * ksub) * dsub + idx];
  }
  for (int idx = threadIdx.x; idx < IPT_QB * dsub; idx += KSUB) {
    int qq = idx / dsub, j = idx - qq * dsub;
    xs[idx] = (q0 + qq < nq) ? xq[(int64_t)(q0 + qq) * ldq + m * dsub + j] : 0.f;
  }
  __syncthreads();
  for (int qq = threadIdx.x / ksub; qq < IPT_QB && q0 + qq < nq; qq += qstep) {
    float acc = 0.f;
    for (int j = 0; j < dsub; j++) acc = __fadd_rn(acc, __fmul_rn(xs[qq * dsub + j], ps[j * ksub + c]));
    ip[((int64_t)(q0 + qq) * M + m) * ksub + c] = acc;
  }
}

// ---------------- precomputed table T[l][m][c] --------------------------------------------
// one CTA per list; thread t computes the entries t, t + KSUB, ... of the list's [M][ksub] row
__global__ void __launch_bounds__(KSUB)
    pq_precompute_table_kernel(const float* __restrict__ coarse, int64_t ldc, const float* __restrict__ pq, int M,
                               int dsub, int ksub, float* __restrict__ T) {
  const int l = blockIdx.x;
  for (int i = threadIdx.x; i < M * ksub; i += KSUB) {
    const int m = i / ksub;
    const float* cl = coarse + (int64_t)l * ldc + m * dsub;
    const float* p = pq + (int64_t)i * dsub;
    float nrm = 0.f, ipv = 0.f;
    for (int j = 0; j < dsub; j++) {
      float pj = p[j];
      nrm = __fadd_rn(nrm, __fmul_rn(pj, pj));
      ipv = __fadd_rn(ipv, __fmul_rn(__ldg(cl + j), pj));
    }
    T[(int64_t)l * M * ksub + i] = __fadd_rn(nrm, __fmul_rn(2.0f, ipv));
  }
}

// ---------------- ADC scan: the IVF-PQ codec of the list scan (list_scan.cuh) -------------------
// entries per thread per tile for the vector-load code layouts (MW = M / 4 code words per entry): per-tile
// bookkeeping (barrier, tau reload, fill estimate, refill) is paid once per PT entries, while LUT + queue +
// two code stages must stay within ~52 KiB so that four CTAs share an SM (M = 16: 2 x 256 entries, 8 KiB;
// 3 x 256 and 4 x 256 entries per tile were slower in a sweep)
__host__ __device__ constexpr int pq_pt(int MW) { return MW == 2 ? 4 : (MW == 4 ? 2 : (MW == 8 ? 2 : 1)); }

__host__ __device__ inline int pq_tile_entries(int M) {
  if (M == 8 || M == 16 || M == 32 || M == 64) return pq_pt(M / 4) * LS_NT;
  int e = 16384 / M;
  e = (e / LS_NT) * LS_NT;
  if (e < LS_NT) e = LS_NT;
  if (e > 1024) e = 1024;
  return e;
}

// Per list the CTA builds the LUT  T[list] + (-2) ip  (precompute_list_tables); under IP the per-query inner-product
// table (L2-resident) IS the LUT and is copied once.  dis = dis0; dis += lut[m][code[m]] for m = 0..M-1.
struct IvfpqCodec {
  using Entry = float;
  static constexpr bool kDis0 = true;
  static constexpr int kMinCtasPerSm = 0;  // shared memory, not registers, sets its CTAs per SM
  const float* ip_table;  // [nq][M][256]
  const float* T;         // [nlist][M][256], L2 only
  int M;
  const float4* ipq4;  // this CTA's query in ip_table

  __host__ __device__ int code_bytes() const { return M; }
  int tile_entries() const { return pq_tile_entries(M); }
  __host__ __device__ static constexpr int pt(int MW) { return pq_pt(MW); }

  __device__ __forceinline__ void cta_begin(float* lut, int q, int metric) {
    ipq4 = reinterpret_cast<const float4*>(ip_table + (int64_t)q * M * KSUB);
    if (metric != kMetricL2) {
      float4* dst = reinterpret_cast<float4*>(lut);
      for (int i = threadIdx.x; i < M * KSUB / 4; i += LS_NT) dst[i] = __ldg(ipq4 + i);
      __syncthreads();
    }
  }
  __device__ __forceinline__ void list_begin(float* lut, int list, int metric) const {
    if (metric == kMetricL2) {
      const float4* Tl = reinterpret_cast<const float4*>(T + (int64_t)list * M * KSUB);
      float4* lut4 = reinterpret_cast<float4*>(lut);
      for (int i = threadIdx.x; i < M * KSUB / 4; i += LS_NT) {
        float4 t = __ldg(Tl + i), a = __ldg(ipq4 + i);
        lut4[i] = make_float4(fmaf(-2.0f, a.x, t.x), fmaf(-2.0f, a.y, t.y), fmaf(-2.0f, a.z, t.z),
                              fmaf(-2.0f, a.w, t.w));
      }
      __syncthreads();
    }
  }
  using Acc = float;
  __device__ __forceinline__ float start(float dis0) const { return dis0; }
  __device__ __forceinline__ float finish(float dis) const { return dis; }
};

template <int METRIC>
cudaError_t launch_scan_m(const IvfpqCodec& c, int nq, const ListScanArgs& a, cudaStream_t st) {
  switch (c.M) {
    case 8: return launch_list_scan<IvfpqCodec, METRIC, 2>(c, nq, a, st);
    case 16: return launch_list_scan<IvfpqCodec, METRIC, 4>(c, nq, a, st);
    case 32: return launch_list_scan<IvfpqCodec, METRIC, 8>(c, nq, a, st);
    case 64: return launch_list_scan<IvfpqCodec, METRIC, 16>(c, nq, a, st);
    default: return launch_list_scan<IvfpqCodec, METRIC, 0>(c, nq, a, st);
  }
}

// ---------------- ADC scan over bit-packed codes (nbits_per_idx < 8) ------------------------------
// Code m of an entry sits at bits [m nbits, (m + 1) nbits) of its code_size = ceil(M nbits / 8) bytes, LSB-first.  The
// table is [M][ksub] fp32, built per list exactly as IvfpqCodec's [M][256] one; an entry's score is dis0, then
// += lut[m][code m] for m = 0..M-1, one fp32 add at a time (PQDecoder order, gamma_index_ivfpq.h:532-536).  Rows are
// code_size bytes apart in the stage, so they start at any byte: the codes are read as the aligned 32-bit words that
// hold them, through a 64-bit bit buffer.
__host__ __device__ inline int pq_packed_tile_entries(int code_size) {  // ~16 KiB of codes, 256..1024 entries
  int e = 16384 / code_size;
  e = (e / LS_NT) * LS_NT;
  return e < LS_NT ? LS_NT : (e > 1024 ? 1024 : e);
}

struct IvfpqPackedCodec {
  using Entry = float;
  static constexpr bool kDis0 = true;
  static constexpr bool kCodeSum = true;
  static constexpr int kMinCtasPerSm = 0;
  const float* ip_table;  // [nq][M][ksub]
  const float* T;         // [nlist][M][ksub], L2 only
  int M, nbits;
  const float* ipq;  // this CTA's query in ip_table

  __host__ __device__ int ksub() const { return 1 << nbits; }
  __host__ __device__ int code_bytes() const { return (M * nbits + 7) / 8; }
  __host__ __device__ int table_entries() const { return (M * ksub() + 3) & ~3; }
  int tile_entries() const { return pq_packed_tile_entries(code_bytes()); }
  __host__ __device__ static constexpr int pt(int) { return 1; }  // not used: MW = 0 only

  __device__ __forceinline__ void cta_begin(float* lut, int q, int metric) {
    ipq = ip_table + (int64_t)q * M * ksub();
    if (metric != kMetricL2) {
      for (int i = threadIdx.x; i < M * ksub(); i += LS_NT) lut[i] = __ldg(ipq + i);
      __syncthreads();
    }
  }
  __device__ __forceinline__ void list_begin(float* lut, int list, int metric) const {
    if (metric == kMetricL2) {
      const float* Tl = T + (int64_t)list * M * ksub();
      for (int i = threadIdx.x; i < M * ksub(); i += LS_NT) lut[i] = fmaf(-2.0f, __ldg(ipq + i), __ldg(Tl + i));
      __syncthreads();
    }
  }
  using Acc = float;
  __device__ __forceinline__ float start(float dis0) const { return dis0; }
  __device__ __forceinline__ float finish(float dis) const { return dis; }
  __device__ __forceinline__ float code_sum(const unsigned char* code, const float* __restrict__ tab, float acc) const {
    const uintptr_t a = reinterpret_cast<uintptr_t>(code);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const int skip = (int)(a & 3) * 8;
    uint64_t bits = w[0] >> skip;  // >= 8 valid bits: the first code (nbits <= 7) needs no refill
    int nb = 32 - skip;
    const uint32_t mask = (1u << nbits) - 1u;
    const int ks = ksub();
    for (int m = 0; m < M; m++, tab += ks) {
      if (nb < nbits) {
        bits |= (uint64_t)(*++w) << nb;
        nb += 32;
      }
      acc += tab[(uint32_t)bits & mask];
      bits >>= nbits;
      nb -= nbits;
    }
    return acc;
  }
};

// ---------------- exact re-rank -------------------------------------------------------------
constexpr int RR_NT = 256;

// The exact score of RR_U rows (nullptr: no row, score unused) against the query q4 (shared memory, d a multiple of 4):
// lane l takes the float4 columns l, l + 32, ... of each row into four FMA accumulators, then (a0 + a1) + (a2 + a3) and
// an xor-shuffle tree, so every lane ends with the same dis[u].  Both re-rank kernels score through this routine only:
// the two-pass kernel's keys are bit-identical to the one-pass kernel's by construction.
template <int RR_U>
__device__ __forceinline__ void rr_exact_scores(const float4* q4, const float4* const (&row)[RR_U], int d, int metric,
                                                float (&dis)[RR_U]) {
  const int lane = threadIdx.x & 31;
  float acc[RR_U][4];
#pragma unroll
  for (int u = 0; u < RR_U; u++) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0.f;
  for (int c = lane; c < (d >> 2); c += 32) {
    const float4 w = q4[c];
    float4 v[RR_U];
#pragma unroll
    for (int u = 0; u < RR_U; u++) v[u] = row[u] ? __ldg(row[u] + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int u = 0; u < RR_U; u++) {
      if (metric == kMetricL2) {
        const float t0 = v[u].x - w.x, t1 = v[u].y - w.y, t2 = v[u].z - w.z, t3 = v[u].w - w.w;
        acc[u][0] = fmaf(t0, t0, acc[u][0]), acc[u][1] = fmaf(t1, t1, acc[u][1]);
        acc[u][2] = fmaf(t2, t2, acc[u][2]), acc[u][3] = fmaf(t3, t3, acc[u][3]);
      } else {
        acc[u][0] = fmaf(v[u].x, w.x, acc[u][0]), acc[u][1] = fmaf(v[u].y, w.y, acc[u][1]);
        acc[u][2] = fmaf(v[u].z, w.z, acc[u][2]), acc[u][3] = fmaf(v[u].w, w.w, acc[u][3]);
      }
    }
  }
#pragma unroll
  for (int u = 0; u < RR_U; u++) {
    dis[u] = (acc[u][0] + acc[u][1]) + (acc[u][2] + acc[u][3]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) dis[u] += __shfl_xor_sync(0xffffffffu, dis[u], off);
  }
}

__device__ __forceinline__ const float4* rr_row(const float* const* raw_segments, int seg_shift, int64_t ld_raw,
                                                 uint32_t vid) {
  return reinterpret_cast<const float4*>(raw_segments[vid >> seg_shift] +
                                         (int64_t)(vid & ((1u << seg_shift) - 1u)) * ld_raw);
}

// RR_U: candidates a warp gathers per iteration.  Four keep 2 KiB of independent row loads in flight per warp, which
// covers HBM latency (eight cost occupancy; the gather is pure latency: recall_num random 4d-byte rows per query).
// Rows in mapped host memory come over PCIe, whose round trip is several times longer: eight per warp there.
template <int RR_U>
__global__ void __launch_bounds__(RR_NT)
    rerank_kernel(const unsigned long long* __restrict__ cand_keys, int ncand, int NP, const float* __restrict__ xq,
                  int64_t ldq, int d, const float* const* __restrict__ raw_segments, int seg_shift, int64_t ld_raw,
                  int k, int metric, FilterArgs f, unsigned long long* __restrict__ out_keys) {
  if (cta_cancelled(f.cancel, kCsRerank)) return;  // before any candidate's row is read (DESIGN.md section 8)
  extern __shared__ __align__(16) unsigned char rr_smem[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(rr_smem);  // [NP]
  float* qs = reinterpret_cast<float*>(buf + NP);                              // [d]
  const int q = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < d; i += RR_NT) qs[i] = xq[(int64_t)q * ldq + i];
  for (int i = threadIdx.x; i < NP; i += RR_NT) buf[i] = kKeySentinel;
  __syncthreads();
  const float4* q4 = reinterpret_cast<const float4*>(qs);
  for (int j0 = warp * RR_U; j0 < ncand; j0 += (RR_NT / 32) * RR_U) {
    uint32_t vid[RR_U];
    const float4* row[RR_U];
#pragma unroll
    for (int u = 0; u < RR_U; u++) {
      const int j = j0 + u;
      const unsigned long long ck = j < ncand ? cand_keys[(int64_t)q * ncand + j] : kKeySentinel;
      vid[u] = (uint32_t)ck;
      row[u] = ck != kKeySentinel ? rr_row(raw_segments, seg_shift, ld_raw, vid[u]) : nullptr;  // recall_idxi[j] < 0 (ivfpq.cc:691)
    }
    float dis[RR_U];
    rr_exact_scores<RR_U>(q4, row, d, metric, dis);
#pragma unroll
    for (int u = 0; u < RR_U; u++)
      if (lane == 0 && row[u] && dis[u] <= f.max_score && dis[u] >= f.min_score)
        buf[j0 + u] = make_key(score2ord(dis[u], metric), vid[u]);
  }
  __syncthreads();
  block_bitonic_sort(buf, NP);
  for (int i = threadIdx.x; i < k; i += RR_NT) out_keys[(int64_t)q * k + i] = i < NP ? buf[i] : kKeySentinel;
}

// ---------------- two-pass exact re-rank over the int8 shadow of the raw rows ---------------------------------------
// Shadow row of y (RawStore, kernels_ivfpq.cu shadow_encode_kernel): cols16 = round_up(dpad, 16) int8 values
// qy = rn(y / s), s = max|y| / 127, zero padded, then float4 {s, e, nrm, 0} with e >= |y - s qy| and nrm >= |s qy|
// (both rounded up).  A row whose scale is zero or not finite has e = nrm = inf: it is unbounded.
//
// Pass 1 bounds every candidate's fp32 score from its shadow row (DESIGN §3, "Exact re-rank"): [lo, hi] surely holds
// the value rr_exact_scores returns.  B = the k-th best hi among the live bounded candidates whose whole interval lies
// inside the score window; a candidate whose lo is worse than B has k candidates surely better than it, so it cannot
// be among the k results.  Pass 2 reads the fp32 rows of the others (lo <= B, so ties at the k-th score survive; and
// every unbounded one) and scores them through rr_exact_scores.
constexpr int RS_U = 4;  // candidates per 8-lane group in pass 1: 16 shadow rows (2.3 KiB at d = 128) in flight per warp
constexpr uint32_t kOrdDead = 0xFFFFFFFFu;   // lo of a dead candidate, hi of one that does not bound B
constexpr uint32_t kOrdNoBound = 0xFFFFFFFEu;  // B with fewer than k bounding candidates: every live one survives

// the k-th smallest of v[0, n) (1 <= k <= n), by an MSB-first radix select over the bytes: four histogram passes
__device__ __forceinline__ uint32_t block_kth_smallest(const uint32_t* v, int n, int k) {
  __shared__ int s_hist[256];
  __shared__ uint32_t s_prefix;
  __shared__ int s_need;
  const int tid = threadIdx.x, lane = tid & 31;
  uint32_t prefix = 0;
  int need = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
      const uint32_t x = v[i];
      if (shift == 24 || (x >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(&s_hist[(x >> shift) & 255], 1);
    }
    __syncthreads();
    if (tid < 32) {
      int h[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; j++) sum += (h[j] = s_hist[lane * 8 + j]);
      int incl = sum;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += t;
      }
      int before = incl - sum;
      if (before < need && need <= incl) {
#pragma unroll
        for (int j = 0; j < 8; j++) {
          if (before < need && need <= before + h[j]) {
            s_prefix = prefix | ((uint32_t)(lane * 8 + j) << shift);
            s_need = need - before;
          }
          before += h[j];
        }
      }
    }
    __syncthreads();
    prefix = s_prefix;
    need = s_need;
  }
  return prefix;
}

// ascending sort of one key per lane
__device__ __forceinline__ unsigned long long warp_sort32(unsigned long long x) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      const unsigned long long y = __shfl_xor_sync(0xffffffffu, x, j);
      const bool keep_min = ((lane & j) == 0) == ((lane & k) == 0);
      x = keep_min ? (x < y ? x : y) : (x < y ? y : x);
    }
  }
  return x;
}

// int8 byte b of w (two's complement) as an exact float: the byte, offset by 128, is the low mantissa byte of 2^23
__device__ __forceinline__ float rs_qy(uint32_t w_biased, int b) {
  return __uint_as_float(__byte_perm(w_biased, 0x4B000000u, 0x7540u + b)) - 8388736.0f;
}

// INTERVALS: write each candidate's pass-1 result to `intervals` (tests); the search instantiates it off
template <int METRIC, bool INTERVALS>
__global__ void __launch_bounds__(RR_NT)
    rerank_prefilter_kernel(const unsigned long long* __restrict__ cand_keys, int ncand, int NP,
                            const float* __restrict__ xq, int64_t ldq, int d, const float* const* __restrict__ raw_segments,
                            int seg_shift, int64_t ld_raw, const unsigned char* const* __restrict__ shadow_segs,
                            int64_t shadow_stride, int cols16, int k, FilterArgs f,
                            unsigned long long* __restrict__ out_keys, int* __restrict__ survivors,
                            uint4* __restrict__ intervals) {
  if (cta_cancelled(f.cancel, kCsRerankPrefilter)) return;
  extern __shared__ __align__(16) unsigned char rr_smem[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(rr_smem);  // [NP] survivors' keys
  float* qs = reinterpret_cast<float*>(buf + NP);                              // [cols16], zero padded
  uint32_t* lo = reinterpret_cast<uint32_t*>(qs + cols16);                     // [NP] best ordinal a candidate can have
  uint32_t* hi = lo + NP;                                                      // [NP] worst ordinal; then survivors' vids
  __shared__ double s_qn;
  __shared__ int s_nsurv;
  const int q = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < cols16; i += RR_NT) qs[i] = i < d ? xq[(int64_t)q * ldq + i] : 0.f;
  for (int i = threadIdx.x; i < NP; i += RR_NT) buf[i] = kKeySentinel;
  if (threadIdx.x == 0) s_nsurv = 0;
  __syncthreads();
  if (warp == 0) {  // |q|, rounded up
    double a = 0.0;
    for (int i = lane; i < d; i += 32) a = __fma_ru((double)qs[i], (double)qs[i], a);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) a = __dadd_ru(a, __shfl_xor_sync(0xffffffffu, a, off));
    if (lane == 0) s_qn = __dsqrt_ru(a);
  }
  __syncthreads();
  // Rounding of fp32 sums of d (cols16) terms in any order, relative (u = 2^-24) ...
  const double u = 0x1p-24;
  const double g1 = 1.01 * (cols16 + 3) * u, gr = 1.01 * (d + 3) * u;
  // ... plus at most 2^-150 per fp32 operation whose result is subnormal (the relative terms alone fail there)
  const double ab = (4.0 * cols16 + 64.0) * 0x1p-149;
  const double qn = s_qn;

  // ---- pass 1: an interval per candidate from its shadow row; 8 lanes x 16 bytes per row ----
  const int g = lane >> 3, sub = lane & 7;
  const int nch = cols16 >> 4;
  const float4* q4 = reinterpret_cast<const float4*>(qs);
  for (int j0 = warp * 4 * RS_U; j0 < ncand; j0 += (RR_NT / 32) * 4 * RS_U) {
    const unsigned char* srow[RS_U];
    float4 meta[RS_U];
#pragma unroll
    for (int u2 = 0; u2 < RS_U; u2++) {
      const int j = j0 + u2 * 4 + g;
      const unsigned long long ck = j < ncand ? cand_keys[(int64_t)q * ncand + j] : kKeySentinel;
      const uint32_t vid = (uint32_t)ck;
      srow[u2] = ck != kKeySentinel
                     ? shadow_segs[vid >> seg_shift] + (int64_t)(vid & ((1u << seg_shift) - 1u)) * shadow_stride
                     : nullptr;
      meta[u2] = srow[u2] ? __ldg(reinterpret_cast<const float4*>(srow[u2] + cols16)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float acc[RS_U];
#pragma unroll
    for (int u2 = 0; u2 < RS_U; u2++) acc[u2] = 0.f;
    for (int c = sub; c < nch; c += 8) {
      uint4 w[RS_U];
#pragma unroll
      for (int u2 = 0; u2 < RS_U; u2++)
        w[u2] = srow[u2] ? __ldg(reinterpret_cast<const uint4*>(srow[u2]) + c) : make_uint4(0u, 0u, 0u, 0u);
      float qv[16];
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const float4 x = q4[c * 4 + t];
        qv[4 * t] = x.x, qv[4 * t + 1] = x.y, qv[4 * t + 2] = x.z, qv[4 * t + 3] = x.w;
      }
#pragma unroll
      for (int u2 = 0; u2 < RS_U; u2++) {
        const uint32_t ww[4] = {w[u2].x ^ 0x80808080u, w[u2].y ^ 0x80808080u, w[u2].z ^ 0x80808080u,
                                w[u2].w ^ 0x80808080u};
#pragma unroll
        for (int i = 0; i < 16; i++) {
          const float y = rs_qy(ww[i >> 2], i & 3);
          if (METRIC == kMetricL2) {
            const float t = fmaf(-meta[u2].x, y, qv[i]);  // q - s qy, one rounding
            acc[u2] = fmaf(t, t, acc[u2]);
          } else {
            acc[u2] = fmaf(qv[i], y, acc[u2]);
          }
        }
      }
    }
#pragma unroll
    for (int u2 = 0; u2 < RS_U; u2++) {
      acc[u2] += __shfl_xor_sync(0xffffffffu, acc[u2], 1);
      acc[u2] += __shfl_xor_sync(0xffffffffu, acc[u2], 2);
      acc[u2] += __shfl_xor_sync(0xffffffffu, acc[u2], 4);
    }
    // lane sub < RS_U of group g finishes candidate j0 + sub * 4 + g
    float a = 0.f;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
    bool live = false;
#pragma unroll
    for (int u2 = 0; u2 < RS_U; u2++)
      if (u2 == sub) a = acc[u2], m = meta[u2], live = srow[u2] != nullptr;
    const int j = j0 + sub * 4 + g;
    if (sub < RS_U && j < ncand) {
      uint32_t jlo = kOrdDead, jhi = kOrdDead;
      float flo = __int_as_float(0x7FC00000), fhi = flo;
      if (live) {
        const double st = a, s = m.x, e = m.y, nrm = m.z;
        double slo, shi, mag;
        if (METRIC == kMetricL2) {
          // real |q - s qy|^2 from the fp32 sum; then |q - y| within e of its root; then the reference's own rounding
          const double r2lo = fmax(0.0, __dmul_rd(__dsub_rd(st, ab), __dsub_rd(1.0, g1)));
          const double r2hi = __dmul_ru(__dadd_ru(st, ab), __dadd_ru(1.0, 2.0 * g1));
          const double rlo = fmax(0.0, __dsub_rd(__dsqrt_rd(r2lo), e));
          const double rhi = __dadd_ru(__dsqrt_ru(r2hi), e);
          slo = fmax(0.0, __dsub_rd(__dmul_rd(__dmul_rd(rlo, rlo), __dsub_rd(1.0, gr)), ab));
          shi = __dadd_ru(__dmul_ru(__dmul_ru(rhi, rhi), __dadd_ru(1.0, gr)), ab);
          mag = shi;
        } else {
          // <q, s qy> = s st within g1 |q| nrm + s ab; <q, y - s qy> within |q| e; the reference's rounding within
          // gr sum |q_i y_i| + ab <= gr |q| (nrm + e) + ab
          const double c = s * st;  // exact: two fp32 factors
          double r = __dmul_ru(__dmul_ru(g1, qn), nrm);
          r = __dadd_ru(r, __dmul_ru(s, ab));
          r = __dadd_ru(r, __dmul_ru(qn, e));
          const double yb = __dmul_ru(qn, __dadd_ru(nrm, e));
          r = __dadd_ru(__dadd_ru(r, __dmul_ru(gr, yb)), ab);
          slo = __dsub_rd(c, r);
          shi = __dadd_ru(c, r);
          mag = __dadd_ru(__dmul_ru(yb, __dadd_ru(1.0, gr)), ab);
        }
        // every partial sum of either evaluation stays below 2^126: no overflow; NaN or inf anywhere: unbounded
        if (mag <= 0x1p126) {
          flo = __double2float_rd(slo), fhi = __double2float_ru(shi);
          jlo = score2ord<METRIC>(METRIC == kMetricL2 ? flo : fhi);
          if (flo >= f.min_score && fhi <= f.max_score) jhi = score2ord<METRIC>(METRIC == kMetricL2 ? fhi : flo);
        } else {
          jlo = 0;
        }
      }
      lo[j] = jlo;
      hi[j] = jhi;
      if (INTERVALS)
        intervals[(int64_t)q * ncand + j] = make_uint4(jlo, jhi, __float_as_uint(flo), __float_as_uint(fhi));
    }
  }
  __syncthreads();

  // ---- the bound, then the survivors' vids (compacted into hi) ----
  uint32_t B = block_kth_smallest(hi, ncand, k < ncand ? k : ncand);
  if (B == kOrdDead) B = kOrdNoBound;
  for (int j0 = 0; j0 < ncand; j0 += RR_NT) {
    const int j = j0 + threadIdx.x;
    const bool keep = j < ncand && lo[j] <= B;
    const unsigned mask = __ballot_sync(0xffffffffu, keep);
    if (mask) {
      int base = 0;
      if (lane == 0) base = atomicAdd(&s_nsurv, __popc(mask));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (keep) hi[base + __popc(mask & ((1u << lane) - 1u))] = (uint32_t)cand_keys[(int64_t)q * ncand + j];
    }
  }
  __syncthreads();
  const int nsurv = s_nsurv;

  // ---- pass 2: exact scores of the survivors ----
  for (int i0 = warp * 4; i0 < nsurv; i0 += (RR_NT / 32) * 4) {
    const float4* row[4];
    uint32_t vid[4];
#pragma unroll
    for (int u2 = 0; u2 < 4; u2++) {
      vid[u2] = i0 + u2 < nsurv ? hi[i0 + u2] : 0u;
      row[u2] = i0 + u2 < nsurv ? rr_row(raw_segments, seg_shift, ld_raw, vid[u2]) : nullptr;
    }
    float dis[4];
    rr_exact_scores<4>(q4, row, d, METRIC, dis);
#pragma unroll
    for (int u2 = 0; u2 < 4; u2++)
      if (lane == 0 && row[u2] && dis[u2] <= f.max_score && dis[u2] >= f.min_score)
        buf[i0 + u2] = make_key(score2ord<METRIC>(dis[u2]), vid[u2]);
  }
  __syncthreads();
  if (nsurv <= 32) {
    if (warp == 0) {
      const unsigned long long x = warp_sort32(lane < NP ? buf[lane] : kKeySentinel);
      if (lane < NP) buf[lane] = x;
    }
    __syncthreads();
  } else {
    block_bitonic_sort(buf, next_pow2(nsurv));
  }
  for (int i = threadIdx.x; i < k; i += RR_NT) out_keys[(int64_t)q * k + i] = i < NP ? buf[i] : kKeySentinel;
  if (survivors && threadIdx.x == 0) survivors[q] = nsurv;
}

// ---------------- the int8 shadow rows (one warp per row) -------------------------------------------------------------
constexpr int SE_NT = 256;
__global__ void __launch_bounds__(SE_NT)
    shadow_encode_kernel(const float* __restrict__ rows, int64_t ld, int64_t n, int cols, int cols16,
                         unsigned char* __restrict__ out, int64_t out_stride) {
  const int64_t r = (int64_t)blockIdx.x * (SE_NT / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const float* y = rows + r * ld;
  unsigned char* o = out + r * out_stride;
  float amax = 0.f;
  bool bad = false;
  for (int i = lane; i < cols; i += 32) {
    const float v = y[i];
    bad |= !isfinite(v);
    amax = fmaxf(amax, fabsf(v));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  bad = __any_sync(0xffffffffu, bad);
  const float s = __fdiv_rn(amax, 127.0f);
  const bool ok = !bad && s > 0.f && isfinite(s);
  double e2 = 0.0, n2 = 0.0;
  for (int i = lane; i < cols16; i += 32) {
    float qv = 0.f;
    if (ok && i < cols) {
      qv = fminf(127.f, fmaxf(-127.f, rintf(__fdiv_rn(y[i], s))));
      const double t = (double)y[i] - (double)s * (double)qv;  // s qv is exact in fp64
      e2 += t * t;
      n2 += (double)qv * (double)qv;  // exact
    }
    o[i] = (unsigned char)(signed char)(int)qv;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    e2 += __shfl_xor_sync(0xffffffffu, e2, off);
    n2 += __shfl_xor_sync(0xffffffffu, n2, off);
  }
  if (lane == 0) {
    float4 m = make_float4(0.f, __int_as_float(0x7F800000), __int_as_float(0x7F800000), 0.f);
    if (ok) {
      // e2 is within (cols + 5) 2^-53 of the exact sum: the factor 1 + 2^-30 covers that for any row width here
      m.x = s;
      m.y = __double2float_ru(__dmul_ru(__dsqrt_ru(e2), 1.0 + 0x1p-30));
      m.z = __double2float_ru(__dmul_ru((double)s, __dsqrt_ru(n2)));
    }
    *reinterpret_cast<float4*>(o + cols16) = m;
  }
}

// ---------------- PQ encode -------------------------------------------------------------------
constexpr int ENC_NT = 256;
constexpr int ENC_MAX_DSUB = 128;

template <int DSUB>
__global__ void __launch_bounds__(ENC_NT)
    pq_encode_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, const float* __restrict__ coarse, int64_t ldc,
                     const int32_t* __restrict__ assign, const float* __restrict__ pq, int M, int dsub_rt, int ksub,
                     uint8_t* __restrict__ codes) {
  extern __shared__ float ps[];  // [ksub][dsub]
  const int dsub = DSUB > 0 ? DSUB : dsub_rt;
  const int m = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * ENC_NT + threadIdx.x;
  for (int idx = threadIdx.x; idx < ksub * dsub; idx += ENC_NT) ps[idx] = pq[(int64_t)m * ksub * dsub + idx];
  __syncthreads();
  if (i >= n) return;
  float r[DSUB > 0 ? DSUB : ENC_MAX_DSUB];
  const float* xi = x + i * ldx + m * dsub;
  const float* ci = (coarse && assign[i] >= 0) ? coarse + (int64_t)assign[i] * ldc + m * dsub : nullptr;
#pragma unroll
  for (int j = 0; j < dsub; j++) r[j] = ci ? __fsub_rn(xi[j], ci[j]) : xi[j];
  float best = FLT_MAX;
  int bi = 0;
  for (int c = 0; c < ksub; c++) {
    float dis = 0.f;
#pragma unroll
    for (int j = 0; j < dsub; j++) {
      float t = __fsub_rn(r[j], ps[c * dsub + j]);
      dis = __fadd_rn(dis, __fmul_rn(t, t));
    }
    if (dis < best) {
      best = dis;
      bi = c;
    }
  }
  codes[i * M + m] = (uint8_t)bi;
}

// one thread per row: [n][M] codes -> [n][ceil(M nbits / 8)] bit-packed rows (PQEncoderGeneric's layout)
__global__ void pq_pack_codes_kernel(const uint8_t* __restrict__ codes, int64_t n, int M, int nbits,
                                     uint8_t* __restrict__ packed) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* src = codes + i * M;
  const int cs = (M * nbits + 7) / 8;
  uint8_t* dst = packed + i * cs;
  uint32_t bits = 0;
  int nb = 0, o = 0;
  for (int m = 0; m < M; m++) {
    bits |= (uint32_t)src[m] << nb;
    nb += nbits;
    while (nb >= 8) {
      dst[o++] = (uint8_t)bits;
      bits >>= 8;
      nb -= 8;
    }
  }
  if (nb > 0) dst[o] = (uint8_t)bits;
}

}  // namespace

cudaError_t launch_pq_ip_table(const float* xq, int64_t ldq, int nq, const float* pq_centroids, int M, int dsub,
                               float* ip, cudaStream_t st, int ksub) {
  if (nq <= 0) return cudaSuccess;
  if (ksub < 2 || ksub > KSUB || (ksub & (ksub - 1))) return cudaErrorInvalidValue;
  size_t smem = ((size_t)dsub * ksub + (size_t)IPT_QB * dsub) * 4;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(pq_ip_table_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  dim3 grid(M, (nq + IPT_QB - 1) / IPT_QB);
  pq_ip_table_kernel<<<grid, KSUB, smem, st>>>(xq, ldq, nq, pq_centroids, M, dsub, ksub, ip);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pq_precompute_table(const float* coarse, int64_t ldc, int nlist, const float* pq_centroids, int M,
                                       int dsub, float* T, cudaStream_t st, int ksub) {
  if (nlist <= 0) return cudaSuccess;
  if (ksub < 1 || ksub > KSUB) return cudaErrorInvalidValue;
  pq_precompute_table_kernel<<<nlist, KSUB, 0, st>>>(coarse, ldc, pq_centroids, M, dsub, ksub, T);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_ivfpq_scan(const float* ip_table, int nq, const int32_t* probe_ids, const float* coarse_dis,
                              int nprobe, int pg, ListDirectory dir, int M, const float* T, int k, int metric,
                              FilterArgs f, unsigned long long* partial, cudaStream_t st, int ld_probe,
                              const int* gate_cnt, int gate_cap, const int* row_limit, bool sorted_out) {
  if (metric == kMetricL2 && !T) return cudaErrorInvalidValue;
  const IvfpqCodec c{ip_table, T, M, nullptr};
  const ListScanArgs a{probe_ids, coarse_dis, nprobe, ld_probe > 0 ? ld_probe : nprobe, pg, dir, k, f,
                       gate_cnt, gate_cap, row_limit, sorted_out, partial};
  if (metric == kMetricL2) return launch_scan_m<kMetricL2>(c, nq, a, st);
  return launch_scan_m<kMetricIP>(c, nq, a, st);
}

int ivfpq_scan_max_k(int M, int nbits) {
  if (M <= 0 || nbits < 1 || nbits > 8) return 0;
  if (nbits == 8) return list_scan_max_k(IvfpqCodec{nullptr, nullptr, M, nullptr});
  return list_scan_max_k(IvfpqPackedCodec{nullptr, nullptr, M, nbits, nullptr});
}

cudaError_t launch_ivfpq_packed_scan(const float* ip_table, int nq, const int32_t* probe_ids, const float* coarse_dis,
                                     int nprobe, int pg, ListDirectory dir, int M, int nbits, const float* T, int k,
                                     int metric, FilterArgs f, unsigned long long* partial, cudaStream_t st) {
  if ((metric == kMetricL2 && !T) || nbits < 1 || nbits > 7) return cudaErrorInvalidValue;
  const IvfpqPackedCodec c{ip_table, T, M, nbits, nullptr};
  const ListScanArgs a{probe_ids, coarse_dis, nprobe, nprobe, pg, dir, k, f, nullptr, 0, nullptr, true, partial};
  if (metric == kMetricL2) return launch_list_scan<IvfpqPackedCodec, kMetricL2, 0>(c, nq, a, st);
  return launch_list_scan<IvfpqPackedCodec, kMetricIP, 0>(c, nq, a, st);
}

// A launch's dynamic shared memory past 48 KiB, together with the kernel's static shared memory (the two-pass
// kernel's radix-select histogram), needs the kernel's opt-in: without it a launch at, e.g., d = 4096 and 2048
// candidates (exactly 48 KiB dynamic) is refused
template <class K>
static cudaError_t rr_opt_in_smem(K kern, size_t smem) {
  cudaFuncAttributes fa;
  if (cudaError_t e = cudaFuncGetAttributes(&fa, kern)) return e;
  if (smem + fa.sharedSizeBytes <= 48 * 1024) return cudaSuccess;
  return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

cudaError_t launch_rerank(const unsigned long long* cand_keys, int ncand, int nq, const float* xq, int64_t ldq, int d,
                          const float* const* raw_segments, int seg_shift, int64_t ld_raw, bool host_rows, int k,
                          int metric, FilterArgs f, unsigned long long* out_keys, cudaStream_t st) {
  if (nq <= 0) return cudaSuccess;
  if (ncand <= 0 || ncand > 8192 || (d & 3)) return cudaErrorInvalidValue;
  int NP = next_pow2(ncand < 2 ? 2 : ncand);  // >= 16 bytes of keys: the query row behind them is read as float4
  size_t smem = (size_t)NP * 8 + (size_t)d * 4;
  auto kern = host_rows ? rerank_kernel<8> : rerank_kernel<4>;
  if (cudaError_t e = rr_opt_in_smem(kern, smem)) return e;
  kern<<<nq, RR_NT, smem, st>>>(cand_keys, ncand, NP, xq, ldq, d, raw_segments, seg_shift, ld_raw, k, metric, f,
                                out_keys);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_rerank_prefilter(const unsigned long long* cand_keys, int ncand, int nq, const float* xq, int64_t ldq,
                                    int d, const float* const* raw_segments, int seg_shift, int64_t ld_raw,
                                    const unsigned char* const* shadow_segs, int64_t shadow_stride, int k, int metric,
                                    FilterArgs f, unsigned long long* out_keys, int* survivors, cudaStream_t st,
                                    uint4* intervals) {
  if (nq <= 0) return cudaSuccess;
  const int cols16 = (d + 15) & ~15;
  if (ncand <= 0 || ncand > 8192 || k <= 0 || k > ncand || (d & 3) || shadow_stride != cols16 + 16)
    return cudaErrorInvalidValue;
  const int NP = next_pow2(ncand < 2 ? 2 : ncand);
  const size_t smem = (size_t)NP * 8 + (size_t)cols16 * 4 + (size_t)NP * 8;
  auto kern = metric == kMetricL2 ? (intervals ? rerank_prefilter_kernel<kMetricL2, true>
                                               : rerank_prefilter_kernel<kMetricL2, false>)
                                  : (intervals ? rerank_prefilter_kernel<kMetricIP, true>
                                               : rerank_prefilter_kernel<kMetricIP, false>);
  if (cudaError_t e = rr_opt_in_smem(kern, smem)) return e;
  kern<<<nq, RR_NT, smem, st>>>(cand_keys, ncand, NP, xq, ldq, d, raw_segments, seg_shift, ld_raw, shadow_segs,
                                shadow_stride, cols16, k, f, out_keys, survivors, intervals);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_shadow_encode(const float* rows, int64_t ld, int64_t n, int cols, unsigned char* out,
                                 int64_t out_stride, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  const int cols16 = (cols + 15) & ~15;
  if (out_stride != cols16 + 16) return cudaErrorInvalidValue;
  const int64_t rows_per_cta = SE_NT / 32;
  shadow_encode_kernel<<<(unsigned)((n + rows_per_cta - 1) / rows_per_cta), SE_NT, 0, st>>>(rows, ld, n, cols, cols16, out,
                                                                                           out_stride);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pq_encode(const float* x, int64_t ldx, int64_t n, const float* coarse, int64_t ldc,
                             const int32_t* assign, const float* pq_centroids, int M, int dsub, uint8_t* codes,
                             cudaStream_t st, int ksub) {
  if (n <= 0) return cudaSuccess;
  if (dsub > ENC_MAX_DSUB || ksub < 1 || ksub > KSUB) return cudaErrorInvalidValue;
  size_t smem = (size_t)ksub * dsub * 4;
  dim3 grid((unsigned)((n + ENC_NT - 1) / ENC_NT), M);
#define GB_ENC(DS)                                                                                               \
  {                                                                                                              \
    if (smem > 48 * 1024) {                                                                                      \
      cudaError_t e =                                                                                            \
          cudaFuncSetAttribute(pq_encode_kernel<DS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);     \
      if (e != cudaSuccess) return e;                                                                            \
    }                                                                                                            \
    pq_encode_kernel<DS><<<grid, ENC_NT, smem, st>>>(x, ldx, n, coarse, ldc, assign, pq_centroids, M, dsub, ksub, codes); \
    note_launch(); \
  }
  switch (dsub) {
    case 2: GB_ENC(2) break;
    case 4: GB_ENC(4) break;
    case 8: GB_ENC(8) break;
    case 16: GB_ENC(16) break;
    case 32: GB_ENC(32) break;
    default: GB_ENC(0) break;
  }
#undef GB_ENC
  return cudaGetLastError();
}

cudaError_t launch_pq_pack_codes(const uint8_t* codes, int64_t n, int M, int nbits, uint8_t* packed, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  if (nbits < 1 || nbits > 8) return cudaErrorInvalidValue;
  pq_pack_codes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(codes, n, M, nbits, packed);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
