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

// RR_U: candidates a warp gathers per iteration.  Four keep 2 KiB of independent row loads in flight per warp, which
// covers HBM latency (eight cost occupancy; the gather is pure latency: recall_num random 4d-byte rows per query).
// Rows in mapped host memory come over PCIe, whose round trip is several times longer: eight per warp there.
template <int RR_U>
__global__ void __launch_bounds__(RR_NT)
    rerank_kernel(const unsigned long long* __restrict__ cand_keys, int ncand, int NP, const float* __restrict__ xq,
                  int64_t ldq, int d, const float* const* __restrict__ raw_segments, int seg_shift, int64_t ld_raw,
                  int k, int metric, FilterArgs f, unsigned long long* __restrict__ out_keys) {
  extern __shared__ __align__(16) unsigned char rr_smem[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(rr_smem);  // [NP]
  float* qs = reinterpret_cast<float*>(buf + NP);                              // [d]
  const int q = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < d; i += RR_NT) qs[i] = xq[(int64_t)q * ldq + i];
  for (int i = threadIdx.x; i < NP; i += RR_NT) buf[i] = kKeySentinel;
  __syncthreads();
  const float4* q4 = reinterpret_cast<const float4*>(qs);
  const uint32_t seg_mask = (1u << seg_shift) - 1u;
  for (int j0 = warp * RR_U; j0 < ncand; j0 += (RR_NT / 32) * RR_U) {
    uint32_t vid[RR_U];
    const float4* row[RR_U];
    bool live[RR_U];
#pragma unroll
    for (int u = 0; u < RR_U; u++) {
      const int j = j0 + u;
      const unsigned long long ck = j < ncand ? cand_keys[(int64_t)q * ncand + j] : kKeySentinel;
      live[u] = ck != kKeySentinel;  // recall_idxi[j] < 0 (ivfpq.cc:691)
      vid[u] = live[u] ? (uint32_t)ck : 0u;
      row[u] = live[u] ? reinterpret_cast<const float4*>(raw_segments[vid[u] >> seg_shift] + (int64_t)(vid[u] & seg_mask) * ld_raw)
                       : nullptr;
    }
    float acc[RR_U][4];
#pragma unroll
    for (int u = 0; u < RR_U; u++) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0.f;
    for (int c = lane; c < (d >> 2); c += 32) {
      const float4 w = q4[c];
      float4 v[RR_U];
#pragma unroll
      for (int u = 0; u < RR_U; u++) v[u] = live[u] ? __ldg(row[u] + c) : make_float4(0.f, 0.f, 0.f, 0.f);
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
      float dis = (acc[u][0] + acc[u][1]) + (acc[u][2] + acc[u][3]);
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) dis += __shfl_xor_sync(0xffffffffu, dis, off);
      if (lane == 0 && live[u] && dis <= f.max_score && dis >= f.min_score) buf[j0 + u] = make_key(score2ord(dis, metric), vid[u]);
    }
  }
  __syncthreads();
  block_bitonic_sort(buf, NP);
  for (int i = threadIdx.x; i < k; i += RR_NT) out_keys[(int64_t)q * k + i] = i < NP ? buf[i] : kKeySentinel;
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

cudaError_t launch_rerank(const unsigned long long* cand_keys, int ncand, int nq, const float* xq, int64_t ldq, int d,
                          const float* const* raw_segments, int seg_shift, int64_t ld_raw, bool host_rows, int k,
                          int metric, FilterArgs f, unsigned long long* out_keys, cudaStream_t st) {
  if (nq <= 0) return cudaSuccess;
  if (ncand <= 0 || ncand > 8192 || (d & 3)) return cudaErrorInvalidValue;
  int NP = next_pow2(ncand < 2 ? 2 : ncand);  // >= 16 bytes of keys: the query row behind them is read as float4
  size_t smem = (size_t)NP * 8 + (size_t)d * 4;
  auto kern = host_rows ? rerank_kernel<8> : rerank_kernel<4>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  kern<<<nq, RR_NT, smem, st>>>(cand_keys, ncand, NP, xq, ldq, d, raw_segments, seg_shift, ld_raw, k, metric, f,
                                out_keys);
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
