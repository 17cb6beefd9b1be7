// IVFPQFastScan: 4-bit PQ encode, per-query uint8 look-up table, and the query-major scan that sums it.
//
// Replaces, in the reference (index/impl/gamma_index_ivfpqfs.{h,cc}, a faiss::IndexIVFPQFastScan with
// by_residual = false):
//   pq.compute_codes with ksub = 16, packed by BitstringWriter                     -> pqfs_encode
//   compute_float_LUT + quantize_lut::round_uint8_per_column (faiss v1.14.1)     -> pqfs_lut
//   the fast-scan accumulation + de-quantisation of IndexIVFFastScan::search     -> ivfpqfs_scan
//
// Codes: sub-quantiser 2j in the low nibble of byte j, 2j + 1 in the high nibble; an odd M leaves the last
// high nibble 0.  Table arithmetic is unfused (__fmul_rn / __fadd_rn) in the order of the IVF-PQ table kernels,
// so the uint8 table and (a, b) are bit-equal to a scalar CPU evaluation.  After quantisation everything is
// integer until the final  accu * (1 / a) + b,  which is evaluated unfused in that order.
#include <float.h>

#include "common.cuh"
#include "kernels.h"
#include "list_scan.cuh"

namespace gb {

namespace {

constexpr int FS_KSUB = 16;

// ---------------- encode: one thread per (vector, code byte) -------------------------------------------------
__global__ void pqfs_encode_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, const float* __restrict__ pq, int M,
                                   int dsub, int MB, uint8_t* __restrict__ codes) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * MB) return;
  const int64_t i = t / MB;
  const int j = (int)(t - i * MB);
  uint32_t out = 0;
  for (int h = 0; h < 2; h++) {
    const int m = 2 * j + h;
    if (m >= M) break;
    const float* xi = x + i * ldx + (int64_t)m * dsub;
    const float* c = pq + (int64_t)m * FS_KSUB * dsub;
    float best = FLT_MAX;
    int bi = 0;
    for (int cc = 0; cc < FS_KSUB; cc++) {  // same distance form as pq_encode_kernel; lowest index wins ties
      float dis = 0.f;
      for (int jj = 0; jj < dsub; jj++) {
        const float tt = __fsub_rn(xi[jj], __ldg(c + cc * dsub + jj));
        dis = __fadd_rn(dis, __fmul_rn(tt, tt));
      }
      if (dis < best) {
        best = dis;
        bi = cc;
      }
    }
    out |= (uint32_t)bi << (4 * h);
  }
  codes[t] = (uint8_t)out;
}

// ---------------- per-query table, quantised to uint8 ------------------------------------------------------
constexpr int LUT_NT = 256;

__global__ void __launch_bounds__(LUT_NT)
    pqfs_lut_kernel(const float* __restrict__ xq, int64_t ldq, const float* __restrict__ pq, int M, int dsub, int metric,
                    uint8_t* __restrict__ lut8, float* __restrict__ ab) {
  extern __shared__ float tab[];  // [M][16], then mins[M], spans[M]
  float* mins = tab + M * FS_KSUB;
  float* spans = mins + M;
  __shared__ float s_a;
  const int q = blockIdx.x, tid = threadIdx.x;
  const float* x = xq + (int64_t)q * ldq;
  for (int i = tid; i < M * FS_KSUB; i += LUT_NT) {
    const int m = i / FS_KSUB;
    const float* c = pq + (int64_t)i * dsub;
    const float* xm = x + m * dsub;
    float acc = 0.f;
    if (metric == kMetricL2) {
      for (int j = 0; j < dsub; j++) {
        const float t = __fsub_rn(xm[j], __ldg(c + j));
        acc = __fadd_rn(acc, __fmul_rn(t, t));
      }
    } else {
      for (int j = 0; j < dsub; j++) acc = __fadd_rn(acc, __fmul_rn(xm[j], __ldg(c + j)));
    }
    tab[i] = acc;
  }
  __syncthreads();
  for (int m = tid; m < M; m += LUT_NT) {  // tab_min / tab_max
    float mn = FLT_MAX, mx = -FLT_MAX;
    for (int c = 0; c < FS_KSUB; c++) {
      const float v = tab[m * FS_KSUB + c];
      if (v < mn) mn = v;
      if (v > mx) mx = v;
    }
    mins[m] = mn;
    spans[m] = __fsub_rn(mx, mn);
  }
  __syncthreads();
  if (tid == 0) {
    float max_span = 0.f, b = 0.f;
    for (int m = 0; m < M; m++) {
      if (spans[m] > max_span) max_span = spans[m];
      b = __fadd_rn(b, mins[m]);
    }
    // every span 0 (all entries of every sub-quantiser equal): faiss divides by zero here; a = 1 keeps the table 0
    s_a = max_span > 0.f ? __fdiv_rn(255.f, max_span) : 1.f;
    ab[2 * q] = s_a;
    ab[2 * q + 1] = b;
  }
  __syncthreads();
  const float a = s_a;
  for (int i = tid; i < M * FS_KSUB; i += LUT_NT) {
    const float v = floorf(__fadd_rn(__fmul_rn(__fsub_rn(tab[i], mins[i / FS_KSUB]), a), 0.5f));
    lut8[(int64_t)q * M * FS_KSUB + i] = (uint8_t)v;
  }
}

// ---------------- scan: the IVFPQFastScan codec of the list scan (list_scan.cuh) ---------------------------
// entries per tile: 16 KiB of codes, between 256 and 1024 entries (a multiple of LS_NT)
__host__ __device__ constexpr int pqfs_tile_entries(int MB) {
  const int e = 16384 / MB / LS_NT * LS_NT;
  return e < LS_NT ? LS_NT : (e > 1024 ? 1024 : e);
}

// The table does not depend on the list (no residual), so the CTA builds the byte-pair table
// T[j][byte] = lut8[2j][lo] + lut8[2j+1][hi] once.  accu = sum_j T[j][code byte j]: uint16 pair entries summed in 32 bits;
// faiss sums 16-bit, which wraps only above 257 sub-quantisers (255 * 257 < 2^16); the index accepts M <= 256
// (IVFPQFastScanIndex::kMaxM), so both are equal.  Score accu * (1 / a) + b.
struct IvfpqfsCodec {
  using Entry = uint16_t;
  static constexpr bool kDis0 = false;
  // 40 registers: for M <= 12 shared memory admits 6 or 7 CTAs per SM
  static constexpr int kMinCtasPerSm = 6;
  const uint8_t* lut8;  // [nq][M][16]
  const float* ab;      // [nq][2]
  int M;
  float one_a, b;  // this CTA's query

  __host__ __device__ int code_bytes() const { return (M + 1) / 2; }
  int tile_entries() const { return pqfs_tile_entries(code_bytes()); }
  __host__ __device__ static constexpr int pt(int MW) { return pqfs_tile_entries(4 * MW) / LS_NT; }

  __device__ __forceinline__ void cta_begin(uint16_t* T, int q, int metric) {
    (void)metric;
    const uint8_t* lq = lut8 + (int64_t)q * M * FS_KSUB;
    for (int i = threadIdx.x; i < code_bytes() * 256; i += LS_NT) {
      const int j = i >> 8, lo = i & 15, hi = (i >> 4) & 15;
      T[i] = (uint16_t)(lq[2 * j * FS_KSUB + lo] + (2 * j + 1 < M ? lq[(2 * j + 1) * FS_KSUB + hi] : 0));
    }
    one_a = __fdiv_rn(1.f, ab[2 * q]);
    b = ab[2 * q + 1];
    __syncthreads();
  }
  __device__ __forceinline__ void list_begin(uint16_t* T, int list, int metric) const {
    (void)T, (void)list, (void)metric;
  }
  using Acc = uint32_t;
  __device__ __forceinline__ uint32_t start(float dis0) const { (void)dis0; return 0u; }
  __device__ __forceinline__ float finish(uint32_t accu) const { return __fadd_rn(__fmul_rn((float)accu, one_a), b); }
};

template <int METRIC>
cudaError_t launch_scan_m(const IvfpqfsCodec& c, int nq, const ListScanArgs& a, cudaStream_t st) {
  switch (c.code_bytes()) {
    case 4: return launch_list_scan<IvfpqfsCodec, METRIC, 1>(c, nq, a, st);
    case 8: return launch_list_scan<IvfpqfsCodec, METRIC, 2>(c, nq, a, st);
    case 16: return launch_list_scan<IvfpqfsCodec, METRIC, 4>(c, nq, a, st);
    case 32: return launch_list_scan<IvfpqfsCodec, METRIC, 8>(c, nq, a, st);
    default: return launch_list_scan<IvfpqfsCodec, METRIC, 0>(c, nq, a, st);
  }
}

}  // namespace

cudaError_t launch_pqfs_encode(const float* x, int64_t ldx, int64_t n, const float* pq_centroids, int M, int dsub, uint8_t* codes,
                               cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  const int64_t work = n * ((M + 1) / 2);
  pqfs_encode_kernel<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(x, ldx, n, pq_centroids, M, dsub, (M + 1) / 2, codes);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pqfs_lut(const float* xq, int64_t ldq, int nq, const float* pq_centroids, int M, int dsub, int metric,
                            uint8_t* lut8, float* ab, cudaStream_t st) {
  if (nq <= 0) return cudaSuccess;
  const size_t smem = ((size_t)M * FS_KSUB + 2 * (size_t)M) * 4;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(pqfs_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  pqfs_lut_kernel<<<nq, LUT_NT, smem, st>>>(xq, ldq, pq_centroids, M, dsub, metric, lut8, ab);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_ivfpqfs_scan(const uint8_t* lut8, const float* ab, int nq, const int32_t* probe_ids, int nprobe, int pg,
                                ListDirectory dir, int M, int k, int metric, FilterArgs f, unsigned long long* partial,
                                cudaStream_t st) {
  const IvfpqfsCodec c{lut8, ab, M, 0.f, 0.f};
  const ListScanArgs a{probe_ids, nullptr, nprobe, nprobe, pg, dir, k, f, nullptr, 0, nullptr, true, partial};
  if (metric == kMetricL2) return launch_scan_m<kMetricL2>(c, nq, a, st);
  return launch_scan_m<kMetricIP>(c, nq, a, st);
}

}  // namespace gb
