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

// ---------------- scan ---------------------------------------------------------------------------------------
constexpr int FS_NT = 256;
constexpr int FS_NST = 2;
constexpr int FS_MAX_PG = 32;  // probes per CTA

// entries per tile: 16 KiB of codes, between 256 and 1024 entries (a multiple of FS_NT)
__host__ __device__ constexpr int pqfs_tile_entries(int MB) {
  const int e = 16384 / MB / FS_NT * FS_NT;
  return e < FS_NT ? FS_NT : (e > 1024 ? 1024 : e);
}

// accu = sum_j T[j][code byte j].  uint16 pair entries summed in 32 bits: faiss sums 16-bit, which wraps only above
// 257 sub-quantisers (255 * 257 < 2^16); the index accepts M <= 256 (IVFPQFastScanIndex::kMaxM), so both are equal.
template <int MW>
__device__ __forceinline__ uint32_t pqfs_accu(const unsigned char* __restrict__ code, const uint16_t* __restrict__ T, int MB) {
  uint32_t accu = 0;
  if (MW > 0) {
    uint32_t w[MW > 0 ? MW : 1];
    if (MW % 4 == 0) {
#pragma unroll
      for (int i = 0; i < MW / 4; i++) {
        const uint4 v = reinterpret_cast<const uint4*>(code)[i];
        w[4 * i] = v.x, w[4 * i + 1] = v.y, w[4 * i + 2] = v.z, w[4 * i + 3] = v.w;
      }
    } else if (MW % 2 == 0) {
#pragma unroll
      for (int i = 0; i < MW / 2; i++) {
        const uint2 v = reinterpret_cast<const uint2*>(code)[i];
        w[2 * i] = v.x, w[2 * i + 1] = v.y;
      }
    } else {
#pragma unroll
      for (int i = 0; i < MW; i++) w[i] = reinterpret_cast<const uint32_t*>(code)[i];
    }
#pragma unroll
    for (int i = 0; i < MW; i++) {
      const uint32_t x = w[i];
      accu += T[(4 * i + 0) * 256 + (x & 0xffu)];
      accu += T[(4 * i + 1) * 256 + ((x >> 8) & 0xffu)];
      accu += T[(4 * i + 2) * 256 + ((x >> 16) & 0xffu)];
      accu += T[(4 * i + 3) * 256 + (x >> 24)];
    }
  } else {
    for (int j = 0; j < MB; j++) accu += T[j * 256 + code[j]];
  }
  return accu;
}

// One CTA per (query, group of pg probes): a TMA bulk ring over the flat (list, tile) sequence of its probes.  The table
// does not depend on the list (no residual), so the byte-pair table T[j][byte] = lut8[2j][lo] + lut8[2j+1][hi] is built
// once per CTA.
template <int METRIC, int MW>
__global__ void __launch_bounds__(FS_NT)
    ivfpqfs_scan_kernel(const uint8_t* __restrict__ lut8, const float* __restrict__ ab, const int32_t* __restrict__ probe_ids,
                        int nprobe, int pg, ListDirectory dir, int M, int MB, int tile_e, int k, int KP, int SORTN, FilterArgs f,
                        unsigned long long* __restrict__ partial) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int tile_bytes = tile_e * MB;
  uint16_t* T = reinterpret_cast<uint16_t*>(smem_raw);  // [MB][256]
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(smem_raw + (size_t)MB * 512);
  unsigned char* stages = reinterpret_cast<unsigned char*>(buf + SORTN);
  __shared__ __align__(8) uint64_t full_bar[FS_NST];
  __shared__ int s_cnt;
  __shared__ unsigned long long s_tau;
  __shared__ int g_list[FS_MAX_PG], g_len[FS_MAX_PG], g_tile0[FS_MAX_PG + 1];

  const int tid = threadIdx.x;
  const int q = blockIdx.y, grp = blockIdx.x;
  unsigned long long* out = partial + ((int64_t)q * gridDim.x + grp) * k;
  const int p0 = grp * pg;
  const int np = min(pg, nprobe - p0);

  if (tid == 0) {
    int acc = 0;
    for (int i = 0; i < np; i++) {
      const int l = probe_ids[(int64_t)q * nprobe + p0 + i];
      const int len = (l >= 0 && l < dir.nlist) ? dir.len[l] : 0;
      g_list[i] = l;
      g_len[i] = len;
      g_tile0[i] = acc;
      acc += (len + tile_e - 1) / tile_e;
    }
    g_tile0[np > 0 ? np : 0] = acc;
    for (int s = 0; s < FS_NST; s++) mbar_init(&full_bar[s], 1);
    mbar_fence_init();
  }
  CandQueue cq{buf, &s_cnt, &s_tau, k, KP, SORTN};
  cq.init();  // __syncthreads inside: g_* and barriers visible
  const int total_tiles = np > 0 ? g_tile0[np] : 0;
  if (total_tiles == 0) {
    for (int i = tid; i < k; i += FS_NT) out[i] = kKeySentinel;
    return;
  }

  int pr_pi = 0;  // producer cursor (thread 0 only)
  auto issue = [&](int gt) {
    while (gt >= g_tile0[pr_pi + 1]) pr_pi++;
    const int ti = gt - g_tile0[pr_pi];
    const int n_e = min(tile_e, g_len[pr_pi] - ti * tile_e);
    const uint32_t bytes = ((uint32_t)n_e * MB + 15u) & ~15u;
    const int s = gt % FS_NST;
    mbar_arrive_expect_tx(&full_bar[s], bytes);
    bulk_g2s(stages + (size_t)s * tile_bytes, dir.codes[g_list[pr_pi]] + (int64_t)ti * tile_e * MB, bytes, &full_bar[s]);
  };
  if (tid == 0)
    for (int gt = 0; gt < FS_NST && gt < total_tiles; gt++) issue(gt);

  const uint8_t* lq = lut8 + (int64_t)q * M * FS_KSUB;
  for (int i = tid; i < MB * 256; i += FS_NT) {
    const int j = i >> 8, lo = i & 15, hi = (i >> 4) & 15;
    T[i] = (uint16_t)(lq[2 * j * FS_KSUB + lo] + (2 * j + 1 < M ? lq[(2 * j + 1) * FS_KSUB + hi] : 0));
  }
  const float one_a = __fdiv_rn(1.f, ab[2 * q]), b = ab[2 * q + 1];
  __syncthreads();

  int pi = -1;  // consumer cursor
  const int64_t* __restrict__ lids = nullptr;
  constexpr int PT = MW > 0 ? pqfs_tile_entries(4 * MW) / FS_NT : 1;
  const int per_thread = MW > 0 ? PT : tile_e / FS_NT;
  int est = 0;  // upper bound of the queue fill, identical in every thread

  for (int gt = 0; gt < total_tiles; gt++) {
    int npi = pi < 0 ? 0 : pi;
    while (gt >= g_tile0[npi + 1]) npi++;
    if (npi != pi) {
      pi = npi;
      lids = dir.ids[g_list[pi]];
    }
    const int ti = gt - g_tile0[pi];
    const int n_e = min(tile_e, g_len[pi] - ti * tile_e);
    const int s = gt % FS_NST;
    mbar_wait(&full_bar[s], (gt / FS_NST) & 1);
    const unsigned long long tau = s_tau;
    const float tb = key_bound<METRIC>(tau);
    const float lo_b = METRIC == kMetricL2 ? f.min_score : fmaxf(tb, f.min_score);
    const float hi_b = METRIC == kMetricL2 ? fminf(tb, f.max_score) : f.max_score;
    const unsigned char* st = stages + (size_t)s * tile_bytes;
    int pushed = 0;

    auto consider = [&](int e, float dis) {
      bool pred = e < n_e && dis <= hi_b && dis >= lo_b;
      unsigned long long key = kKeySentinel;
      if (pred) {
        const int64_t raw = lids[(int64_t)ti * tile_e + e];
        pred = raw >= 0;  // tombstone
        const uint32_t vid = (uint32_t)raw;
        if (pred) pred = ctx_is_valid(f.del_bits, f.filter_bits, vid);
        key = make_key(score2ord<METRIC>(dis), vid);
        pred = pred && key < tau;
      }
      cq.push_warp(pred, key);
      pushed |= pred ? 1 : 0;
    };
    auto score = [&](uint32_t accu) { return __fadd_rn(__fmul_rn((float)accu, one_a), b); };
    if (MW > 0) {
      uint32_t accu[PT];
#pragma unroll
      for (int u = 0; u < PT; u++) accu[u] = pqfs_accu<MW>(st + (size_t)(u * FS_NT + tid) * MB, T, MB);  // stale bytes past n_e are masked
#pragma unroll
      for (int u = 0; u < PT; u++) consider(u * FS_NT + tid, score(accu[u]));
    } else {
      for (int u = 0; u < per_thread; u++) {
        const int e = u * FS_NT + tid;
        consider(e, e < n_e ? score(pqfs_accu<0>(st + (size_t)e * MB, T, MB)) : 0.f);
      }
    }
    est += __syncthreads_count(pushed) * per_thread;  // stage consumed + pushes done
    if (tid == 0 && gt + FS_NST < total_tiles) issue(gt + FS_NST);
    if (gt + 1 < total_tiles && est + tile_e > cq.cap()) {
      cq.flush();
      est = 0;
    }
  }
  __syncthreads();
  cq.flush(true);
  for (int i = tid; i < k; i += FS_NT) out[i] = buf[i];
}

template <int METRIC, int MW>
cudaError_t launch_scan_t(const uint8_t* lut8, const float* ab, int nq, const int32_t* probe_ids, int nprobe, int pg,
                          ListDirectory dir, int M, int k, FilterArgs f, unsigned long long* partial, cudaStream_t st) {
  const int MB = (M + 1) / 2;
  const int tile_e = pqfs_tile_entries(MB);
  const int KP = next_pow2(k < 16 ? 16 : k);
  const int SORTN = next_pow2(KP + tile_e + tile_e / 2);  // cap >= tile_e: one tile always fits after a flush
  const size_t smem = (size_t)MB * 512 + (size_t)SORTN * 8 + (size_t)FS_NST * tile_e * MB;
  if (smem > 227 * 1024) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(ivfpqfs_scan_kernel<METRIC, MW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  dim3 grid((nprobe + pg - 1) / pg, nq);
  ivfpqfs_scan_kernel<METRIC, MW><<<grid, FS_NT, smem, st>>>(lut8, ab, probe_ids, nprobe, pg, dir, M, MB, tile_e, k, KP, SORTN,
                                                             f, partial);
  note_launch();
  return cudaGetLastError();
}

template <int METRIC>
cudaError_t launch_scan_m(const uint8_t* lut8, const float* ab, int nq, const int32_t* probe_ids, int nprobe, int pg,
                          ListDirectory dir, int M, int k, FilterArgs f, unsigned long long* partial, cudaStream_t st) {
#define GB_FS(MW) return launch_scan_t<METRIC, MW>(lut8, ab, nq, probe_ids, nprobe, pg, dir, M, k, f, partial, st)
  switch ((M + 1) / 2) {  // code bytes
    case 4: GB_FS(1);
    case 8: GB_FS(2);
    case 16: GB_FS(4);
    case 32: GB_FS(8);
    default: GB_FS(0);
  }
#undef GB_FS
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
  if (nq <= 0 || nprobe <= 0) return cudaSuccess;
  if (k <= 0 || k > 4096 || nq > 65535 || pg < 1 || pg > FS_MAX_PG) return cudaErrorInvalidValue;
  if (metric == kMetricL2) return launch_scan_m<kMetricL2>(lut8, ab, nq, probe_ids, nprobe, pg, dir, M, k, f, partial, st);
  return launch_scan_m<kMetricIP>(lut8, ab, nq, probe_ids, nprobe, pg, dir, M, k, f, partial, st);
}

}  // namespace gb
