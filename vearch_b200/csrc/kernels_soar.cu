// SOAR spilling (DESIGN.md §8): the spilled-list choice at add time and the duplicate-free selection at search time.
//
// Spilled list of a row x with primary list a (r = x - c_a, r' = x - c'), over every list c' != a:
//   loss(c') = |r'|^2 + lambda <r, r'>^2 / |r|^2,   the smallest loss, the lower list id among equals
// (Sun et al., "SOAR: improved indexing for approximate nearest neighbor search", NeurIPS 2023, eq. 7).
#include "common.cuh"
#include "kernels.h"

namespace gb {

namespace {

constexpr int kSoarRows = 32;   // rows per CTA: 8 warps x 4 rows
constexpr int kSoarCols = 64;   // centroids per tile: 32 lanes x 2
constexpr int kSoarDk = 32;     // dimensions per shared-memory chunk
constexpr int kSoarCpad = kSoarCols + 2;

// lexicographic (loss, list): NaN losses never win
__device__ __forceinline__ bool soar_better(float l, int c, float bl, int bc) {
  return l < bl || (l == bl && c < bc);
}

// One CTA per 32 rows; every tile of 64 centroids is contracted against the rows and their residuals in one pass over
// the dimensions: e = sum (x - c')^2 and p = sum r (x - c') per (row, centroid), fp32 in dimension order.  Both terms
// are formed from the differences directly (not from the expanded dot products), so neither cancels.
__global__ void __launch_bounds__(256)
    soar_spill_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d, const float* __restrict__ cent,
                      int64_t ldc, int nlist, const int32_t* __restrict__ primary, float lambda, int32_t* __restrict__ out) {
  __shared__ float xs[kSoarRows][kSoarDk + 1];
  __shared__ float rs[kSoarRows][kSoarDk + 1];
  __shared__ __align__(16) float cs[kSoarDk][kSoarCpad];
  __shared__ float s_rn[kSoarRows];
  __shared__ int s_prim[kSoarRows];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t row0 = (int64_t)blockIdx.x * kSoarRows;

  // |r|^2 of every row, one warp per row, fixed order; a row without a valid primary list gets NaN
  for (int i = warp; i < kSoarRows; i += 8) {
    const int64_t row = row0 + i;
    const int a = row < n ? primary[row] : -1;
    float s = 0.f;
    if (a >= 0 && a < nlist)
      for (int j = lane; j < d; j += 32) {
        const float r = x[row * ldx + j] - cent[(int64_t)a * ldc + j];
        s = fmaf(r, r, s);
      }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      s_rn[i] = (a >= 0 && a < nlist) ? s : __int_as_float(0x7fc00000);
      s_prim[i] = a;
    }
  }
  __syncthreads();

  float best[4];
  int bestc[4];
#pragma unroll
  for (int i = 0; i < 4; i++) best[i] = __int_as_float(0x7f800000), bestc[i] = INT_MAX;

  for (int c0 = 0; c0 < nlist; c0 += kSoarCols) {
    float e[4][2], p[4][2];
#pragma unroll
    for (int i = 0; i < 4; i++) e[i][0] = e[i][1] = p[i][0] = p[i][1] = 0.f;
    for (int k0 = 0; k0 < d; k0 += kSoarDk) {
      __syncthreads();
      for (int t = threadIdx.x; t < kSoarRows * kSoarDk; t += 256) {
        const int i = t / kSoarDk, j = t - i * kSoarDk;
        const int64_t row = row0 + i;
        const int a = s_prim[i];
        float xv = 0.f, rv = 0.f;
        if (row < n && k0 + j < d) {
          xv = x[row * ldx + k0 + j];
          rv = (a >= 0 && a < nlist) ? xv - cent[(int64_t)a * ldc + k0 + j] : 0.f;
        }
        xs[i][j] = xv;
        rs[i][j] = rv;
      }
      for (int t = threadIdx.x; t < kSoarCols * kSoarDk; t += 256) {
        const int c = t / kSoarDk, j = t - c * kSoarDk;
        cs[j][c] = (c0 + c < nlist && k0 + j < d) ? cent[(int64_t)(c0 + c) * ldc + k0 + j] : 0.f;
      }
      __syncthreads();
      const int kend = min(kSoarDk, d - k0);
      for (int j = 0; j < kend; j++) {
        const float2 cv = *reinterpret_cast<const float2*>(&cs[j][2 * lane]);
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const float xv = xs[warp * 4 + i][j], rv = rs[warp * 4 + i][j];
          const float d0 = xv - cv.x, d1 = xv - cv.y;
          e[i][0] = fmaf(d0, d0, e[i][0]);
          e[i][1] = fmaf(d1, d1, e[i][1]);
          p[i][0] = fmaf(rv, d0, p[i][0]);
          p[i][1] = fmaf(rv, d1, p[i][1]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float rn = s_rn[warp * 4 + i];
      const int a = s_prim[warp * 4 + i];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int c = c0 + 2 * lane + h;
        if (c >= nlist || c == a) continue;
        const float loss = fmaf(lambda * p[i][h], p[i][h] / rn, e[i][h]);
        if (loss <= 3.4028235e38f && soar_better(loss, c, best[i], bestc[i])) best[i] = loss, bestc[i] = c;
      }
    }
  }
  // the warp's 32 candidates of each of its rows -> the row's best
#pragma unroll
  for (int i = 0; i < 4; i++) {
    float bl = best[i];
    int bc = bestc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ol = __shfl_xor_sync(0xffffffffu, bl, o);
      const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
      if (soar_better(ol, oc, bl, bc)) bl = ol, bc = oc;
    }
    const int64_t row = row0 + warp * 4 + i;
    if (lane == 0 && row < n) {
      const float rn = s_rn[warp * 4 + i];
      // |r| = 0 or not finite, or no finite loss: the caller's fallback list
      out[row] = (rn > 0.f && rn <= 3.4028235e38f && bc != INT_MAX) ? bc : -1;
    }
  }
}

// Per query, the first k keys of m sorted keys whose vid has not occurred earlier in key order.  The (vid, position)
// pairs are sorted in shared memory (bitonic), so a position whose vid equals its predecessor's in that order is a later
// copy; the survivors are compacted in key order by a block prefix sum.
constexpr int kDedupeThreads = 512;
__global__ void __launch_bounds__(kDedupeThreads)
    dedupe_keys_kernel(const unsigned long long* __restrict__ keys, int64_t ld, int m, int k,
                       unsigned long long* __restrict__ out, int64_t out_stride) {
  extern __shared__ unsigned long long sv[];  // [NP] (vid << 32 | position), then [m] dup flags as bytes
  const int q = blockIdx.x;
  int NP = 1;
  while (NP < m) NP <<= 1;
  unsigned char* dup = reinterpret_cast<unsigned char*>(sv + NP);
  __shared__ int s_warp[kDedupeThreads / 32];
  const unsigned long long* row = keys + (int64_t)q * ld;
  for (int i = threadIdx.x; i < NP; i += blockDim.x) {
    unsigned long long v = ~0ull;
    if (i < m) {
      const unsigned long long key = row[i];
      if (key != kKeySentinel) v = ((key & 0xFFFFFFFFull) << 32) | (unsigned)i;
      dup[i] = 0;
    }
    sv[i] = v;
  }
  __syncthreads();
  for (int size = 2; size <= NP; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < NP; i += blockDim.x) {
        const int j = i ^ stride;
        if (j > i) {
          const unsigned long long a = sv[i], b = sv[j];
          const bool up = (i & size) == 0;
          if ((a > b) == up) sv[i] = b, sv[j] = a;
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x + 1; i < NP; i += blockDim.x) {
    const unsigned long long v = sv[i];
    if (v != ~0ull && (v >> 32) == (sv[i - 1] >> 32)) dup[(unsigned)v] = 1;
  }
  __syncthreads();
  // block prefix sum of the survivors, each thread over a contiguous run of positions
  const int per = (m + blockDim.x - 1) / blockDim.x;
  const int b0 = threadIdx.x * per, b1 = min(m, b0 + per);
  int cnt = 0;
  for (int i = b0; i < b1; i++) cnt += !dup[i];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int before = incl - cnt;
  for (int w = 0; w < warp; w++) before += s_warp[w];
  int total = 0;
  for (int w = 0; w < kDedupeThreads / 32; w++) total += s_warp[w];
  unsigned long long* o = out + (int64_t)q * out_stride;
  for (int i = b0, r = before; i < b1 && r < k; i++)
    if (!dup[i]) o[r++] = row[i];
  for (int r = total + threadIdx.x; r < k; r += blockDim.x) o[r] = kKeySentinel;
}

}  // namespace

cudaError_t launch_soar_spill(const float* x, int64_t ldx, int64_t n, int d, const float* centroids, int64_t ldc, int nlist,
                              const int32_t* primary, float lambda, int32_t* out, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  soar_spill_kernel<<<(unsigned)((n + kSoarRows - 1) / kSoarRows), 256, 0, st>>>(x, ldx, n, d, centroids, ldc, nlist, primary,
                                                                               lambda, out);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_dedupe_keys(const unsigned long long* keys, int64_t ld, int nrows, int m, int k, unsigned long long* out,
                               int64_t out_stride, cudaStream_t st) {
  if (nrows <= 0) return cudaSuccess;
  if (m < 1 || m > kDedupeMaxKeys || k < 1 || k > m) return cudaErrorInvalidValue;
  int NP = 1;
  while (NP < m) NP <<= 1;
  const size_t smem = (size_t)NP * 8 + (size_t)m;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(dedupe_keys_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  dedupe_keys_kernel<<<nrows, kDedupeThreads, smem, st>>>(keys, ld, m, k, out, out_stride);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
