// K1 / K2 / K6 / K8: exact fp32 tiled distance kernel (register-blocked, CUDA-core FMA).
//
// Replaces faiss::fvec_L2sqr / fvec_inner_product inner loops of GammaFLATIndex::Search
// (index/impl/gamma_index_flat.cc:224-281), the coarse quantiser quantizer->search / assign
// (gamma_index_ivfflat.cc:427,568; gamma_index_ivfpq.cc:478,595) and the assign step of k-means
// (faiss Clustering, called from gamma_index_ivfflat.cc:407 / gamma_index_ivfpq.cc:372).
//
// L2 is evaluated in the direct form sum((x-y)^2), the same form fvec_L2sqr uses, so list
// membership and returned scores do not suffer the cancellation of |x|^2+|y|^2-2xy; on
// integer-valued data every partial sum is exact and results are bit-equal to the oracle.
// Roofline: fp32 FMA issue (2 instructions per pair-element for L2, 1 for IP); DESIGN.md K1.
#include "common.cuh"
#include "kernels.h"

#include <atomic>

namespace gb {

static std::atomic<long long> g_launches{0};
void note_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }

namespace {

constexpr int BM = 128, BN = 64, BK = 16, TM = 8, TN = 4, NT = 256;
constexpr int EPI_WRITE = 0, EPI_ARGMIN = 1;

template <int METRIC, int EPI>
__global__ void __launch_bounds__(NT)
    dist_tile_kernel(const float* __restrict__ X, int64_t ldx, int n, const float* __restrict__ C, int64_t ldc, int m,
                     int d, float* __restrict__ out, int64_t ldo, unsigned long long* __restrict__ best,
                     int col_base) {
  __shared__ __align__(16) float Xs[BK][BM + 4];
  __shared__ __align__(16) float Cs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int row0 = blockIdx.y * BM, col0 = blockIdx.x * BN;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; i++)
#pragma unroll
    for (int j = 0; j < TN; j++) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < d; k0 += BK) {
#pragma unroll
    for (int i = 0; i < 2; i++) {  // X tile: 128 rows x 16 k = 512 float4
      int f = tid + i * NT;
      int row = f >> 2, kq = f & 3;
      int gr = row0 + row, gk = k0 + kq * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gr < n && gk < d) v = __ldg(reinterpret_cast<const float4*>(X + (int64_t)gr * ldx + gk));
      Xs[kq * 4 + 0][row] = v.x;
      Xs[kq * 4 + 1][row] = v.y;
      Xs[kq * 4 + 2][row] = v.z;
      Xs[kq * 4 + 3][row] = v.w;
    }
    {  // C tile: 64 rows x 16 k = 256 float4
      int row = tid >> 2, kq = tid & 3;
      int gr = col0 + row, gk = k0 + kq * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gr < m && gk < d) v = __ldg(reinterpret_cast<const float4*>(C + (int64_t)gr * ldc + gk));
      Cs[kq * 4 + 0][row] = v.x;
      Cs[kq * 4 + 1][row] = v.y;
      Cs[kq * 4 + 2][row] = v.z;
      Cs[kq * 4 + 3][row] = v.w;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; kk++) {
      float a[TM], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&Xs[kk][ty * TM]);
      float4 a1 = *reinterpret_cast<const float4*>(&Xs[kk][ty * TM + 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Cs[kk][tx * TN]);
      a[0] = a0.x, a[1] = a0.y, a[2] = a0.z, a[3] = a0.w, a[4] = a1.x, a[5] = a1.y, a[6] = a1.z, a[7] = a1.w;
      b[0] = b0.x, b[1] = b0.y, b[2] = b0.z, b[3] = b0.w;
#pragma unroll
      for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) {
          if (METRIC == kMetricL2) {
            float t = a[i] - b[j];
            acc[i][j] = fmaf(t, t, acc[i][j]);
          } else {
            acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
          }
        }
    }
    __syncthreads();
  }

  if (EPI == EPI_WRITE) {
#pragma unroll
    for (int i = 0; i < TM; i++) {
      int gr = row0 + ty * TM + i;
      if (gr >= n) continue;
      int gc = col0 + tx * TN;
      float* o = out + (int64_t)gr * ldo + gc;
      if (gc + 3 < m && (ldo & 3) == 0) {
        *reinterpret_cast<float4*>(o) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      } else {
#pragma unroll
        for (int j = 0; j < TN; j++)
          if (gc + j < m) o[j] = acc[i][j];
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < TM; i++) {
      int gr = row0 + ty * TM + i;
      unsigned long long kbest = kKeySentinel;
#pragma unroll
      for (int j = 0; j < TN; j++) {
        int gc = col0 + tx * TN + j;
        if (gc < m) {
          unsigned long long key = make_key(argmin_ord<METRIC>(acc[i][j]), (uint32_t)(gc + col_base));
          kbest = key < kbest ? key : kbest;
        }
      }
      // the 16 threads that share this row are the 16 lanes of one half-warp
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) {
        unsigned long long o = __shfl_xor_sync(0xffffffffu, kbest, off);
        kbest = o < kbest ? o : kbest;
      }
      if (tx == 0 && gr < n && kbest != kKeySentinel) atomicMin(best + gr, kbest);
    }
  }
}

__global__ void fill_u64_kernel(unsigned long long* p, int64_t n, unsigned long long v) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void pad_rows_kernel(const float* __restrict__ src, int64_t n, int d, float* __restrict__ dst, int64_t ldd) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = n * ldd;
  if (i >= total) return;
  int64_t r = i / ldd;
  int c = (int)(i - r * ldd);
  dst[i] = c < d ? src[r * d + c] : 0.f;
}

template <int METRIC, int EPI>
cudaError_t launch_tile(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d, float* out,
                        int64_t ldo, unsigned long long* best, int col_base, cudaStream_t st) {
  if (n <= 0 || m <= 0) return cudaSuccess;
  dim3 grid((m + BN - 1) / BN, (n + BM - 1) / BM);
  if (grid.y > 65535) return cudaErrorInvalidValue;
  dist_tile_kernel<METRIC, EPI><<<grid, NT, 0, st>>>(X, ldx, n, C, ldc, m, d, out, ldo, best, col_base);
  note_launch();
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_dist_matrix(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d,
                               int metric, float* out, int64_t ldo, cudaStream_t st) {
  if ((d & 3) || (ldx & 3) || (ldc & 3)) return cudaErrorInvalidValue;
  // keep grid.y under 65535 rows of tiles
  const int max_rows = 65535 * BM;
  for (int r0 = 0; r0 < n; r0 += max_rows) {
    int nr = n - r0 < max_rows ? n - r0 : max_rows;
    cudaError_t e = metric == kMetricL2
                        ? launch_tile<kMetricL2, EPI_WRITE>(X + (int64_t)r0 * ldx, ldx, nr, C, ldc, m, d,
                                                            out + (int64_t)r0 * ldo, ldo, nullptr, 0, st)
                        : launch_tile<kMetricIP, EPI_WRITE>(X + (int64_t)r0 * ldx, ldx, nr, C, ldc, m, d,
                                                            out + (int64_t)r0 * ldo, ldo, nullptr, 0, st);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_dist_argmin(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d,
                               int metric, unsigned long long* best, int col_base, cudaStream_t st) {
  if ((d & 3) || (ldx & 3) || (ldc & 3)) return cudaErrorInvalidValue;
  const int max_rows = 65535 * BM;
  for (int r0 = 0; r0 < n; r0 += max_rows) {
    int nr = n - r0 < max_rows ? n - r0 : max_rows;
    cudaError_t e = metric == kMetricL2
                        ? launch_tile<kMetricL2, EPI_ARGMIN>(X + (int64_t)r0 * ldx, ldx, nr, C, ldc, m, d, nullptr, 0,
                                                             best + r0, col_base, st)
                        : launch_tile<kMetricIP, EPI_ARGMIN>(X + (int64_t)r0 * ldx, ldx, nr, C, ldc, m, d, nullptr, 0,
                                                             best + r0, col_base, st);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_fill_u64(unsigned long long* p, int64_t n, unsigned long long v, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  fill_u64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, n, v);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pad_rows(const float* src, int64_t n, int d, float* dst, int64_t ldd, cudaStream_t st) {
  int64_t total = n * ldd;
  if (total <= 0) return cudaSuccess;
  pad_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(src, n, d, dst, ldd);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
