// OPQ rotation solve (DESIGN.md §5, OPQ bar): each training round's orthogonal Procrustes problem on the device.
//
// For A = X^T Y (d x d) the round's rotation is R = V U^T, A = U S V^T.  The SVD is jacobi_svd.h's one-sided
// (Hestenes) Jacobi restated in fp64 on the device, with the same skip, stop and sweep-cap rules and the same null-column
// test; only the pair order (round robin instead of row cyclic) and the completion of U's null columns differ.  The
// columns of A and V are stored as rows (at[j][i] = A[i][j]) so that every pair reads two contiguous vectors; at
// d = 1024 A and V are 16 MB together and stay in L2 between steps.
#include <cooperative_groups.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace gb {

namespace {

namespace cg = cooperative_groups;

constexpr int kJacobiThreads = 256;
constexpr int kJacobiMaxSweeps = 60;  // jacobi_svd.h
constexpr int kGemmTile = 64, kGemmK = 16, kGemmThreads = 256;

// sum of v over the CTA in a fixed order (warp butterflies, then the warps' partials in warp order): every thread gets
// the same bits.  red: blockDim.x / 32 doubles of shared memory; synchronised on return.
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += red[w];
  __syncthreads();
  return s;
}

// at[j][i] = xty[i][j] as fp64, vt = I
__global__ void opq_prep_kernel(const float* __restrict__ xty, int64_t ldx, int d, double* __restrict__ at,
                                double* __restrict__ vt) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)d * d) return;
  const int j = (int)(e / d), i = (int)(e % d);
  at[e] = (double)xty[(int64_t)i * ldx + j];
  vt[e] = i == j ? 1.0 : 0.0;
}

// Every sweep of the one-sided Jacobi in one cooperative launch.  A sweep is nplay - 1 steps of the round-robin
// (circle) tournament over nplay = d rounded up to even players; a step's nplay / 2 pairs are disjoint, so the CTAs
// rotate them independently, and a grid barrier separates the steps.  Player nplay - 1 stays put while the others
// rotate; with d odd it is a bye.  Each sweep's largest |gamma| / sqrt(alpha beta) goes to off[sweep % 3] (three
// words, so that the one being reset is neither read nor written by any CTA at the time); off[0] is zero at launch.
// Columns are read and written through L2 (.cg): another SM wrote them in an earlier step.
__global__ void __launch_bounds__(kJacobiThreads)
    opq_jacobi_kernel(double* __restrict__ at, double* __restrict__ vt, int d, unsigned long long* __restrict__ off,
                      int* __restrict__ sweeps_out) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double red[3][kJacobiThreads / 32];
  const int nplay = d + (d & 1), npairs = nplay / 2;
  int sweep = 0;
  while (sweep < kJacobiMaxSweeps) {
    if (blockIdx.x == 0 && threadIdx.x == 0) off[(sweep + 1) % 3] = 0;
    double offl = 0;
    for (int step = 0; step < nplay - 1; step++) {
      for (int k = blockIdx.x; k < npairs; k += gridDim.x) {
        int p, q;
        if (k == 0) {
          p = step, q = nplay - 1;
        } else {
          p = (step + k) % (nplay - 1), q = (step - k + nplay - 1) % (nplay - 1);
        }
        if (p > q) {
          const int t = p;
          p = q, q = t;
        }
        if (q >= d) continue;  // the bye of an odd d
        double* ap = at + (int64_t)p * d;
        double* aq = at + (int64_t)q * d;
        double al = 0, be = 0, ga = 0;
        for (int i = threadIdx.x; i < d; i += blockDim.x) {
          const double x = __ldcg(ap + i), y = __ldcg(aq + i);
          al += x * x, be += y * y, ga += x * y;
        }
        al = block_sum(al, red[0]);
        be = block_sum(be, red[1]);
        ga = block_sum(ga, red[2]);
        if (fabs(ga) <= 1e-15 * sqrt(al * be) || ga == 0) continue;
        offl = fmax(offl, fabs(ga) / sqrt(al * be + 1e-300));
        const double zeta = (be - al) / (2.0 * ga);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
        double* vp = vt + (int64_t)p * d;
        double* vq = vt + (int64_t)q * d;
        for (int i = threadIdx.x; i < d; i += blockDim.x) {
          const double x = __ldcg(ap + i), y = __ldcg(aq + i);
          const double u = __ldcg(vp + i), w = __ldcg(vq + i);
          __stcg(ap + i, c * x - sn * y);
          __stcg(aq + i, sn * x + c * y);
          __stcg(vp + i, c * u - sn * w);
          __stcg(vq + i, sn * u + c * w);
        }
      }
      if (step == nplay - 2 && threadIdx.x == 0 && offl > 0)
        atomicMax(off + sweep % 3, (unsigned long long)__double_as_longlong(offl));  // >= 0: bits order as values
      grid.sync();
    }
    const double o = __longlong_as_double((long long)__ldcg(off + sweep % 3));
    sweep++;
    if (o < 1e-12) break;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *sweeps_out = sweep;
}

// nrm[j] = |column j of A V|, one warp per column
__global__ void opq_colnorm_kernel(const double* __restrict__ at, int d, double* __restrict__ nrm) {
  const int j = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (j >= d) return;
  double s = 0;
  for (int i = lane; i < d; i += 32) s += at[(int64_t)j * d + i] * at[(int64_t)j * d + i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) nrm[j] = sqrt(s);
}

// One CTA per column j: U's column j (ut[j]) is A V's normalised, or 0 and null[j] = 1 when its norm is at most
// d eps times the largest (jacobi_svd.h's test)
__global__ void opq_unit_cols_kernel(const double* __restrict__ at, int d, const double* __restrict__ nrm,
                                     double* __restrict__ ut, int* __restrict__ null_col) {
  __shared__ double red[32];
  const int j = blockIdx.x;
  double m = 0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) m = fmax(m, nrm[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) m = fmax(m, red[w]);
  const double tol = d * 2.220446049250313e-16 * m, nj = nrm[j];
  const bool keep = nj > tol;
  for (int i = threadIdx.x; i < d; i += blockDim.x) ut[(int64_t)j * d + i] = keep ? at[(int64_t)j * d + i] / nj : 0.0;
  if (threadIdx.x == 0) null_col[j] = keep ? 0 : 1;
}

// C[i][j] = sum_k A[k][i] B[k][j] over k < d, d x d fp64, in k order.  projector: C = I - that.  c64 (row stride d)
// and c32 (float of the same value, row stride ld32) are each written when not null.
__global__ void __launch_bounds__(kGemmThreads)
    opq_gemm_tn_kernel(const double* __restrict__ A, const double* __restrict__ B, int d, int projector,
                       double* __restrict__ c64, float* __restrict__ c32, int64_t ld32) {
  __shared__ double as[kGemmK][kGemmTile], bs[kGemmK][kGemmTile];
  const int i0 = blockIdx.y * kGemmTile, j0 = blockIdx.x * kGemmTile;
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;  // 4 x 4 outputs each: rows i0 + ty + 16 r, cols j0 + tx + 16 c
  double acc[4][4] = {};
  for (int k0 = 0; k0 < d; k0 += kGemmK) {
    for (int e = threadIdx.x; e < kGemmK * kGemmTile; e += kGemmThreads) {
      const int kk = e / kGemmTile, c = e % kGemmTile;
      const bool in = k0 + kk < d;
      as[kk][c] = in && i0 + c < d ? A[(int64_t)(k0 + kk) * d + i0 + c] : 0.0;
      bs[kk][c] = in && j0 + c < d ? B[(int64_t)(k0 + kk) * d + j0 + c] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGemmK; kk++) {
      double a[4], b[4];
#pragma unroll
      for (int r = 0; r < 4; r++) a[r] = as[kk][ty + 16 * r], b[r] = bs[kk][tx + 16 * r];
#pragma unroll
      for (int r = 0; r < 4; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) acc[r][c] = fma(a[r], b[c], acc[r][c]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const int i = i0 + ty + 16 * r, j = j0 + tx + 16 * c;
      if (i >= d || j >= d) continue;
      const double v = projector ? (i == j ? 1.0 : 0.0) - acc[r][c] : acc[r][c];
      if (c64) c64[(int64_t)i * d + j] = v;
      if (c32) c32[(int64_t)i * ld32 + j] = (float)v;
    }
}

// One CTA: e = the lowest index of the largest diagonal entry of the projector P; w = P's column e, normalised (P is
// symmetric, so its row e is read)
__global__ void opq_pick_kernel(const double* __restrict__ P, int d, double* __restrict__ w) {
  __shared__ double red[32], s_v[32];
  __shared__ int s_i[32], s_e;
  double bv = -1;
  int be = d;
  for (int e = threadIdx.x; e < d; e += blockDim.x) {
    const double v = P[(int64_t)e * d + e];
    if (v > bv) bv = v, be = e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oe = __shfl_xor_sync(0xffffffffu, be, o);
    if (ov > bv || (ov == bv && oe < be)) bv = ov, be = oe;
  }
  if ((threadIdx.x & 31) == 0) s_v[threadIdx.x >> 5] = bv, s_i[threadIdx.x >> 5] = be;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); k++)
      if (s_v[k] > bv || (s_v[k] == bv && s_i[k] < be)) bv = s_v[k], be = s_i[k];
    s_e = be < d ? be : 0;  // no diagonal entry above -1 only when P is not finite
  }
  __syncthreads();
  const int e = s_e;
  double s = 0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) s += P[(int64_t)e * d + i] * P[(int64_t)e * d + i];
  s = block_sum(s, red);
  const double inv = 1.0 / sqrt(s);
  for (int i = threadIdx.x; i < d; i += blockDim.x) w[i] = P[(int64_t)e * d + i] * inv;
}

// y = P w, one warp per row
__global__ void opq_project_kernel(const double* __restrict__ P, int d, const double* __restrict__ w,
                                   double* __restrict__ y) {
  const int i = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= d) return;
  double s = 0;
  for (int k = lane; k < d; k += 32) s += P[(int64_t)i * d + k] * w[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) y[i] = s;
}

// One CTA: U's column j = w = y / |y|
__global__ void opq_fill_col_kernel(const double* __restrict__ y, int d, double* __restrict__ w,
                                    double* __restrict__ ut, int j) {
  __shared__ double red[32];
  double s = 0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) s += y[i] * y[i];
  s = block_sum(s, red);
  const double inv = 1.0 / sqrt(s);
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    const double v = y[i] * inv;
    w[i] = v;
    ut[(int64_t)j * d + i] = v;
  }
}

// P -= w w^T
__global__ void opq_rank1_kernel(double* __restrict__ P, int d, const double* __restrict__ w) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)d * d) return;
  P[e] -= w[e / d] * w[e % d];
}

unsigned blocks_for(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

size_t opq_procrustes_ws_bytes(int d) {
  return (size_t)d * d * 8 * 4 + (size_t)d * 8 * 3 + 3 * 8 + ((size_t)d + 1) * 4;
}

cudaError_t opq_procrustes_device(const float* xty, int64_t ldx, int d, void* ws, float* r32, int64_t ld32,
                                  double* r64, int* sweeps, cudaStream_t st) {
  if (d < 1) return cudaErrorInvalidValue;
  const size_t dd = (size_t)d * d;
  double* at = (double*)ws;
  double* vt = at + dd;
  double* ut = vt + dd;
  double* P = ut + dd;
  double* nrm = P + dd;
  double* w = nrm + d;
  double* y = w + d;
  unsigned long long* off = (unsigned long long*)(y + d);
  int* flags = (int*)(off + 3);  // [d] null columns, then the sweep count
  cudaError_t e;
  const int64_t n = (int64_t)d * d;
  opq_prep_kernel<<<blocks_for(n, 256), 256, 0, st>>>(xty, ldx, d, at, vt);
  if ((e = cudaMemsetAsync(off, 0, 3 * 8, st)) != cudaSuccess) return e;

  int dev = 0, nsm = 0, per_sm = 0;
  if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
  if ((e = cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, opq_jacobi_kernel, kJacobiThreads, 0)) != cudaSuccess)
    return e;
  const int npairs = (d + 1) / 2;
  const int grid = std::max(1, std::min(npairs, per_sm * nsm));  // every CTA resident: the grid barrier needs it
  int* sweeps_dev = flags + d;
  void* args[] = {&at, &vt, &d, &off, &sweeps_dev};
  if ((e = cudaLaunchCooperativeKernel((void*)opq_jacobi_kernel, grid, kJacobiThreads, args, 0, st)) != cudaSuccess)
    return e;
  opq_colnorm_kernel<<<blocks_for((int64_t)d * 32, 256), 256, 0, st>>>(at, d, nrm);
  opq_unit_cols_kernel<<<d, 256, 0, st>>>(at, d, nrm, ut, flags);
  note_launch(4);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;

  std::vector<int> hflags(d + 1);
  if ((e = cudaMemcpyAsync(hflags.data(), flags, (size_t)(d + 1) * 4, cudaMemcpyDeviceToHost, st)) != cudaSuccess ||
      (e = cudaStreamSynchronize(st)) != cudaSuccess)
    return e;
  if (sweeps) *sweeps = hflags[d];
  const dim3 tiles(blocks_for(d, kGemmTile), blocks_for(d, kGemmTile));
  // Null columns: P = I - U_keep U_keep^T once; per null column, the column of P with the largest diagonal entry,
  // normalised, projected through P again (Gram-Schmidt twice, as jacobi_svd.h does) and normalised becomes U's
  // column, and P loses its direction.
  bool first = true;
  for (int j = 0; j < d; j++) {
    if (!hflags[j]) continue;
    if (first) {
      opq_gemm_tn_kernel<<<tiles, kGemmThreads, 0, st>>>(ut, ut, d, 1, P, nullptr, 0);
      note_launch();
      first = false;
    }
    opq_pick_kernel<<<1, 1024, 0, st>>>(P, d, w);
    opq_project_kernel<<<blocks_for((int64_t)d * 32, 256), 256, 0, st>>>(P, d, w, y);
    opq_fill_col_kernel<<<1, 1024, 0, st>>>(y, d, w, ut, j);
    opq_rank1_kernel<<<blocks_for(n, 256), 256, 0, st>>>(P, d, w);
    note_launch(4);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  // R = V U^T: R[i][j] = sum_k vt[k][i] ut[k][j]
  opq_gemm_tn_kernel<<<tiles, kGemmThreads, 0, st>>>(vt, ut, d, 0, r64, r32, ld32);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
