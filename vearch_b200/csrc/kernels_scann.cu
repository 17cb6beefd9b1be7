// VEARCH: ScaNN-style anisotropic 4-bit codes, per-query fixed-point look-up tables and the query-major scan that sums
// them (DESIGN.md §3 K14).
//
// Replaces, in the reference (index/impl/scann/gamma_index_vearch.cc over ScaNN 1.2.1's asymmetric hashing, read from
// its sources; ScaNN itself is not built here):
//   CoordinateDescentAHQuantize / IndexDatapoint (asymmetric_hashing_impl.cc:250-540)   -> scann_encode
//   CreateRawFloatLookupTable + ConvertLookupToFixedPoint (:553-665), INT8_LUT16         -> scann_lut
//   the INT8_LUT16 accumulation and its de-quantisation (querying.h: x * (1 / multiplier)) -> vearch_scan
//
// Blocks (VARIABLE_CHUNK projection): nsub blocks of w = d / nsub dims, then one block of the d % nsub remaining dims
// when there are any.  Block b covers dims [b w, b w + width_b); its 16 centres are the codebook floats
// [16 b w + c width_b, + width_b) (codebook [16 d] floats in all).  Codes: block 2j in the low nibble of byte j, 2j + 1
// in the high nibble (the last high nibble 0 for an odd block count), as IVFPQFastScan packs them.
//
// Every statistic and cost of the encoder is fp64 with explicit __d*_rn operations, in the reference's index order, and
// every table operation fp32 with __f*_rn, so no contraction reorders them: codes, tables and scores are byte- and
// bit-equal to the numpy twin (oracle_scann/ah.py).
#include <float.h>
#include <math.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "kernels.h"
#include "list_scan.cuh"

namespace gb {

namespace {

constexpr int SC_K = 16;  // centres per block (num_clusters_per_block)

struct ScannBlocks {
  int nsub, w, nb;  // full blocks, their width, blocks in all
  __host__ __device__ ScannBlocks(int d, int nsub_) : nsub(nsub_), w(d / nsub_), nb(nsub_ + (d % nsub_ ? 1 : 0)) {}
  __host__ __device__ int start(int b) const { return b * w; }
  __host__ __device__ int width(int b, int d) const { return b < nsub ? w : d - nsub * w; }
};

// ---------------- encode: one warp per vector ---------------------------------------------------------------------
constexpr int ENC_MAX_WARPS = 8;
constexpr int kMaxRounds = 10;  // CoordinateDescentAHQuantize's kMaxRounds

__host__ __device__ inline size_t enc_warp_smem(int nb) {
  // rn, pr [nb][16] fp64, the selected residual norms [nb] fp64, the visit order [nb] int, the codes [nb] bytes
  return ((size_t)nb * SC_K * 16 + (size_t)nb * 8 + (size_t)nb * 4 + (size_t)nb + 15) & ~(size_t)15;
}

__global__ void scann_encode_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, const int32_t* __restrict__ lists,
                                    const float* __restrict__ cents, int64_t ldc, int d, int nsub,
                                    const float* __restrict__ cb, double t, bool shaped, uint8_t* __restrict__ codes) {
  extern __shared__ __align__(16) unsigned char sm_enc[];
  const ScannBlocks B(d, nsub);
  const int nb = B.nb;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + wib;
  if (i >= n) return;
  unsigned char* base = sm_enc + (size_t)wib * enc_warp_smem(nb);
  double* rn = reinterpret_cast<double*>(base);
  double* pr = rn + nb * SC_K;
  double* selnorm = pr + nb * SC_K;
  int* order = reinterpret_cast<int*>(selnorm + nb);
  uint8_t* sel = reinterpret_cast<uint8_t*>(order + nb);
  const int cbytes = (nb + 1) / 2;
  // a row without a list (deleted before it was indexed: index_batch gives it list -1) has no residual; its code is
  // never stored, so it is written as zeros without reading any centroid
  if (lists && lists[i] < 0) {
    for (int j = lane; j < cbytes; j += 32) codes[i * cbytes + j] = 0;
    return;
  }
  const float* xi = x + i * ldx;
  const float* ci = lists ? cents + (int64_t)lists[i] * ldc : nullptr;

  // the original vector's chunked norm (every lane the same fp64 sum, dims in order)
  double n2 = 0.0;
  for (int j = 0; j < d; j++) {
    const double v = (double)xi[j];
    n2 = __dadd_rn(n2, __dmul_rn(v, v));
  }
  const double inv_norm = __ddiv_rn(1.0, sqrt(n2));

  // residual statistics of every (block, centre): lanes over the pairs, dims of a block in order
  for (int p = lane; p < nb * SC_K; p += 32) {
    const int b = p / SC_K, c = p % SC_K;
    const int s0 = B.start(b), wb = B.width(b, d);
    const float* cc = cb + (int64_t)SC_K * s0 + (int64_t)c * wb;
    double r2 = 0.0, par = 0.0;
    for (int j = 0; j < wb; j++) {
      const float xv = xi[s0 + j];
      const float rv = ci ? __fsub_rn(xv, ci[s0 + j]) : xv;  // the residual to the list (IP) or the raw row (L2)
      const double rc = __dsub_rn((double)rv, (double)cc[j]);
      r2 = __dadd_rn(r2, __dmul_rn(rc, rc));
      par = __dadd_rn(par, __dmul_rn(__dmul_rn(rc, (double)xv), inv_norm));
    }
    rn[p] = r2;
    pr[p] = par;
  }
  __syncwarp();
  // InitializeToMinResidualNorm: the first minimum of each block
  for (int b = lane; b < nb; b += 32) {
    int best = 0;
    for (int c = 1; c < SC_K; c++)
      if (rn[b * SC_K + c] < rn[b * SC_K + best]) best = c;
    sel[b] = (uint8_t)best;
    selnorm[b] = rn[b * SC_K + best];
  }
  __syncwarp();
  if (shaped) {
    // ComputeParallelCostMultiplier(t, |x|^2, d)
    const double t2n = __ddiv_rn(__dmul_rn(t, t), n2);
    const double eta = __ddiv_rn(t2n, __ddiv_rn(__dsub_rn(1.0, t2n), (double)d - 1.0));
    // ComputeParallelResidualComponent: blocks in index order
    double par = 0.0;
    for (int b = 0; b < nb; b++) par = __dadd_rn(par, pr[b * SC_K + sel[b]]);
    // blocks by decreasing selected residual norm, a stable order among equals (ScaNN's ZipSortBranchOptimized
    // leaves their order unspecified); a NaN norm (a NaN coordinate or centre) counts as the smallest, so the ranks are
    // a permutation whatever the values
    for (int b = lane; b < nb; b += 32) {
      int r = 0;
      const double v = selnorm[b];
      const bool vn = isnan(v);
      for (int j = 0; j < nb; j++) {
        const double a = selnorm[j];
        const bool an = isnan(a);
        r += (an != vn ? vn : (an ? j < b : (a > v || (a == v && j < b)))) ? 1 : 0;
      }
      order[r] = b;
    }
    __syncwarp();
    bool changed = true;
    for (int round = 0; changed && round < kMaxRounds; round++) {
      changed = false;
      for (int v = 0; v < nb; v++) {
        const int b = order[v];
        const int cur = sel[b];
        // OptimizeSingleSubspace: lane c tries centre c; a move must not raise the parallel norm and must lower
        // eta * dpar + dperp below 0; the first (lowest) centre of the smallest cost wins
        const double old_rn = rn[b * SC_K + cur], old_pr = pr[b * SC_K + cur];
        double cost = 0.0, npar = 0.0;
        bool ok = false;
        if (lane < SC_K && lane != cur) {
          npar = __dadd_rn(__dsub_rn(par, old_pr), pr[b * SC_K + lane]);
          const double pnd = __dsub_rn(__dmul_rn(npar, npar), __dmul_rn(par, par));
          if (!(pnd > 0.0)) {
            const double perp = __dsub_rn(__dsub_rn(rn[b * SC_K + lane], old_rn), pnd);
            cost = __dadd_rn(__dmul_rn(eta, pnd), perp);
            ok = cost < 0.0;  // false for NaN
          }
        }
        if (__ballot_sync(0xffffffffu, ok) == 0u) continue;
        int bi = ok ? lane : SC_K;
        double bc = cost;
#pragma unroll
        for (int off = 8; off > 0; off >>= 1) {
          const double oc = __shfl_xor_sync(0xffffffffu, bc, off);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
          if (oi < SC_K && (bi == SC_K || oc < bc || (oc == bc && oi < bi))) bc = oc, bi = oi;
        }
        bi = __shfl_sync(0xffffffffu, bi, 0);
        par = __shfl_sync(0xffffffffu, npar, bi);
        if (lane == 0) sel[b] = (uint8_t)bi;
        __syncwarp();
        changed = true;
      }
    }
  }
  __syncwarp();
  for (int j = lane; j < cbytes; j += 32)
    codes[i * cbytes + j] = (uint8_t)(sel[2 * j] | (2 * j + 1 < nb ? sel[2 * j + 1] << 4 : 0));
}

// ---------------- per-query fixed-point table ----------------------------------------------------------------------
constexpr int LUT_NT = 256;

__global__ void __launch_bounds__(LUT_NT)
    scann_lut_kernel(const float* __restrict__ xq, int64_t ldq, int d, int nsub, const float* __restrict__ cb, int metric,
                     uint8_t* __restrict__ lut, float* __restrict__ mult) {
  extern __shared__ float tab[];  // [nb][16]
  __shared__ float s_red[LUT_NT / 32];
  const ScannBlocks B(d, nsub);
  const int q = blockIdx.x, tid = threadIdx.x;
  const float* x = xq + (int64_t)q * ldq;
  float mx = 0.f;
  for (int p = tid; p < B.nb * SC_K; p += LUT_NT) {
    const int b = p / SC_K, c = p % SC_K;
    const int s0 = B.start(b), wb = B.width(b, d);
    const float* cc = cb + (int64_t)SC_K * s0 + (int64_t)c * wb;
    float acc = 0.f;
    if (metric == kMetricL2) {  // SquaredL2Distance
      for (int j = 0; j < wb; j++) {
        const float u = __fsub_rn(x[s0 + j], cc[j]);
        acc = __fadd_rn(acc, __fmul_rn(u, u));
      }
    } else {  // DotProductDistance: -<q_b, c>
      for (int j = 0; j < wb; j++) acc = __fadd_rn(acc, __fmul_rn(x[s0 + j], cc[j]));
      acc = -acc;
    }
    tab[p] = acc;
    mx = fmaxf(mx, fabsf(acc));
  }
  // MaxAbsValue of the whole table (a maximum: any order)
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if ((tid & 31) == 0) s_red[tid >> 5] = mx;
  __syncthreads();
  float m = s_red[0];
  for (int w = 1; w < LUT_NT / 32; w++) m = fmaxf(m, s_red[w]);
  // ComputeMultiplierByQuantile at quantile 1: 127 / max(sqrt(FLT_EPSILON), max |entry|)
  const float lim = sqrtf(FLT_EPSILON);
  const float mul = __fdiv_rn(127.f, lim < m ? m : lim);
  if (tid == 0) mult[q] = mul;
  // TRUNCATE conversion (the proto default) plus the uint8 bias 128
  for (int p = tid; p < B.nb * SC_K; p += LUT_NT)
    lut[(int64_t)q * B.nb * SC_K + p] = (uint8_t)((int)__fmul_rn(tab[p], mul) + 128);
}

// ---------------- the leaf term <q, c_l> of every probe (IP) -----------------------------------------------------
__global__ void scann_leaf_kernel(const float* __restrict__ xq, int64_t ldq, int nq, const int32_t* __restrict__ probe_ids,
                                  int nprobe, const float* __restrict__ cents, int64_t ldc, int nlist, int d,
                                  float* __restrict__ leaf) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)nq * nprobe) return;
  const int q = (int)(t / nprobe);
  const int l = probe_ids[t];
  float acc = 0.f;
  if (l >= 0 && l < nlist) {
    const float* x = xq + (int64_t)q * ldq;
    const float* c = cents + (int64_t)l * ldc;
    for (int j = 0; j < d; j++) acc = __fadd_rn(acc, __fmul_rn(x[j], c[j]));
  }
  leaf[t] = acc;
}

// ---------------- scan: the VEARCH codec of the list scan (list_scan.cuh) ------------------------------------------
// entries per tile: about 16 KiB of codes, between 256 and 1024 entries (a multiple of LS_NT); above 64-byte codes the
// 256-entry floor makes a tile larger (32 KiB at 128 bytes, 256 blocks)
__host__ __device__ constexpr int vearch_tile_entries(int cbytes) {
  const int e = 16384 / cbytes / LS_NT * LS_NT;
  return e < LS_NT ? LS_NT : (e > 1024 ? 1024 : e);
}

// One table per query (the table does not depend on the list: under IP the list's term is added separately), so the
// CTA builds the byte-pair table T[j][byte] = (lut[2j][lo] - 128) + (lut[2j+1][hi] - 128) once; an entry's integer sum
// s = sum_j T[j][code byte j] (|s| <= 127 * 512 < 2^31).  Score: L2 f32(s) * (1 / m);  IP leaf - f32(s) * (1 / m), where
// leaf = <q, c_l> (scann_leaf_kernel) arrives as the probe's coarse distance.
struct VearchAcc {
  int32_t s;
  float leaf;
  __device__ __forceinline__ VearchAcc& operator+=(int v) {
    s += v;
    return *this;
  }
};

struct VearchCodec {
  using Entry = int16_t;
  static constexpr bool kDis0 = true;
  static constexpr int kMinCtasPerSm = 4;
  const uint8_t* lut;  // [nq][nb][16]
  const float* mult;   // [nq]
  int nb;
  bool ip;
  float inv_m;  // this CTA's query

  __host__ __device__ int code_bytes() const { return (nb + 1) / 2; }
  int tile_entries() const { return vearch_tile_entries(code_bytes()); }
  __host__ __device__ static constexpr int pt(int MW) { return vearch_tile_entries(4 * MW) / LS_NT; }

  __device__ __forceinline__ void cta_begin(int16_t* T, int q, int metric) {
    (void)metric;
    const uint8_t* lq = lut + (int64_t)q * nb * SC_K;
    for (int i = threadIdx.x; i < code_bytes() * 256; i += LS_NT) {
      const int j = i >> 8, lo = i & 15, hi = (i >> 4) & 15;
      T[i] = (int16_t)(((int)lq[2 * j * SC_K + lo] - 128) + (2 * j + 1 < nb ? (int)lq[(2 * j + 1) * SC_K + hi] - 128 : 0));
    }
    inv_m = __fdiv_rn(1.f, mult[q]);
    __syncthreads();
  }
  __device__ __forceinline__ void list_begin(int16_t* T, int list, int metric) const {
    (void)T, (void)list, (void)metric;
  }
  using Acc = VearchAcc;
  __device__ __forceinline__ VearchAcc start(float dis0) const { return VearchAcc{0, dis0}; }
  __device__ __forceinline__ float finish(VearchAcc a) const {
    const float v = __fmul_rn((float)a.s, inv_m);
    return ip ? __fsub_rn(a.leaf, v) : v;
  }
};

template <int METRIC>
cudaError_t launch_scan_cb(const VearchCodec& c, int nq, const ListScanArgs& a, cudaStream_t st) {
  switch (c.code_bytes()) {
    case 4: return launch_list_scan<VearchCodec, METRIC, 1>(c, nq, a, st);
    case 8: return launch_list_scan<VearchCodec, METRIC, 2>(c, nq, a, st);
    case 16: return launch_list_scan<VearchCodec, METRIC, 4>(c, nq, a, st);
    case 32: return launch_list_scan<VearchCodec, METRIC, 8>(c, nq, a, st);
    default: return launch_list_scan<VearchCodec, METRIC, 0>(c, nq, a, st);
  }
}

}  // namespace

int scann_blocks(int d, int nsub) { return ScannBlocks(d, nsub).nb; }

cudaError_t launch_scann_encode(const float* x, int64_t ldx, int64_t n, const int32_t* lists, const float* cents, int64_t ldc,
                                int d, int nsub, const float* codebook, double ns_threshold, uint8_t* codes, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  const int nb = ScannBlocks(d, nsub).nb;
  const size_t per_warp = enc_warp_smem(nb);
  // about 96 KiB of statistics per CTA: two CTAs per SM at every block count
  const int warps = (int)std::max<size_t>(1, std::min<size_t>(ENC_MAX_WARPS, (96 * 1024) / per_warp));
  const size_t smem = per_warp * warps;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(scann_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  // noise shaping only under IP (residual codes) with a finite threshold (GetConfig forces NaN under L2)
  const bool shaped = lists != nullptr && !std::isnan(ns_threshold);
  const int64_t grid = (n + warps - 1) / warps;
  scann_encode_kernel<<<(unsigned)grid, warps * 32, smem, st>>>(x, ldx, n, lists, cents, ldc, d, nsub, codebook, ns_threshold,
                                                                 shaped, codes);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_scann_lut(const float* xq, int64_t ldq, int nq, int d, int nsub, const float* codebook, int metric,
                             uint8_t* lut, float* mult, cudaStream_t st) {
  if (nq <= 0) return cudaSuccess;
  const size_t smem = (size_t)ScannBlocks(d, nsub).nb * SC_K * 4;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(scann_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  scann_lut_kernel<<<nq, LUT_NT, smem, st>>>(xq, ldq, d, nsub, codebook, metric, lut, mult);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_scann_leaf(const float* xq, int64_t ldq, int nq, const int32_t* probe_ids, int nprobe, const float* cents,
                              int64_t ldc, int nlist, int d, float* leaf, cudaStream_t st) {
  const int64_t work = (int64_t)nq * nprobe;
  if (work <= 0) return cudaSuccess;
  scann_leaf_kernel<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(xq, ldq, nq, probe_ids, nprobe, cents, ldc, nlist, d, leaf);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_vearch_scan(const uint8_t* lut, const float* mult, const float* leaf, int nq, const int32_t* probe_ids,
                               int nprobe, int pg, ListDirectory dir, int nb, int k, int metric, FilterArgs f,
                               unsigned long long* partial, cudaStream_t st) {
  const VearchCodec c{lut, mult, nb, metric == kMetricIP, 0.f};
  const ListScanArgs a{probe_ids, leaf, nprobe, nprobe, pg, dir, k, f, nullptr, 0, nullptr, true, partial};
  if (metric == kMetricL2) return launch_scan_cb<kMetricL2>(c, nq, a, st);
  return launch_scan_cb<kMetricIP>(c, nq, a, st);
}

int vearch_scan_max_k(int nb) { return list_scan_max_k(VearchCodec{nullptr, nullptr, nb, true, 0.f}); }

}  // namespace gb
