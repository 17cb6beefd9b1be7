// IVFRABITQ kernels (K13): the multi-bit RaBitQ encoder of residuals, the per-(query, list) query quantisation and the
// estimator codec of the query-major list scan (list_scan.cuh).  The arithmetic contract is DESIGN.md §3 K13; the numpy
// twin oracle_rabitq/rabitq.py repeats every floating-point operation below in the same order.
//
// Notation: B bits per dimension, W = ceil(d / 32) words per bit-plane, M = 2^(B-1) - 1.
//
// Entry (4 (B W + 3) bytes): B bit-planes of W words, plane p holding bit B-1-p of u_i at bit i & 31 of word i >> 5 (the
// sign plane first), then the fp32 factors |r|^2, f = |r|^2 / <o, r>, S = sum_i o_i, with o_i = u_i + 1/2 - 2^(B-1).
// Padding bits are 0.
//
// Encoder (one warp per vector): u_i's top bit is r_i > 0, its magnitude m_i = min(floor(t |r_i|), M) for the t > 0
// maximising cos(o, r).  The critical points t = j / |r_i| (fp64 quotients, exact in order: two distinct such fractions
// differ by far more than an fp64 rounding) are visited in increasing (t, i) order by a warp arg-min; N2 = sum |r_i| (2 m_i
// + 1) is updated in fp64 in that order, D4 = sum (2 m_i + 1)^2 exactly, and at the end of every group of equal t the
// state scores obj = N2 * N2 / D4 (fp64).  The first maximum wins, so a tie goes to the smaller t.
//
// Estimate of <o, v> (v = q - c_l under L2, q under IP), over an entry's L lanes, lane l taking words l, l + L, ...:
//   qb = 0: acc_l = fp32 sum over its words in order, dims 0..31 of a word in order, of o_i * v_i (unfused); the L partial
//           sums are added by an xor butterfly, offsets L/2, ..., 1.
//   qb > 0: A = sum_i u_i vbar_i by bit-plane AND + popc (integers, any order), X = 2 A + (1 - 2^B) sum_i vbar_i (int64),
//           <o, v> ~ delta * (float(X) * 0.5) + lo * S.
// Score: L2  (|r|^2 + dis0) - 2 (f <o, v>),   IP  <q, c_l> + f <o, v>.
#include <float.h>
#include <math_constants.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "list_scan.cuh"

namespace gb {
namespace {

constexpr int RQ_HDR = 32;  // table header words: base, delta, lo, sum vbar, then per-warp sums / minima / maxima

__host__ __device__ inline int rq_words(int d) { return (d + 31) / 32; }
// lanes per entry: the largest power of two <= W, at most 8 up to d = 992; a whole warp from d = 1024 (W >= 32), so a
// tile of LS_NT / 32 = 8 entries keeps two stages, the k' = 4096 queue and the table inside the shared memory at every
// d <= kRabitqMaxDim and nb_bits <= 9
__host__ __device__ inline int rq_lanes(int d) {
  const int W = rq_words(d);
  return W >= 32 ? 32 : (W >= 8 ? 8 : (W >= 4 ? 4 : (W >= 2 ? 2 : 1)));
}

// ---------------- encoder ---------------------------------------------------------------------------------
constexpr int ENC_MAX_WARPS = 4;

__device__ __forceinline__ void rq_lane_min(const double* nxt, int d, int lane, double* k, int* idx) {
  double bk = CUDART_INF;
  int bi = 0x7fffffff;
  for (int i = lane; i < d; i += 32)
    if (nxt[i] < bk) bk = nxt[i], bi = i;
  *k = bk;
  *idx = bi;
}

__device__ __forceinline__ void rq_warp_min(double* k, int* idx) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const double ok = __shfl_xor_sync(0xffffffffu, *k, off);
    const int oi = __shfl_xor_sync(0xffffffffu, *idx, off);
    if (ok < *k || (ok == *k && oi < *idx)) *k = ok, *idx = oi;
  }
}

__global__ void __launch_bounds__(ENC_MAX_WARPS * 32)
    rabitq_encode_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, const int32_t* __restrict__ lists,
                         const float* __restrict__ cents, int64_t ldc, int d, int B, uint8_t* __restrict__ codes) {
  extern __shared__ __align__(16) unsigned char enc_smem[];
  const int W = rq_words(d), dp = 32 * W;
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* nxt = reinterpret_cast<double*>(enc_smem) + (size_t)warp * dp;
  float* r = reinterpret_cast<float*>(reinterpret_cast<double*>(enc_smem) + (size_t)nw * dp) + (size_t)warp * dp;
  int* m = reinterpret_cast<int*>(reinterpret_cast<float*>(reinterpret_cast<double*>(enc_smem) + (size_t)nw * dp) +
                                  (size_t)nw * dp) + (size_t)warp * dp;
  const int64_t row = (int64_t)blockIdx.x * nw + warp;
  if (row >= n) return;  // the whole warp: no block-wide barrier follows
  const int M = (1 << (B - 1)) - 1;
  const float* xr = x + row * ldx;
  const float* c = cents + (int64_t)lists[row] * ldc;
  for (int i = lane; i < dp; i += 32) {
    const float ri = i < d ? __fsub_rn(xr[i], c[i]) : 0.f;
    const float a = fabsf(ri);
    r[i] = ri;
    m[i] = 0;
    nxt[i] = (i < d && M > 0 && a > 0.f) ? __ddiv_rn(1.0, (double)a) : CUDART_INF;
  }
  __syncwarp();
  double N2 = 0.0, nr2 = 0.0;
  if (lane == 0) {
    for (int i = 0; i < d; i++) {
      const double ri = (double)r[i];
      N2 = __dadd_rn(N2, fabs(ri));
      nr2 = __dadd_rn(nr2, __dmul_rn(ri, ri));
    }
  }
  N2 = __shfl_sync(0xffffffffu, N2, 0);
  nr2 = __shfl_sync(0xffffffffu, nr2, 0);
  double D4 = (double)d;
  double best = __ddiv_rn(__dmul_rn(N2, N2), D4), bestN2 = N2, bestT = -1.0;
  double lk, gk;
  int li, gi;
  rq_lane_min(nxt, d, lane, &lk, &li);
  gk = lk, gi = li;
  rq_warp_min(&gk, &gi);
  while (gk < CUDART_INF) {
    const int i = gi;
    const double T = gk;
    const float a = fabsf(r[i]);
    const int mi = m[i] + 1;
    N2 = __dadd_rn(N2, 2.0 * (double)a);
    D4 = __dadd_rn(D4, 8.0 * (double)mi);
    __syncwarp();
    if ((i & 31) == lane) {
      m[i] = mi;
      nxt[i] = mi < M ? __ddiv_rn((double)(mi + 1), (double)a) : CUDART_INF;
      rq_lane_min(nxt, d, lane, &lk, &li);
    }
    __syncwarp();
    gk = lk, gi = li;
    rq_warp_min(&gk, &gi);
    if (gk != T) {  // the last event of its group: a state m(t) for t in [T, next t)
      const double obj = __ddiv_rn(__dmul_rn(N2, N2), D4);
      if (obj > best) best = obj, bestN2 = N2, bestT = T;
    }
  }
  // codes of the best state: m_i = #{j <= M : j / |r_i| <= bestT}
  uint32_t* out = reinterpret_cast<uint32_t*>(codes + row * (int64_t)(4 * (B * W + 3)));
  int ssum = 0;
  const int half = 1 << (B - 1);
  for (int w = 0; w < W; w++) {
    const int i = 32 * w + lane;
    uint32_t u = 0;
    if (i < d) {
      const float ri = r[i];
      const double a = (double)fabsf(ri);
      int mm = 0;
      if (bestT >= 0.0 && a > 0.0 && M > 0) {
        mm = (int)fmin((double)M, floor(bestT * a));
        while (mm < M && __ddiv_rn((double)(mm + 1), a) <= bestT) mm++;
        while (mm > 0 && __ddiv_rn((double)mm, a) > bestT) mm--;
      }
      u = ri > 0.f ? (uint32_t)(half + mm) : (uint32_t)(half - 1 - mm);
      ssum += 2 * (int)u + 1 - 2 * half;
    }
    for (int p = 0; p < B; p++) {
      const uint32_t bits = __ballot_sync(0xffffffffu, (u >> (B - 1 - p)) & 1u);
      if (lane == 0) out[p * W + w] = bits;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) ssum += __shfl_xor_sync(0xffffffffu, ssum, off);
  if (lane == 0) {
    float* fac = reinterpret_cast<float*>(out + B * W);
    fac[0] = __double2float_rn(nr2);
    fac[1] = bestN2 > 0.0 ? __double2float_rn(__ddiv_rn(nr2, __dmul_rn(bestN2, 0.5))) : 0.f;
    fac[2] = __fmul_rn(__int2float_rn(ssum), 0.5f);
  }
}

// ---------------- the estimator codec of the list scan ----------------------------------------------------
__host__ __device__ inline int rq_tile_entries(int cb, int L) {  // ~16 KiB of codes, a multiple of LS_NT / L, <= 1024
  const int g = LS_NT / L;
  int e = 16384 / cb / g * g;
  return e < g ? g : (e > 1024 ? 1024 : e);
}

struct RabitqCodec {
  using Entry = uint32_t;
  static constexpr bool kDis0 = false;  // dis0 and <q, c_l> are recomputed in list_begin, in the twin's order
  static constexpr bool kCodeSum = true;
  static constexpr bool kLanes = true;
  static constexpr int kMinCtasPerSm = 0;
  const float* queries;  // [nq][ldq] fp32, zero padded
  int64_t ldq;
  const float* cents;  // [nlist][ldc]
  int64_t ldc;
  int d, B, qb, metric;
  const float* qrow = nullptr;  // this CTA's query (cta_begin)

  __host__ __device__ int W() const { return rq_words(d); }
  __host__ __device__ int lanes() const { return rq_lanes(d); }
  __host__ __device__ int code_bytes() const { return 4 * (B * W() + 3); }
  __host__ __device__ int table_entries() const { return (RQ_HDR + 32 * W() + qb * W() + 3) & ~3; }
  int tile_entries() const { return rq_tile_entries(code_bytes(), lanes()); }
  __host__ __device__ static constexpr int pt(int) { return 1; }  // not used: MW = 0 only

  __device__ __forceinline__ void cta_begin(uint32_t* tab, int q, int) {
    (void)tab;
    qrow = queries + (int64_t)q * ldq;
  }

  // v (padding 0) and, for qb > 0, its qb bit-planes; header: base (dis0 under L2, <q, c_l> under IP), delta, lo, sum vbar.
  // Sums: thread t adds dims t, t + LS_NT, ... in order; a warp adds its 32 partials by an xor butterfly (16, ..., 1);
  // thread 0 adds the warp totals in warp order.
  __device__ void list_begin(uint32_t* tab, int list, int) const {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int W = this->W();
    const float* c = cents + (int64_t)list * ldc;
    float* v = reinterpret_cast<float*>(tab + RQ_HDR);
    float s = 0.f, mn = FLT_MAX, mx = -FLT_MAX;
    for (int i = tid; i < 32 * W; i += LS_NT) {
      float vi = 0.f;
      if (i < d) {
        const float qi = qrow[i], ci = c[i];
        if (metric == kMetricL2) {
          vi = __fsub_rn(qi, ci);
          s = __fadd_rn(s, __fmul_rn(vi, vi));
        } else {
          vi = qi;
          s = __fadd_rn(s, __fmul_rn(qi, ci));
        }
        mn = fminf(mn, vi);
        mx = fmaxf(mx, vi);
      }
      v[i] = vi;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, off));
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    float* hdr = reinterpret_cast<float*>(tab);
    if (lane == 0) hdr[8 + warp] = s, hdr[16 + warp] = mn, hdr[24 + warp] = mx;
    __syncthreads();
    if (tid == 0) {
      float base = hdr[8], lo = hdr[16], hi = hdr[24];
      for (int w = 1; w < LS_NT / 32; w++) {
        base = __fadd_rn(base, hdr[8 + w]);
        lo = fminf(lo, hdr[16 + w]);
        hi = fmaxf(hi, hdr[24 + w]);
      }
      hdr[0] = base;
      hdr[1] = (qb > 0 && hi > lo) ? __fdiv_rn(__fsub_rn(hi, lo), (float)((1 << qb) - 1)) : 0.f;
      hdr[2] = lo;
      tab[3] = 0u;
    }
    __syncthreads();
    if (qb > 0) {
      const float delta = hdr[1], lo = hdr[2];
      const int vmax = (1 << qb) - 1;
      uint32_t* planes = tab + RQ_HDR + 32 * W;
      int sv = 0;
      for (int w = tid; w < W; w += LS_NT) {
        uint32_t pl[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
        for (int k = 0; k < 32; k++) {
          const int i = 32 * w + k;
          int vb = 0;
          if (i < d && delta > 0.f) vb = min(max((int)rintf(__fdiv_rn(__fsub_rn(v[i], lo), delta)), 0), vmax);
          sv += vb;
#pragma unroll
          for (int b = 0; b < 8; b++) pl[b] |= (uint32_t)((vb >> b) & 1) << k;
        }
        for (int b = 0; b < qb; b++) planes[b * W + w] = pl[b];
      }
      if (sv) atomicAdd(reinterpret_cast<int*>(tab + 3), sv);
      __syncthreads();
    }
  }

  using Acc = float;  // not used: score_lanes scores the entries
  __device__ __forceinline__ float start(float) const { return 0.f; }
  __device__ __forceinline__ float finish(float a) const { return a; }

  __device__ __forceinline__ float score_lanes(const unsigned char* code, const uint32_t* __restrict__ tab, int lane) const {
    const int W = this->W(), L = lanes();
    const uint32_t* cw = reinterpret_cast<const uint32_t*>(code);
    const float* fac = reinterpret_cast<const float*>(cw + B * W);
    const float* hdr = reinterpret_cast<const float*>(tab);
    float ip;
    if (qb == 0) {
      const float* v = reinterpret_cast<const float*>(tab + RQ_HDR);
      float acc = 0.f;
      for (int w = lane; w < W; w += L) {
        uint32_t p[9];
#pragma unroll
        for (int pp = 0; pp < 9; pp++) p[pp] = pp < B ? cw[pp * W + w] : 0u;
        for (int k = 0; k < 32; k++) {
          uint32_t u = 0;
#pragma unroll
          for (int pp = 0; pp < 9; pp++)
            if (pp < B) u = (u << 1) | ((p[pp] >> k) & 1u);
          const float o = __fmul_rn((float)(2 * (int)u + 1 - (1 << B)), 0.5f);
          acc = __fadd_rn(acc, __fmul_rn(o, v[32 * w + k]));
        }
      }
      for (int off = L >> 1; off > 0; off >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, off));
      ip = acc;
    } else {
      const uint32_t* vb = tab + RQ_HDR + 32 * W;
      int A = 0;
      for (int w = lane; w < W; w += L) {
        for (int pp = 0; pp < B; pp++) {
          const uint32_t pw = cw[pp * W + w];
          int s = 0;
          for (int b = 0; b < qb; b++) s += __popc(pw & vb[b * W + w]) << b;
          A += s << (B - 1 - pp);
        }
      }
      for (int off = L >> 1; off > 0; off >>= 1) A += __shfl_xor_sync(0xffffffffu, A, off);
      const long long X = 2LL * A + (long long)(1 - (1 << B)) * (long long)(int)tab[3];
      ip = __fadd_rn(__fmul_rn(hdr[1], __fmul_rn(__ll2float_rn(X), 0.5f)), __fmul_rn(hdr[2], fac[2]));
    }
    const float t = __fmul_rn(fac[1], ip);
    return metric == kMetricL2 ? __fsub_rn(__fadd_rn(fac[0], hdr[0]), __fmul_rn(2.f, t)) : __fadd_rn(hdr[0], t);
  }
};

// est[out_off[j] + e] = score of entry e of list l_of[j] for query q_of[j]: the scan's own codec, one CTA per pair
__global__ void __launch_bounds__(LS_NT)
    rabitq_estimate_kernel(RabitqCodec c, ListDirectory dir, const int32_t* __restrict__ q_of,
                           const int32_t* __restrict__ l_of, const int64_t* __restrict__ out_off, float* __restrict__ out) {
  extern __shared__ __align__(16) uint32_t est_tab[];
  const int j = blockIdx.x, tid = threadIdx.x;
  const int l = l_of[j];
  c.cta_begin(est_tab, q_of[j], c.metric);
  c.list_begin(est_tab, l, c.metric);
  const int len = dir.len[l], cb = c.code_bytes(), L = c.lanes();
  const unsigned char* base = dir.codes[l];
  for (int e0 = 0; e0 < len; e0 += LS_NT / L) {
    const int e = e0 + tid / L;
    const float sc = c.score_lanes(base + (size_t)min(e, len - 1) * cb, est_tab, tid & (L - 1));
    if ((tid & (L - 1)) == 0 && e < len) out[out_off[j] + e] = sc;
  }
}

}  // namespace

int rabitq_code_bytes(int d, int nb_bits) { return 4 * (nb_bits * rq_words(d) + 3); }

cudaError_t launch_rabitq_encode(const float* x, int64_t ldx, int64_t n, const int32_t* lists, const float* cents, int64_t ldc,
                                 int d, int nb_bits, uint8_t* codes, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  if (d <= 0 || d > kRabitqMaxDim || nb_bits < 1 || nb_bits > 9) return cudaErrorInvalidValue;
  const size_t per_warp = (size_t)32 * rq_words(d) * 16;  // fp64 key, fp32 residual, int magnitude per dimension
  const int nw = (int)std::max<size_t>(1, std::min<size_t>(ENC_MAX_WARPS, (size_t)(96 * 1024) / per_warp));
  const size_t smem = per_warp * nw;
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(rabitq_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  rabitq_encode_kernel<<<(unsigned)((n + nw - 1) / nw), nw * 32, smem, st>>>(x, ldx, n, lists, cents, ldc, d, nb_bits, codes);
  note_launch();
  return cudaGetLastError();
}

int rabitq_scan_max_k(int d, int nb_bits, int qb) {
  return list_scan_max_k(RabitqCodec{nullptr, 0, nullptr, 0, d, nb_bits, qb, kMetricL2});
}

cudaError_t launch_rabitq_scan(const float* xq, int64_t ldq, int nq, const float* cents, int64_t ldc, int d, int nb_bits, int qb,
                               const int32_t* probe_ids, int nprobe, int pg, ListDirectory dir, int k, int metric, FilterArgs f,
                               unsigned long long* partial, cudaStream_t st) {
  const RabitqCodec c{xq, ldq, cents, ldc, d, nb_bits, qb, metric};
  const ListScanArgs a{probe_ids, nullptr, nprobe, nprobe, pg, dir, k, f, nullptr, 0, nullptr, true, partial};
  if (metric == kMetricL2) return launch_list_scan<RabitqCodec, kMetricL2, 0>(c, nq, a, st);
  return launch_list_scan<RabitqCodec, kMetricIP, 0>(c, nq, a, st);
}

cudaError_t launch_rabitq_estimate(const float* xq, int64_t ldq, const float* cents, int64_t ldc, int d, int nb_bits, int qb,
                                   int metric, ListDirectory dir, const int32_t* q_of, const int32_t* l_of,
                                   const int64_t* out_off, int npairs, float* out, cudaStream_t st) {
  if (npairs <= 0) return cudaSuccess;
  const RabitqCodec c{xq, ldq, cents, ldc, d, nb_bits, qb, metric};
  const size_t smem = (size_t)c.table_entries() * 4;
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(rabitq_estimate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  rabitq_estimate_kernel<<<npairs, LS_NT, smem, st>>>(c, dir, q_of, l_of, out_off, out);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
