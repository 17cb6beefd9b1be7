// K3: IVF-Flat inverted-list scan (query-major), the HBM-roofline kernel of the path.
//
// Replaces GammaIVFFlatIndex::search_preassigned (index/impl/gamma_index_ivfflat.cc:579-787,
// pmode-0 loop :695-733) and GammaIVFFlatScanner::scan_codes (gamma_index_ivfflat.h:63-91):
//   for each query, for each probed list, for each entry j:
//     skip if ids[j] & kDelIdxMask, skip if !IsValid(vid), dis = L2sqr/IP(x, vec_j),
//     keep if IsSimilarScoreValid(dis) and better than the current k-th best.
//
// Two kernels.  ivfflat_scan_warp_kernel serves every d with a compile-time geometry (dispatch_warp);
// ivfflat_scan_kernel, the generic one, any other d: one CTA per (query, probed list, list split).
// The list's rows stream HBM -> shared memory through a ring of TMA 1-D bulk copies (cp.async.bulk +
// mbarrier complete_tx), so the copy engine keeps up to 4 x 16 KB in flight per CTA with no register
// staging.  The ring is 4 stages deep wherever the CTA's shared memory allows it; above d = 2436 at
// k = 4096 it shrinks to 3 and then 2 stages (ivfflat_scan_stages), which serves every d up to
// ivfflat_scan_max_dim().  LPR lanes share one row (float4 chunks, rotated start so both the row and
// the query reads are bank-conflict-free), partial sums meet through warp shuffles, and candidates
// that beat the running k-th best go to the CandQueue (common.cuh).  List ids are only read for
// candidates that beat the threshold.
//
// Algorithmic bytes: (4*d + 8) per scanned entry (SURVEY.md 8d); roofline: HBM.
#include <float.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace gb {

namespace {

constexpr int IVF_NT = 128;
constexpr int IVF_NST = 4;                 // pipeline stages: the deepest ring (ivfflat_scan_stages picks 4, 3 or 2)
constexpr int IVF_MIN_NST = 2;
constexpr size_t IVF_CTA_SMEM = 227 * 1024; // sm_90: shared memory of one CTA, static and dynamic
constexpr int IVF_STAGE_BYTES = 16 * 1024; // target bytes per stage
constexpr int IVF_CHUNK_ROWS = 8192;       // rows per CTA (long lists are split)

struct IvfGeom {
  int LPR, G, R, T, J, S;
  int stage_bytes;
};

__host__ __device__ inline IvfGeom ivf_geom(int d) {
  IvfGeom g;
  g.S = d >> 2;
  int lpr = 1;
  while (lpr < 32 && g.S / (lpr * 2) >= 8) lpr <<= 1;  // aim for >= 8 float4 chunks per lane
  g.LPR = lpr;
  g.G = IVF_NT / lpr;
  g.J = (g.S + lpr - 1) / lpr;
  int row_bytes = d * 4;
  int r = IVF_STAGE_BYTES / (g.G * row_bytes);
  g.R = r < 1 ? 1 : r;
  g.T = g.G * g.R;
  g.stage_bytes = g.T * row_bytes;
  return g;
}

template <int METRIC>
__global__ void __launch_bounds__(IVF_NT)
    ivfflat_scan_kernel(const float* __restrict__ xq, int64_t ldq, int d, const int32_t* __restrict__ probe_ids,
                        int nprobe, int nsplit, ListDirectory dir, IvfGeom g, int nst, int k, int KP, int SORTN,
                        FilterArgs f, unsigned long long* __restrict__ partial) {
  if (cta_cancelled(f.cancel, kCsIvfflatScan)) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* stages = reinterpret_cast<float*>(smem_raw);
  float* qs = reinterpret_cast<float*>(smem_raw + (size_t)nst * g.stage_bytes);
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(qs + d);
  __shared__ __align__(8) uint64_t full_bar[IVF_NST];
  __shared__ int s_cnt;
  __shared__ unsigned long long s_tau;

  const int tid = threadIdx.x;
  const int q = blockIdx.y;
  const int part = blockIdx.x;
  const int probe = part / nsplit, split = part - probe * nsplit;
  unsigned long long* out = partial + ((int64_t)q * gridDim.x + part) * k;

  const int list = probe_ids[(int64_t)q * nprobe + probe];
  int len = 0;
  if (list >= 0 && list < dir.nlist) len = dir.len[list];
  const int r0 = split * IVF_CHUNK_ROWS;
  const int r1 = min(len, r0 + IVF_CHUNK_ROWS);
  if (r0 >= r1) {  // nothing to scan: "not enough centroids" (ivfflat.cc:653) or empty split
    for (int i = tid; i < k; i += IVF_NT) out[i] = kKeySentinel;
    return;
  }
  const float* __restrict__ lvecs = dir.vecs[list];
  const int64_t* __restrict__ lids = dir.ids[list];

  CandQueue cq{buf, &s_cnt, &s_tau, k, KP, SORTN};
  for (int i = tid; i < d; i += IVF_NT) qs[i] = xq[(int64_t)q * ldq + i];
  if (tid == 0) {
    for (int s = 0; s < nst; s++) mbar_init(&full_bar[s], 1);
    mbar_fence_init();
  }
  cq.init();  // includes __syncthreads()

  const int ntiles = (r1 - r0 + g.T - 1) / g.T;
  const int row_bytes = d * 4;
  auto issue = [&](int t) {
    int s = t % nst;
    int rows = min(g.T, r1 - (r0 + t * g.T));
    uint32_t bytes = (uint32_t)rows * row_bytes;
    mbar_arrive_expect_tx(&full_bar[s], bytes);
    bulk_g2s(reinterpret_cast<unsigned char*>(stages) + (size_t)s * g.stage_bytes,
             lvecs + (int64_t)(r0 + t * g.T) * d, bytes, &full_bar[s]);
  };
  if (tid == 0)
    for (int t = 0; t < nst && t < ntiles; t++) issue(t);

  const int grp = tid / g.LPR;      // row slot inside a round
  const int p = tid - grp * g.LPR;  // lane inside the row group
  const float4* qs4 = reinterpret_cast<const float4*>(qs);

  for (int t = 0; t < ntiles; t++) {
    const int s = t % nst;
    mbar_wait(&full_bar[s], (t / nst) & 1);
    const int tile_rows = min(g.T, r1 - (r0 + t * g.T));
    const unsigned long long tau = s_tau;
    const uint32_t tau_hi = (uint32_t)(tau >> 32);
    const float4* st4 = reinterpret_cast<const float4*>(reinterpret_cast<unsigned char*>(stages) + (size_t)s * g.stage_bytes);

    for (int r = 0; r < g.R; r++) {
      const int rit = r * g.G + grp;  // row in tile
      const bool valid = rit < tile_rows;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      if (valid) {
        const float4* rowp = st4 + (size_t)rit * g.S;
        int jj = rit % g.J;  // rotated start: bank-conflict-free for S % 8 == 0
#pragma unroll 4
        for (int j = 0; j < g.J; j++) {
          int c = p + g.LPR * jj;
          if (c < g.S) {
            float4 v = rowp[c];
            float4 w = qs4[c];
            if (METRIC == kMetricL2) {
              float t0 = v.x - w.x, t1 = v.y - w.y, t2 = v.z - w.z, t3 = v.w - w.w;
              a0 = fmaf(t0, t0, a0), a1 = fmaf(t1, t1, a1), a2 = fmaf(t2, t2, a2), a3 = fmaf(t3, t3, a3);
            } else {
              a0 = fmaf(v.x, w.x, a0), a1 = fmaf(v.y, w.y, a1), a2 = fmaf(v.z, w.z, a2), a3 = fmaf(v.w, w.w, a3);
            }
          }
          jj = (jj + 1 == g.J) ? 0 : jj + 1;
        }
      }
      float dis = (a0 + a1) + (a2 + a3);
      for (int off = g.LPR >> 1; off > 0; off >>= 1) dis += __shfl_xor_sync(0xffffffffu, dis, off);

      bool pred = valid && p == 0 && dis <= f.max_score && dis >= f.min_score;
      unsigned long long key = kKeySentinel;
      if (pred) {
        uint32_t ord = score2ord<METRIC>(dis);
        pred = ord <= tau_hi;
        if (pred) {
          int64_t raw = lids[r0 + t * g.T + rit];
          pred = raw >= 0;  // top bit set => tombstone (gamma_index_ivfflat.h:72)
          uint32_t vid = (uint32_t)raw;
          if (pred) pred = ctx_is_valid(f.del_bits, f.filter_bits, vid);
          key = make_key(ord, vid);
          pred = pred && key < tau;
        }
      }
      cq.push_warp(pred, key);
    }
    __syncthreads();  // stage s fully consumed, all pushes of this tile done
    const int c_now = s_cnt;
    if (tid == 0 && t + nst < ntiles) issue(t + nst);
    __syncthreads();  // everyone holds the same c_now before any warp pushes again
    if (t + 1 < ntiles && c_now + g.T > cq.cap()) cq.flush();
  }
  cq.flush(true);
  for (int i = tid; i < k; i += IVF_NT) out[i] = buf[i];
}

void ivf_cq_geometry(int k, int T, int* KP, int* SORTN) {
  *KP = next_pow2(k < 16 ? 16 : k);
  *SORTN = next_pow2(*KP + 2 * T);
}

// dynamic shared memory of ivfflat_scan_kernel with an nst-stage ring: the stages, the query, the candidate queue
size_t ivf_scan_smem(const IvfGeom& g, int d, int k, int nst) {
  int KP, SORTN;
  ivf_cq_geometry(k, g.T, &KP, &SORTN);
  return (size_t)nst * g.stage_bytes + (size_t)d * 4 + (size_t)SORTN * 8;
}

// ---- fixed-geometry kernel (dimensions with an instantiation) --------------------------------
// One CTA per query x group of pg (probe, split) work items; the group's rows form one flat tile
// sequence across list boundaries.  Every WARP owns its slice of that sequence (tiles w, w+4, ...), its
// own ring of TMA bulk copies with its own mbarriers (lane 0 produces), its own threshold and its
// own candidate queue (count and tau live in registers, pushes are ballot-compacted, flushes are
// warp-level bitonic sorts).  No block-wide barrier exists until the final 4-way merge, so a warp
// never waits for another warp's memory latency.
// LPR >= 8 lanes share a row, lane p owns float4 chunks {p + LPR*j, j < J} (S = LPR*J).  A
// quarter-warp then reads 8 consecutive float4 of ONE row, so shared-memory reads are
// conflict-free without rotation and the query chunks sit in registers (4*J floats per lane).
constexpr int IVF_MAX_PG = 32;  // work items (probe, split) per CTA

__device__ __forceinline__ void warp_bitonic_sort(unsigned long long* a, int n, int lane) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < n; i += 32) {
        int ixj = i ^ j;
        if (ixj > i) {
          unsigned long long x = a[i], y = a[ixj];
          bool up = ((i & k) == 0);
          if ((x > y) == up) {
            a[i] = y;
            a[ixj] = x;
          }
        }
      }
      __syncwarp();
    }
  }
}

constexpr int IVF_NWARP = IVF_NT / 32;
constexpr int IVF_MAX_NST = 8;
// ring geometry, a sweep result: resident CTAs matter more than ring depth, so the rings stay shallow --
// 16 KiB per CTA per ring slot (4 KiB per warp) and 2 slots
constexpr int IVF_WARP_STAGE_BYTES = 16 * 1024;
constexpr int IVF_WARP_NST = 2;
static_assert(IVF_WARP_NST <= IVF_MAX_NST, "the kernel holds at most IVF_MAX_NST mbarriers per warp");

template <int METRIC, int LPR, int J>
__global__ void __launch_bounds__(IVF_NT)
    ivfflat_scan_warp_kernel(const float* __restrict__ xq, int64_t ldq, const int32_t* __restrict__ probe_ids,
                             int nprobe, int nsplit, int pg, ListDirectory dir, int R, int nst, int k, int KP, int SORTNW,
                             FilterArgs f, unsigned long long* __restrict__ partial) {
  if (cta_cancelled(f.cancel, kCsIvfflatScanWarp)) return;
  constexpr int S = LPR * J;
  constexpr int RPW = 32 / LPR;  // rows per warp round
  constexpr int ROW_BYTES = S * 16;
  const int TW = RPW * R;  // rows per warp tile
  const int stage_bytes = TW * ROW_BYTES;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw + (size_t)IVF_NWARP * nst * stage_bytes);
  unsigned long long* fin = keys + (size_t)IVF_NWARP * SORTNW;  // [IVF_NWARP * KP]
  __shared__ __align__(8) uint64_t bars[IVF_NWARP][IVF_MAX_NST];
  __shared__ int g_list[IVF_MAX_PG], g_r0[IVF_MAX_PG], g_r1[IVF_MAX_PG], g_tile0[IVF_MAX_PG + 1];

  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int q = blockIdx.y, grp_id = blockIdx.x;
  unsigned long long* out = partial + ((int64_t)q * gridDim.x + grp_id) * k;
  const int nitems = nprobe * nsplit;
  const int i0 = grp_id * pg;
  const int ni = min(pg, nitems - i0);

  if (tid == 0) {
    int acc = 0;
    for (int i = 0; i < ni; i++) {
      const int item = i0 + i;
      const int probe = item / nsplit, split = item - probe * nsplit;
      const int list = probe_ids[(int64_t)q * nprobe + probe];
      int len = 0;
      if (list >= 0 && list < dir.nlist) len = dir.len[list];
      const int r0 = split * IVF_CHUNK_ROWS;
      const int r1 = min(len, r0 + IVF_CHUNK_ROWS);
      g_list[i] = list;
      g_r0[i] = r0;
      g_r1[i] = r1 > r0 ? r1 : r0;
      g_tile0[i] = acc;
      acc += r1 > r0 ? (r1 - r0 + TW - 1) / TW : 0;
    }
    g_tile0[ni > 0 ? ni : 0] = acc;
    for (int ww = 0; ww < IVF_NWARP; ww++)
      for (int s = 0; s < nst; s++) mbar_init(&bars[ww][s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  const int total_tiles = ni > 0 ? g_tile0[ni] : 0;
  if (total_tiles == 0) {
    for (int i = tid; i < k; i += IVF_NT) out[i] = kKeySentinel;
    return;
  }

  unsigned long long* wbuf = keys + (size_t)w * SORTNW;
  for (int i = lane; i < SORTNW; i += 32) wbuf[i] = kKeySentinel;
  __syncwarp();
  const int capw = SORTNW - KP;
  unsigned long long tau = kKeySentinel;
  int cnt = 0;
  const int rowslot = lane / LPR, p = lane % LPR;
  float4 qreg[J];
  {
    const float4* q4 = reinterpret_cast<const float4*>(xq + (int64_t)q * ldq);
#pragma unroll
    for (int j = 0; j < J; j++) qreg[j] = __ldg(q4 + p + LPR * j);
  }
  unsigned char* wstage = smem_raw + (size_t)w * nst * stage_bytes;
  const int n_my = total_tiles > w ? (total_tiles - w + IVF_NWARP - 1) / IVF_NWARP : 0;

  auto warp_flush = [&]() {
    for (int i = KP + cnt + lane; i < SORTNW; i += 32) wbuf[i] = kKeySentinel;
    __syncwarp();
    warp_bitonic_sort(wbuf, SORTNW, lane);
    tau = wbuf[k - 1];
    cnt = 0;
    __syncwarp();
  };

  int pr_pi = 0;  // producer cursor (lane 0)
  auto issue = [&](int li) {
    const int gt = w + IVF_NWARP * li;
    while (gt >= g_tile0[pr_pi + 1]) pr_pi++;
    const int ti = gt - g_tile0[pr_pi];
    const int row0 = g_r0[pr_pi] + ti * TW;
    const int rows = min(TW, g_r1[pr_pi] - row0);
    const uint32_t bytes = (uint32_t)rows * ROW_BYTES;
    const int s = li % nst;
    mbar_arrive_expect_tx(&bars[w][s], bytes);
    bulk_g2s(wstage + (size_t)s * stage_bytes, dir.vecs[g_list[pr_pi]] + (int64_t)row0 * (S * 4), bytes, &bars[w][s]);
  };
  if (lane == 0)
    for (int li = 0; li < nst && li < n_my; li++) issue(li);

  int pi = 0;
  for (int li = 0; li < n_my; li++) {
    const int gt = w + IVF_NWARP * li;
    while (gt >= g_tile0[pi + 1]) pi++;
    const int64_t* __restrict__ lids = dir.ids[g_list[pi]];
    const int ti = gt - g_tile0[pi];
    const int row0 = g_r0[pi] + ti * TW;
    const int tile_rows = min(TW, g_r1[pi] - row0);
    const int s = li % nst;
    mbar_wait(&bars[w][s], (li / nst) & 1);
    const float4* st4 = reinterpret_cast<const float4*>(wstage + (size_t)s * stage_bytes);
    for (int r = 0; r < R; r++) {
      const int rit = r * RPW + rowslot;
      const bool valid = rit < tile_rows;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      if (valid) {
        const float4* rowp = st4 + (size_t)rit * S + p;
#pragma unroll
        for (int j = 0; j < J; j++) {
          float4 v = rowp[LPR * j];
          float4 wq = qreg[j];
          if (METRIC == kMetricL2) {
            float t0 = v.x - wq.x, t1 = v.y - wq.y, t2 = v.z - wq.z, t3 = v.w - wq.w;
            a0 = fmaf(t0, t0, a0), a1 = fmaf(t1, t1, a1), a2 = fmaf(t2, t2, a2), a3 = fmaf(t3, t3, a3);
          } else {
            a0 = fmaf(v.x, wq.x, a0), a1 = fmaf(v.y, wq.y, a1), a2 = fmaf(v.z, wq.z, a2), a3 = fmaf(v.w, wq.w, a3);
          }
        }
      }
      float dis = (a0 + a1) + (a2 + a3);
#pragma unroll
      for (int off = LPR >> 1; off > 0; off >>= 1) dis += __shfl_xor_sync(0xffffffffu, dis, off);

      bool pred = valid && p == 0 && dis <= f.max_score && dis >= f.min_score;
      unsigned long long key = kKeySentinel;
      if (pred) {
        uint32_t ord = score2ord<METRIC>(dis);
        pred = ord <= (uint32_t)(tau >> 32);
        if (pred) {
          int64_t raw = lids[row0 + rit];
          pred = raw >= 0;  // top bit set => tombstone (gamma_index_ivfflat.h:72)
          uint32_t vid = (uint32_t)raw;
          if (pred) pred = ctx_is_valid(f.del_bits, f.filter_bits, vid);
          key = make_key(ord, vid);
          pred = pred && key < tau;
        }
      }
      const unsigned mask = __ballot_sync(0xffffffffu, pred);
      if (mask) {
        if (pred) wbuf[KP + cnt + __popc(mask & ((1u << lane) - 1u))] = key;
        cnt += __popc(mask);
        if (cnt + RPW > capw) warp_flush();  // warp-uniform
      }
    }
    __syncwarp();  // every lane is done with stage s
    if (lane == 0 && li + nst < n_my) issue(li + nst);
  }
  warp_flush();
  __syncthreads();
  // merge the four per-warp top-KP lists
  const int NF = IVF_NWARP * KP;
  for (int i = tid; i < NF; i += IVF_NT) fin[i] = keys[(size_t)(i / KP) * SORTNW + (i % KP)];
  __syncthreads();
  block_bitonic_sort(fin, NF);
  for (int i = tid; i < k; i += IVF_NT) out[i] = fin[i];
}

// work items (probe, split) per CTA: ~16k rows of work per CTA, enough tiles to amortise start-up, enough CTAs to
// balance; one item per CTA when lists are split
inline int warp_pg(int nprobe, int nsplit, int avg_len) {
  const int per = avg_len > 0 ? 16384 / avg_len : 1;
  int pg = per < 1 ? 1 : (per > IVF_MAX_PG ? IVF_MAX_PG : per);
  if (nsplit > 1) pg = 1;
  return pg > nprobe * nsplit ? nprobe * nsplit : pg;
}

template <int METRIC, int LPR, int J>
cudaError_t launch_warp(const float* xq, int64_t ldq, int nq, const int32_t* probe_ids, int nprobe, int nsplit, int pg,
                        ListDirectory dir, int k, FilterArgs f, unsigned long long* partial, cudaStream_t st) {
  constexpr int S = LPR * J, RPW = 32 / LPR, ROW_BYTES = S * 16;
  int R = IVF_WARP_STAGE_BYTES / IVF_NWARP / (RPW * ROW_BYTES);
  if (R < 1) R = 1;
  const int TW = RPW * R;
  const int KP = next_pow2(k < 16 ? 16 : k);
  const int SORTNW = next_pow2(KP + 2 * RPW + TW);
  size_t smem =
      (size_t)IVF_NWARP * IVF_WARP_NST * TW * ROW_BYTES + (size_t)IVF_NWARP * SORTNW * 8 + (size_t)IVF_NWARP * KP * 8;
  // large k (KP = 4096 needs >= 416 KiB; at d 1536 k > 1024 already does not fit): the generic kernel, whose queue is
  // one per CTA rather than one per warp, takes it
  if (smem > 227 * 1024) return cudaErrorNotSupported;
  cudaError_t e = cudaFuncSetAttribute(ivfflat_scan_warp_kernel<METRIC, LPR, J>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const int nitems = nprobe * nsplit;
  dim3 grid((nitems + pg - 1) / pg, nq);
  ivfflat_scan_warp_kernel<METRIC, LPR, J><<<grid, IVF_NT, smem, st>>>(xq, ldq, probe_ids, nprobe, nsplit, pg, dir, R,
                                                                       IVF_WARP_NST, k, KP, SORTNW, f, partial);
  note_launch();
  return cudaGetLastError();
}

// returns cudaErrorNotSupported when no instantiation serves d or its shared memory does not fit k (caller falls back to
// the generic kernel)
template <int METRIC>
cudaError_t dispatch_warp(int S, const float* xq, int64_t ldq, int nq, const int32_t* probe_ids, int nprobe,
                          int nsplit, int pg, ListDirectory dir, int k, FilterArgs f, unsigned long long* partial,
                          cudaStream_t st) {
#define GB_WARP(LPR, J) \
  if (S == (LPR) * (J)) return launch_warp<METRIC, LPR, J>(xq, ldq, nq, probe_ids, nprobe, nsplit, pg, dir, k, f, partial, st)
  GB_WARP(8, 1);   // d = 32
  GB_WARP(8, 2);   // d = 64
  GB_WARP(8, 3);   // d = 96
  GB_WARP(8, 4);   // d = 128
  GB_WARP(8, 5);
  GB_WARP(8, 6);   // d = 192
  GB_WARP(8, 7);
  GB_WARP(8, 8);   // d = 256
  GB_WARP(16, 5);
  GB_WARP(16, 6);  // d = 384
  GB_WARP(16, 7);
  GB_WARP(16, 8);  // d = 512
  GB_WARP(32, 5);
  GB_WARP(32, 6);  // d = 768
  GB_WARP(32, 7);
  GB_WARP(32, 8);  // d = 1024
  GB_WARP(32, 12); // d = 1536
#undef GB_WARP
  return cudaErrorNotSupported;
}

// ivfflat_scan_kernel's own __shared__ arrays (the mbarriers, the queue's radix histogram: 1152 B with CUDA 12.9), which
// count against the same per-CTA limit as the dynamic window.  Read from the current device's image of the kernel; a
// failure is returned (and cleared from the runtime's last error), never cached.
cudaError_t ivf_static_smem(size_t* out) {
  cudaFuncAttributes a, b;
  cudaError_t e = cudaFuncGetAttributes(&a, ivfflat_scan_kernel<kMetricL2>);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&b, ivfflat_scan_kernel<kMetricIP>);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return e;
  }
  *out = std::max(a.sharedSizeBytes, b.sharedSizeBytes);
  return cudaSuccess;
}

int stages_beside(size_t static_smem, int d, int k) {
  if (d <= 0 || (d & 3) || k <= 0 || k > 4096) return 0;
  const IvfGeom g = ivf_geom(d);
  for (int nst = IVF_NST; nst >= IVF_MIN_NST; nst--)
    if (ivf_scan_smem(g, d, k, nst) + static_smem <= IVF_CTA_SMEM) return nst;
  return 0;
}

}  // namespace

cudaError_t ivfflat_scan_stages(int d, int k, int* nst) {
  size_t st = 0;
  const cudaError_t e = ivf_static_smem(&st);
  if (e != cudaSuccess) return e;
  *nst = stages_beside(st, d, k);
  return cudaSuccess;
}

cudaError_t ivfflat_scan_max_dim(int* max_d) {
  size_t st = 0;
  const cudaError_t e = ivf_static_smem(&st);
  if (e != cudaSuccess) return e;
  int d = 4;
  while (stages_beside(st, d + 4, 4096) > 0) d += 4;
  *max_d = d;
  return cudaSuccess;
}

int ivfflat_scan_nparts(int nprobe, int max_list_len) {
  int nsplit = (max_list_len + IVF_CHUNK_ROWS - 1) / IVF_CHUNK_ROWS;
  if (nsplit < 1) nsplit = 1;
  return nprobe * nsplit;
}

cudaError_t launch_ivfflat_scan(const float* xq, int64_t ldq, int nq, int d, const int32_t* probe_ids, int nprobe,
                                ListDirectory dir, int max_list_len, int avg_list_len, int k, int metric, FilterArgs f,
                                unsigned long long* partial, int* nparts_out, const char** kernel_out, cudaStream_t st) {
  if (nq <= 0 || nprobe <= 0) return cudaSuccess;
  if ((d & 3) || k <= 0 || k > 4096 || nq > 65535) return cudaErrorInvalidValue;
  IvfGeom g = ivf_geom(d);
  int nparts = ivfflat_scan_nparts(nprobe, max_list_len);
  int nsplit = nparts / nprobe;
  if (nparts_out) *nparts_out = nparts;
  if (ldq % 4 == 0) {
    const int pg = warp_pg(nprobe, nsplit, avg_list_len);
    cudaError_t fe = metric == kMetricL2 ? dispatch_warp<kMetricL2>(d >> 2, xq, ldq, nq, probe_ids, nprobe, nsplit, pg,
                                                                    dir, k, f, partial, st)
                                         : dispatch_warp<kMetricIP>(d >> 2, xq, ldq, nq, probe_ids, nprobe, nsplit, pg,
                                                                    dir, k, f, partial, st);
    if (fe != cudaErrorNotSupported) {
      if (nparts_out) *nparts_out = (nparts + pg - 1) / pg;  // partial[q][group][k]
      if (kernel_out) *kernel_out = "ivfflat_scan_warp_kernel";
      return fe;
    }
  }
  if (kernel_out) *kernel_out = "ivfflat_scan_kernel";
  // the deepest ring that fits: 4 stages wherever they fit (every d <= 2436 at k = 4096), else 3 or 2
  int nst = 0;
  cudaError_t e = ivfflat_scan_stages(d, k, &nst);
  if (e != cudaSuccess) return e;
  if (nst == 0) return cudaErrorInvalidValue;  // d above ivfflat_scan_max_dim(), which create_index refuses
  int KP, SORTN;
  ivf_cq_geometry(k, g.T, &KP, &SORTN);
  const size_t smem = ivf_scan_smem(g, d, k, nst);
  dim3 grid(nparts, nq);
  auto kern = metric == kMetricL2 ? ivfflat_scan_kernel<kMetricL2> : ivfflat_scan_kernel<kMetricIP>;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<grid, IVF_NT, smem, st>>>(xq, ldq, d, probe_ids, nprobe, nsplit, dir, g, nst, k, KP, SORTN, f, partial);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
