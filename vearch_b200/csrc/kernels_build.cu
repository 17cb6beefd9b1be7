// K6 / K8 / T1 build-side kernels: k-means centroid update, residuals, column slicing, row
// gather, normalisation and the inverted-list append.
//
// Replaces, in the reference: the centroid update of faiss::Clustering (driven from
// gamma_index_ivfflat.cc:407 and gamma_index_ivfpq.cc:372), compute_residuals
// (gamma_index_ivfpq.cc:378-391), the training-slab merge (gamma_index_ivfflat.cc:377-405) and
// RTInvertIndex::AddKeys / RealTimeMemData::AddKeys (index/realtime/realtime_mem_data.cc:258-296).
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace gb {

namespace {

// one CTA per cluster; members are summed in the given (point) order so the result equals a
// sequential CPU accumulation bit for bit, then scaled by 1/count (faiss: c *= 1/hassign).
__global__ void __launch_bounds__(128)
    segment_mean_kernel(const float* __restrict__ x, int64_t ldx, int d, const int32_t* __restrict__ perm,
                        const int32_t* __restrict__ off, float* __restrict__ centroids, int64_t ldc) {
  const int c = blockIdx.x;
  const int b = off[c], e = off[c + 1];
  for (int j = threadIdx.x; j < d; j += blockDim.x) {
    float acc = 0.f;
    int i = b;
    for (; i + 4 <= e; i += 4) {
      float v0 = x[(int64_t)perm[i] * ldx + j], v1 = x[(int64_t)perm[i + 1] * ldx + j];
      float v2 = x[(int64_t)perm[i + 2] * ldx + j], v3 = x[(int64_t)perm[i + 3] * ldx + j];
      acc += v0;
      acc += v1;
      acc += v2;
      acc += v3;
    }
    for (; i < e; i++) acc += x[(int64_t)perm[i] * ldx + j];
    float out = 0.f;
    if (e > b) out = acc * (1.0f / (float)(e - b));
    centroids[(int64_t)c * ldc + j] = out;
  }
}

__global__ void residual_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d,
                                const float* __restrict__ centroids, int64_t ldc, const int32_t* __restrict__ assign,
                                float* __restrict__ out, int64_t ldo) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = n * ldo;
  if (i >= total) return;
  int64_t r = i / ldo;
  int c = (int)(i - r * ldo);
  out[i] = c < d ? x[r * ldx + c] - centroids[(int64_t)assign[r] * ldc + c] : 0.f;
}

__global__ void slice_cols_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int col0, int w,
                                  float* __restrict__ out, int64_t ldo) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = n * ldo;
  if (i >= total) return;
  int64_t r = i / ldo;
  int c = (int)(i - r * ldo);
  out[i] = c < w ? x[r * ldx + col0 + c] : 0.f;
}

__global__ void gather_rows_kernel(const float* __restrict__ x, int64_t ldx, const int32_t* __restrict__ idx, int64_t n,
                                   int d, float* __restrict__ out, int64_t ldo) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = n * ldo;
  if (i >= total) return;
  int64_t r = i / ldo;
  int c = (int)(i - r * ldo);
  out[i] = c < d ? x[(int64_t)idx[r] * ldx + c] : 0.f;
}

// one warp per row; fixed reduction order => deterministic
__global__ void normalize_rows_kernel(float* __restrict__ x, int64_t ldx, int64_t n, int d) {
  int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (r >= n) return;
  float* row = x + r * ldx;
  float s = 0.f;
  for (int j = lane; j < d; j += 32) s = fmaf(row[j], row[j], s);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (s > 0.f) {
    float inv = 1.0f / sqrtf(s);
    for (int j = lane; j < d; j += 32) row[j] *= inv;
  }
}

// one warp per appended row (float4 copies)
__global__ void ivf_append_vecs_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d,
                                       const int32_t* __restrict__ list, const int32_t* __restrict__ pos,
                                       float* const* __restrict__ list_vecs, int64_t* const* __restrict__ list_ids,
                                       int64_t vid0) {
  int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (r >= n) return;
  int l = list[r];
  if (l < 0) return;  // skipped (deleted before indexing, gamma_index_ivfflat.cc:436)
  int p = pos[r];
  const float4* src = reinterpret_cast<const float4*>(x + r * ldx);
  float4* dst = reinterpret_cast<float4*>(list_vecs[l] + (int64_t)p * d);
  for (int c = lane; c < (d >> 2); c += 32) dst[c] = src[c];
  if (lane == 0) list_ids[l][p] = vid0 + r;
}

__global__ void ivf_append_codes_kernel(const uint8_t* __restrict__ codes, int64_t n, int M,
                                        const int32_t* __restrict__ list, const int32_t* __restrict__ pos,
                                        uint8_t* const* __restrict__ list_codes, int64_t* const* __restrict__ list_ids,
                                        int64_t vid0) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  int l = list[r];
  if (l < 0) return;
  int p = pos[r];
  const uint8_t* src = codes + r * M;
  uint8_t* dst = list_codes[l] + (int64_t)p * M;
  if ((M & 3) == 0) {
    for (int j = 0; j < M; j += 4) *reinterpret_cast<uint32_t*>(dst + j) = *reinterpret_cast<const uint32_t*>(src + j);
  } else {
    for (int j = 0; j < M; j++) dst[j] = src[j];
  }
  list_ids[l][p] = vid0 + r;
}

inline unsigned blocks_for(int64_t total, int bs) { return (unsigned)((total + bs - 1) / bs); }

// column means, one CTA per column (rows strided over the threads, tree reduction in shared memory)
__global__ void __launch_bounds__(256)
    col_mean_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, float* __restrict__ mean) {
  __shared__ double acc[256];
  const int j = blockIdx.x;
  double a = 0;
  for (int64_t i = threadIdx.x; i < n; i += 256) a += x[i * ldx + j];
  acc[threadIdx.x] = a;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) acc[threadIdx.x] += acc[threadIdx.x + off];
    __syncthreads();
  }
  if (threadIdx.x == 0) mean[j] = (float)(acc[0] / (double)n);
}

__global__ void center_rows_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d, const float* __restrict__ mean,
                                   float* __restrict__ out, int64_t ldo) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * ldo) return;
  const int64_t i = idx / ldo;
  const int j = (int)(idx - i * ldo);
  out[idx] = j < d ? x[i * ldx + j] - mean[j] : 0.f;
}

__global__ void transpose_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d, float* __restrict__ out,
                                 int64_t ldo) {
  __shared__ float tile[32][33];
  const int64_t i0 = (int64_t)blockIdx.x * 32;
  const int j0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int64_t i = i0 + r;
    const int j = j0 + threadIdx.x;
    tile[r][threadIdx.x] = (i < n && j < d) ? x[i * ldx + j] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int j = j0 + r;
    const int64_t i = i0 + threadIdx.x;
    if (j < d && i < n) out[(int64_t)j * ldo + i] = tile[threadIdx.x][r];
  }
}

__global__ void pq_decode_kernel(const uint8_t* __restrict__ codes, int64_t n, const float* __restrict__ pq, int M, int dsub,
                                 float* __restrict__ recon, int64_t ldr) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int d = M * dsub;
  if (idx >= n * d) return;
  const int64_t i = idx / d;
  const int c = (int)(idx - i * d);
  const int m = c / dsub, j = c - m * dsub;
  recon[i * ldr + c] = pq[((int64_t)m * 256 + codes[i * M + m]) * dsub + j];
}

}  // namespace

cudaError_t launch_center_rows(const float* x, int64_t ldx, int64_t n, int d, float* mean, float* out, int64_t ldo,
                               cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  col_mean_kernel<<<d, 256, 0, st>>>(x, ldx, n, mean);
  note_launch();
  center_rows_kernel<<<blocks_for(n * ldo, 256), 256, 0, st>>>(x, ldx, n, d, mean, out, ldo);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_transpose(const float* x, int64_t ldx, int64_t n, int d, float* out, int64_t ldo, cudaStream_t st) {
  if (n <= 0 || d <= 0) return cudaSuccess;
  dim3 grid((unsigned)((n + 31) / 32), (unsigned)((d + 31) / 32)), block(32, 8);
  transpose_kernel<<<grid, block, 0, st>>>(x, ldx, n, d, out, ldo);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_pq_decode(const uint8_t* codes, int64_t n, const float* pq_centroids, int M, int dsub, float* recon,
                             int64_t ldr, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  pq_decode_kernel<<<blocks_for(n * M * dsub, 256), 256, 0, st>>>(codes, n, pq_centroids, M, dsub, recon, ldr);
  note_launch();
  return cudaGetLastError();
}


cudaError_t launch_segment_mean(const float* x, int64_t ldx, int d, const int32_t* perm, const int32_t* off, int k,
                                float* centroids, int64_t ldc, cudaStream_t st) {
  if (k <= 0) return cudaSuccess;
  segment_mean_kernel<<<k, 128, 0, st>>>(x, ldx, d, perm, off, centroids, ldc);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_residual(const float* x, int64_t ldx, int64_t n, int d, const float* centroids, int64_t ldc,
                            const int32_t* assign, float* out, int64_t ldo, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  residual_kernel<<<blocks_for(n * ldo, 256), 256, 0, st>>>(x, ldx, n, d, centroids, ldc, assign, out, ldo);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_slice_cols(const float* x, int64_t ldx, int64_t n, int col0, int w, float* out, int64_t ldo,
                              cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  slice_cols_kernel<<<blocks_for(n * ldo, 256), 256, 0, st>>>(x, ldx, n, col0, w, out, ldo);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_gather_rows(const float* x, int64_t ldx, const int32_t* idx, int64_t n, int d, float* out,
                               int64_t ldo, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  gather_rows_kernel<<<blocks_for(n * ldo, 256), 256, 0, st>>>(x, ldx, idx, n, d, out, ldo);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_normalize_rows(float* x, int64_t ldx, int64_t n, int d, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  normalize_rows_kernel<<<blocks_for(n * 32, 256), 256, 0, st>>>(x, ldx, n, d);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_ivf_append_vecs(const float* x, int64_t ldx, int64_t n, int d, const int32_t* list, const int32_t* pos,
                                   float* const* list_vecs, int64_t* const* list_ids, int64_t vid0, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  ivf_append_vecs_kernel<<<blocks_for(n * 32, 256), 256, 0, st>>>(x, ldx, n, d, list, pos, list_vecs, list_ids, vid0);
  note_launch();
  return cudaGetLastError();
}

__global__ void ivf_rowptrs_kernel(ListDirectory dir, int ld, const float** rowptr) {
  const int l = blockIdx.x;
  const int len = dir.len[l];
  const int64_t* ids = dir.ids[l];
  const float* rows = dir.vecs[l];
  for (int p = threadIdx.x; p < len; p += blockDim.x) {
    const int64_t id = ids[p];
    if (id >= 0) rowptr[id] = rows + (int64_t)p * ld;  // top bit set: tombstoned by Update
  }
}

cudaError_t launch_ivf_rowptrs(ListDirectory dir, int ld, const float** rowptr, cudaStream_t st) {
  if (dir.nlist <= 0) return cudaSuccess;
  ivf_rowptrs_kernel<<<dir.nlist, 256, 0, st>>>(dir, ld, rowptr);
  note_launch();
  return cudaGetLastError();
}

// ---- purge: stable compaction of a set of lists (RealTimeMemData::CompactBucket, realtime_mem_data.cc:94-146) ----
// The selected lists are cut into chunks of kPurgeChunk entries, one CTA per chunk, so one long list spreads over the
// device and a thousand short ones cost one launch.
namespace {

// live = not tombstoned and not set in the deletion bitmap: what every list scan tests before it scores an entry
__device__ __forceinline__ bool purge_live(int64_t id, const uint32_t* __restrict__ del_bits) {
  return id >= 0 && !(del_bits && bit_test(del_bits, (uint32_t)id));
}

__global__ void __launch_bounds__(256)
    purge_count_kernel(ListDirectory dir, const int* __restrict__ sel_list, const PurgeChunk* __restrict__ chunks,
                       const uint32_t* __restrict__ del_bits, int* __restrict__ chunk_cnt, unsigned long long* vid_range) {
  __shared__ int s_cnt;
  __shared__ unsigned long long s_min, s_max;
  if (threadIdx.x == 0) s_cnt = 0, s_min = ~0ull, s_max = 0;
  __syncthreads();
  const PurgeChunk c = chunks[blockIdx.x];
  const int list = sel_list[c.sel];
  const int64_t* __restrict__ ids = dir.ids[list];
  const int end = min(c.first + kPurgeChunk, dir.len[list]);
  int cnt = 0;
  unsigned long long lo = ~0ull, hi = 0;
  for (int p = c.first + threadIdx.x; p < end; p += blockDim.x) {
    const int64_t id = ids[p];
    cnt += purge_live(id, del_bits);
    const unsigned long long vid = (unsigned long long)(id & ~kDelIdxMask);
    lo = min(lo, vid);
    hi = max(hi, vid);
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  for (int o = 16; o; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&s_cnt, cnt);
    atomicMin(&s_min, lo);
    atomicMax(&s_max, hi);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    chunk_cnt[blockIdx.x] = s_cnt;
    atomicMin(vid_range, s_min);
    atomicMax(vid_range + 1, s_max);
  }
}

// one warp per selected list: its chunks' live counts -> exclusive offsets in place, the total to sel_live
__global__ void __launch_bounds__(32)
    purge_scan_kernel(const int* __restrict__ sel_chunk0, int* __restrict__ chunk_cnt, int* __restrict__ sel_live) {
  const int c0 = sel_chunk0[blockIdx.x], c1 = sel_chunk0[blockIdx.x + 1];
  const int lane = threadIdx.x;
  int carry = 0;
  for (int b = c0; b < c1; b += 32) {
    const int v = b + lane < c1 ? chunk_cnt[b + lane] : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (b + lane < c1) chunk_cnt[b + lane] = carry + incl - v;
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) sel_live[blockIdx.x] = carry;
}

// V: the widest unit (<= 16 bytes) that divides code_bytes and both bases.  Ranks come from ballots over the chunk in
// position order, so survivors keep their order; the codes then move as one flat run of units, consecutive threads on
// consecutive units of the destination: a warp or more shares a long row, and a warp covers many short ones.
template <typename V>
__global__ void __launch_bounds__(256)
    purge_scatter_kernel(ListDirectory dir, const int* __restrict__ sel_list, const PurgeChunk* __restrict__ chunks,
                         const uint32_t* __restrict__ del_bits, const int* __restrict__ chunk_off, int code_bytes,
                         void* const* __restrict__ dst_data, int64_t* const* __restrict__ dst_ids,
                         unsigned long long* __restrict__ newpos, int64_t vid_min, int copies) {
  __shared__ int s_src[kPurgeChunk];
  __shared__ int s_warp[8];
  const PurgeChunk c = chunks[blockIdx.x];
  const int list = sel_list[c.sel];
  const int64_t* __restrict__ ids = dir.ids[list];
  int64_t* __restrict__ out_ids = dst_ids[c.sel];
  const int end = min(c.first + kPurgeChunk, dir.len[list]);
  const int off = chunk_off[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int nlive = 0;
  for (int p0 = c.first; p0 < end; p0 += 256) {
    const int p = p0 + threadIdx.x;
    const int64_t id = p < end ? ids[p] : -1;
    const bool live = p < end && purge_live(id, del_bits);
    const unsigned m = __ballot_sync(0xffffffffu, live);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int before = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) {
      const int v = s_warp[w];
      before += w < warp ? v : 0;
      tot += v;
    }
    if (live) {
      const int r = nlive + before + __popc(m & ((1u << lane) - 1u));
      s_src[r] = p;
      out_ids[off + r] = id;
      const unsigned long long np = ((unsigned long long)list << 32) | (unsigned)(off + r);
      if (copies == 1) {
        newpos[id - vid_min] = np;
      } else {  // the vid's first live entry met takes the first slot, its other one the second
        unsigned long long* slot = newpos + 2 * (id - vid_min);
        if (atomicCAS(slot, ~0ull, np) != ~0ull) slot[1] = np;
      }
    }
    nlive += tot;
    __syncthreads();
  }
  const int vpr = code_bytes / (int)sizeof(V);  // units per row
  const V* __restrict__ src = reinterpret_cast<const V*>(dir.codes[list]);
  V* __restrict__ dst = reinterpret_cast<V*>(dst_data[c.sel]) + (int64_t)off * vpr;
  const int units = nlive * vpr;  // <= kPurgeChunk x 16 KiB / sizeof(V)
#pragma unroll 4
  for (int u = threadIdx.x; u < units; u += 256) {
    const int e = u / vpr;
    dst[u] = src[(int64_t)s_src[e] * vpr + (u - e * vpr)];
  }
}

}  // namespace

cudaError_t launch_purge_count(ListDirectory dir, const int* sel_list, const int* sel_chunk0, int nsel,
                               const PurgeChunk* chunks, int nchunks, const uint32_t* del_bits, int* chunk_off,
                               int* sel_live, unsigned long long* vid_range, cudaStream_t st) {
  if (nsel <= 0 || nchunks <= 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(vid_range, 0xFF, 8, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(vid_range + 1, 0, 8, st);
  if (e != cudaSuccess) return e;
  purge_count_kernel<<<nchunks, 256, 0, st>>>(dir, sel_list, chunks, del_bits, chunk_off, vid_range);
  purge_scan_kernel<<<nsel, 32, 0, st>>>(sel_chunk0, chunk_off, sel_live);
  note_launch(2);
  return cudaGetLastError();
}

cudaError_t launch_purge_scatter(ListDirectory dir, const int* sel_list, const PurgeChunk* chunks, int nchunks,
                                 const uint32_t* del_bits, const int* chunk_off, int code_bytes, int align,
                                 void* const* dst_data, int64_t* const* dst_ids, unsigned long long* newpos,
                                 int64_t vid_min, cudaStream_t st, int copies) {
  if (nchunks <= 0) return cudaSuccess;
  if (code_bytes <= 0 || code_bytes > kPurgeMaxCodeBytes || align <= 0 || code_bytes % align) return cudaErrorInvalidValue;
  if (copies != 1 && copies != 2) return cudaErrorInvalidValue;
#define GB_PURGE_SCATTER(V)                                                                                          \
  purge_scatter_kernel<V><<<nchunks, 256, 0, st>>>(dir, sel_list, chunks, del_bits, chunk_off, code_bytes, dst_data, \
                                                   dst_ids, newpos, vid_min, copies)
  switch (align) {
    case 16: GB_PURGE_SCATTER(uint4); break;
    case 8: GB_PURGE_SCATTER(uint2); break;
    case 4: GB_PURGE_SCATTER(uint32_t); break;
    case 2: GB_PURGE_SCATTER(uint16_t); break;
    case 1: GB_PURGE_SCATTER(uint8_t); break;
    default: return cudaErrorInvalidValue;
  }
#undef GB_PURGE_SCATTER
  note_launch();
  return cudaGetLastError();
}

namespace {
// consecutive threads on consecutive units of the destination, as the purge's scatter; ids move in units of at most
// 8 bytes, since a chunk's ids need not fill a 16-byte unit
template <typename V>
__global__ void __launch_bounds__(256)
    list_pack_kernel(const PackChunk* __restrict__ chunks, int src_cb, int dst_cb) {
  using I = typename std::conditional<(sizeof(V) > 8), uint2, V>::type;
  const PackChunk c = chunks[blockIdx.x];
  const int svpr = src_cb / (int)sizeof(V), dvpr = dst_cb / (int)sizeof(V);
  const V* __restrict__ src = reinterpret_cast<const V*>(c.src_codes);
  V* __restrict__ dst = reinterpret_cast<V*>(c.dst_codes);
  const int units = c.n * dvpr;  // <= max(kPackChunkBytes, one code) / sizeof(V)
#pragma unroll 4
  for (int u = threadIdx.x; u < units; u += 256) {
    const int e = u / dvpr;
    dst[u] = src[(int64_t)e * svpr + (u - e * dvpr)];
  }
  const I* __restrict__ sid = reinterpret_cast<const I*>(c.src_ids);
  I* __restrict__ did = reinterpret_cast<I*>(c.dst_ids);
  const int iunits = c.n * (8 / (int)sizeof(I));
#pragma unroll 4
  for (int u = threadIdx.x; u < iunits; u += 256) did[u] = sid[u];
}
}  // namespace

cudaError_t launch_list_pack(const PackChunk* chunks, int nchunks, int src_cb, int dst_cb, int align, cudaStream_t st) {
  if (nchunks <= 0) return cudaSuccess;
  if (dst_cb <= 0 || dst_cb > src_cb || align <= 0 || src_cb % align || dst_cb % align) return cudaErrorInvalidValue;
  switch (align) {
    case 16: list_pack_kernel<uint4><<<nchunks, 256, 0, st>>>(chunks, src_cb, dst_cb); break;
    case 8: list_pack_kernel<uint2><<<nchunks, 256, 0, st>>>(chunks, src_cb, dst_cb); break;
    case 4: list_pack_kernel<uint32_t><<<nchunks, 256, 0, st>>>(chunks, src_cb, dst_cb); break;
    case 2: list_pack_kernel<uint16_t><<<nchunks, 256, 0, st>>>(chunks, src_cb, dst_cb); break;
    case 1: list_pack_kernel<uint8_t><<<nchunks, 256, 0, st>>>(chunks, src_cb, dst_cb); break;
    default: return cudaErrorInvalidValue;
  }
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_ivf_append_codes(const uint8_t* codes, int64_t n, int M, const int32_t* list, const int32_t* pos,
                                    uint8_t* const* list_codes, int64_t* const* list_ids, int64_t vid0,
                                    cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  ivf_append_codes_kernel<<<blocks_for(n, 256), 256, 0, st>>>(codes, n, M, list, pos, list_codes, list_ids, vid0);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
