// K7: result selection and merge.
//
// Replaces the faiss heap usage of the reference: heap_heapify / heap_pop / heap_push /
// heap_replace_top / heap_reorder in GammaFLATIndex::Search (gamma_index_flat.cc:208-281),
// the scanners (gamma_index_ivfflat.h:83-87, gamma_index_ivfpq.h:340-346), the thread-local
// heap merges heap_addn (gamma_index_flat.cc:334-340, gamma_index_ivfflat.cc:764-770,
// gamma_index_ivfpq.cc:902-911) and the coarse quantiser's per-row k-select.
//
// One CTA per row.  The stream of candidates is filtered against the running k-th best (tau);
// survivors go to a shared-memory queue that is sorted (block bitonic) only when it fills up.
// Filters are applied before selection, exactly as the CPU scan does (IsValid, score window).
#include <float.h>

#include "common.cuh"
#include "kernels.h"

namespace gb {

namespace {

constexpr int SEL_NT = 256;
constexpr int SEL_ITEMS = 4;  // per thread per round

template <bool KEYS_IN>
__global__ void __launch_bounds__(SEL_NT)
    select_rows_kernel(const void* __restrict__ in, int64_t ld, int m, int64_t id_base, int k, int KP, int SORTN,
                       int metric, FilterArgs f, unsigned long long* __restrict__ out_keys, int64_t out_stride) {
  if (cta_cancelled(f.cancel, kCsSelectRows)) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(smem_raw);
  __shared__ int s_cnt;
  __shared__ unsigned long long s_tau;
  CandQueue cq{buf, &s_cnt, &s_tau, k, KP, SORTN};
  cq.init();

  const int64_t row = blockIdx.x;
  const float* srow = KEYS_IN ? nullptr : reinterpret_cast<const float*>(in) + row * ld;
  const unsigned long long* krow = KEYS_IN ? reinterpret_cast<const unsigned long long*>(in) + row * ld : nullptr;
  const int per_round = SEL_NT * SEL_ITEMS;

  for (int base = 0; base < m; base += per_round) {
    unsigned long long tau = s_tau;
    unsigned long long key[SEL_ITEMS];
    bool ok[SEL_ITEMS];
#pragma unroll
    for (int u = 0; u < SEL_ITEMS; u++) {
      int col = base + u * SEL_NT + threadIdx.x;
      ok[u] = col < m;
      key[u] = kKeySentinel;
      if (ok[u]) {
        if (KEYS_IN) {
          key[u] = krow[col];
        } else {
          float s = srow[col];
          ok[u] = (s <= f.max_score) && (s >= f.min_score);
          key[u] = make_key(score2ord(s, metric), (uint32_t)(id_base + col));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < SEL_ITEMS; u++) {
      bool p = ok[u] && key[u] < tau;
      if (!KEYS_IN && p) p = ctx_is_valid(f.del_bits, f.filter_bits, (uint32_t)key[u]);
      cq.push_warp(p, key[u]);
    }
    __syncthreads();
    const int c_now = s_cnt;
    __syncthreads();  // same snapshot in every thread before any warp pushes again
    if (base + per_round < m && c_now + per_round > cq.cap()) cq.flush();
  }
  cq.flush(true);
  for (int i = threadIdx.x; i < k; i += blockDim.x) out_keys[row * out_stride + i] = buf[i];
}

__global__ void decode_keys_kernel(const unsigned long long* __restrict__ keys, int64_t ld, int k, int metric,
                                   float* __restrict__ out_dis, int64_t* __restrict__ out_ids, int64_t id_or) {
  const int64_t row = blockIdx.x;
  const unsigned long long* kr = keys + row * ld;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    unsigned long long key = kr[i];
    int j = i;
    if (key != kKeySentinel && metric == kMetricIP) {
      // heap_reorder on a CMin heap lists equal scores with the larger id first
      uint32_t hi = (uint32_t)(key >> 32);
      int s = i, e = i + 1;
      while (s > 0 && (uint32_t)(kr[s - 1] >> 32) == hi) s--;
      while (e < k && kr[e] != kKeySentinel && (uint32_t)(kr[e] >> 32) == hi) e++;
      j = s + (e - 1 - i);
    }
    if (key == kKeySentinel) {
      out_dis[row * k + i] = metric == kMetricL2 ? FLT_MAX : -FLT_MAX;  // heap neutral values
      out_ids[row * k + i] = -1;
    } else {
      out_dis[row * k + j] = ord2score((uint32_t)(key >> 32), metric);
      out_ids[row * k + j] = (int64_t)(uint32_t)key | id_or;
    }
  }
}

__global__ void split_keys_kernel(const unsigned long long* __restrict__ keys, int64_t n, int metric,
                                  float* __restrict__ out_scores, int32_t* __restrict__ out_ids) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long key = keys[i];
  if (key == kKeySentinel) {
    if (out_scores) out_scores[i] = metric == kMetricL2 ? FLT_MAX : -FLT_MAX;
    out_ids[i] = -1;
  } else {
    if (out_scores) out_scores[i] = ord2score((uint32_t)(key >> 32), metric);
    out_ids[i] = (int32_t)(uint32_t)key;
  }
}

void select_geometry(int k, int m, int* KP, int* SORTN) {
  *KP = next_pow2(k < 16 ? 16 : k);
  if (*KP - k < k / 4 && *KP < 4096) *KP *= 2;  // slack for the radix-select flush to stop early (common.cuh)
  int per_round = SEL_NT * SEL_ITEMS;
  *SORTN = next_pow2(*KP + (m < per_round ? m : per_round));  // single-round inputs never flush mid-way
}

template <bool KEYS_IN>
cudaError_t launch_select(const void* in, int64_t ld, int nrows, int m, int64_t id_base, int k, int metric, FilterArgs f,
                          unsigned long long* out_keys, int64_t out_stride, cudaStream_t st) {
  if (nrows <= 0) return cudaSuccess;
  if (k <= 0 || k > 4096) return cudaErrorInvalidValue;
  int KP, SORTN;
  select_geometry(k, m, &KP, &SORTN);
  size_t smem = (size_t)SORTN * 8;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(select_rows_kernel<KEYS_IN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return e;
  }
  select_rows_kernel<KEYS_IN><<<nrows, SEL_NT, smem, st>>>(in, ld, m, id_base, k, KP, SORTN, metric, f, out_keys,
                                                         out_stride);
                                                         note_launch();
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_select_scores(const float* scores, int64_t ld, int nrows, int m, int64_t id_base, int k, int metric,
                                 FilterArgs f, unsigned long long* out_keys, int64_t out_stride, cudaStream_t st) {
  return launch_select<false>(scores, ld, nrows, m, id_base, k, metric, f, out_keys, out_stride, st);
}

cudaError_t launch_select_keys(const unsigned long long* keys, int64_t ld, int nrows, int m, int k,
                               unsigned long long* out_keys, int64_t out_stride, cudaStream_t st) {
  FilterArgs f{nullptr, nullptr, -FLT_MAX, FLT_MAX};
  return launch_select<true>(keys, ld, nrows, m, 0, k, kMetricL2, f, out_keys, out_stride, st);
}

cudaError_t launch_decode_keys(const unsigned long long* keys, int64_t ld, int nrows, int k, int metric, float* out_dis,
                               int64_t* out_ids, int64_t id_or, cudaStream_t st) {
  if (nrows <= 0) return cudaSuccess;
  decode_keys_kernel<<<nrows, 128, 0, st>>>(keys, ld, k, metric, out_dis, out_ids, id_or);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_split_keys(const unsigned long long* keys, int64_t n, int metric, float* out_scores, int32_t* out_ids,
                              cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  split_keys_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(keys, n, metric, out_scores, out_ids);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
