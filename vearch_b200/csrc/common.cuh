// Device-side building blocks shared by every kernel of the gamma hot path (sm_90a).
//
//  * 64-bit result keys: (order-preserving score bits << 32) | vid.  One unsigned compare gives
//    the total order the engine returns: L2 ascending / IP descending score, smaller vid first
//    among equal scores.  For an id-ordered scan this IS the faiss CMax heap order gamma's FLAT
//    index produces (index/impl/gamma_index_flat.cc:224-281; DESIGN.md "tie rule").
//  * CandQueue: threshold + candidate queue top-k kept in shared memory (K7).
//  * mbarrier / cp.async.bulk (TMA 1-D bulk copy, SASS UBLKCP) wrappers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "kernels.h"

namespace gb {


constexpr unsigned long long kKeySentinel = 0xFFFFFFFFFFFFFFFFull;
constexpr int64_t kDelIdxMask = (int64_t)1 << 63;  // realtime_mem_data.h:26 tombstone bit

// ---- order-preserving float <-> uint32 -------------------------------------------------
__host__ __device__ __forceinline__ uint32_t f2ord(float f) {
#ifdef __CUDA_ARCH__
  uint32_t b = __float_as_uint(f);
#else
  uint32_t b;
  memcpy(&b, &f, 4);
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(uint32_t o) {
  uint32_t b = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, 4);
  return f;
#endif
}
// smaller key == better result
template <int METRIC>
__host__ __device__ __forceinline__ uint32_t score2ord(float s) {
  return METRIC == kMetricL2 ? f2ord(s) : ~f2ord(s);
}
__host__ __device__ __forceinline__ uint32_t score2ord(float s, int metric) {
  return metric == kMetricL2 ? f2ord(s) : ~f2ord(s);
}
// ord of an arg-min key (k-means and list assignment): a NaN score ranks after every number, whatever its sign bit
// and the metric, as faiss's `dis < best` never takes one
template <int METRIC>
__host__ __device__ __forceinline__ uint32_t argmin_ord(float s) {
  return s != s ? 0xFFFFFFFFu : score2ord<METRIC>(s);
}
__host__ __device__ __forceinline__ float ord2score(uint32_t o, int metric) {
  return metric == kMetricL2 ? ord2f(o) : ord2f(~o);
}
__host__ __device__ __forceinline__ unsigned long long make_key(uint32_t ord, uint32_t vid) {
  return ((unsigned long long)ord << 32) | vid;
}

// float image of the bound: a score can only matter if it is on the good side of it.  The two
// sentinels (no bound yet / slot without a candidate stream) map to +-inf / NaN so the compare does the right thing.
template <int METRIC>
__device__ __forceinline__ float key_bound(unsigned long long tau) {
  const uint32_t hi = (uint32_t)(tau >> 32);
  if (METRIC == kMetricL2) return hi >= 0xFF800000u ? __int_as_float(0x7F800000) : ord2f(hi);
  const uint32_t x = ~hi;
  return x <= 0x007FFFFFu ? __int_as_float(0xFF800000) : ord2f(x);
}

// dense LSB-first bitmaps (util/bitmap_manager.h): bit id -> word id>>5, mask 1<<(id&31)
__device__ __forceinline__ bool bit_test(const uint32_t* __restrict__ bm, uint32_t id) {
  return (__ldg(bm + (id >> 5)) >> (id & 31)) & 1u;
}
// RetrievalContext::IsValid (common/gamma_common_data.h:98-106)
__device__ __forceinline__ bool ctx_is_valid(const uint32_t* del_bits, const uint32_t* filter_bits, uint32_t vid) {
  if (filter_bits && !bit_test(filter_bits, vid)) return false;
  if (del_bits && bit_test(del_bits, vid)) return false;
  return true;
}

// ---- cancellation (DESIGN.md section 8) ---------------------------------------------------
// Every translation unit has its own copy of the skip counters (no relocatable device code); each registers a reader
// with register_cancel_skips when the library loads.
namespace {
__device__ unsigned long long g_cancel_skips[kCancelSites];
cudaError_t take_cancel_skips_tu(int device, unsigned long long* acc) {
  unsigned long long h[kCancelSites];
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaMemcpyFromSymbol(h, g_cancel_skips, sizeof(h));
  if (e == cudaErrorInvalidSymbol) {  // no kernel of this unit polls: the compiler dropped its counters
    cudaGetLastError();
    return cudaSuccess;
  }
  if (e != cudaSuccess) return e;
  for (int i = 0; i < kCancelSites; i++) acc[i] += h[i];
  const unsigned long long z[kCancelSites] = {};
  return cudaMemcpyToSymbol(g_cancel_skips, z, sizeof(z));
}
[[maybe_unused]] const int g_cancel_skips_reader = register_cancel_skips(&take_cancel_skips_tu);
}  // namespace

// The CTA-wide poll of a cancel word (CancelPoll), called by every thread of the CTA at a work-unit boundary, before
// any mbarrier is initialised: one thread reads `seen` and, in one CTA of kCancelPollStride, the host word itself
// (system scope: the host sets it while the kernel runs; reads of one host address from every CTA would queue on
// PCIe), the barrier hands its answer to the whole CTA, and a CTA that is to skip counts itself once in its kernel's
// counter.  A null word costs one uniform branch and no barrier.
__device__ __forceinline__ bool cta_cancelled(CancelPoll c, int site) {
  if (c.word == nullptr) return false;
  const bool first = threadIdx.x == 0 && threadIdx.y == 0 && threadIdx.z == 0;
  int set = 0;
  if (first) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(c.seen) : "memory");
    const unsigned b = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
    if (v == 0 && b % kCancelPollStride == 0) {
      asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(c.word) : "memory");
      if (v) asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(c.seen), "r"(1u) : "memory");
    }
    set = v != 0;
  }
  set = __syncthreads_or(set);
  if (set && first) atomicAdd(&g_cancel_skips[site], 1ull);
  return set != 0;
}

// ---- shared-memory helpers ---------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      " .reg .pred p;\n"
      " mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      " selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (complete_tx::bytes).
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- block-wide bitonic sort of uint64 keys in shared memory (ascending), n a power of two.
// Caller guarantees a __syncthreads() happened after the last write to a[]; returns synchronised.
__device__ __forceinline__ void block_bitonic_sort(unsigned long long* a, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
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
      __syncthreads();
    }
  }
}

// ---- CandQueue: top-k by threshold + candidate queue -------------------------------------
// buf[0, KP)      current best keys, sorted ascending, sentinel padded  (KP = pow2 >= k)
// buf[KP, SORTN)  unsorted candidates that beat tau when they were pushed
// A flush sorts the whole buffer and re-derives tau = k-th best.  Candidates that do not beat
// tau are never stored, so after the first flush pushes become rare (expected k*ln(n/k)).
struct CandQueue {
  unsigned long long* buf;
  int* cnt;                 // shared
  unsigned long long* tau;  // shared
  int k, KP, SORTN;

  __device__ __forceinline__ int cap() const { return SORTN - KP; }

  __device__ __forceinline__ void init() {
    for (int i = threadIdx.x; i < SORTN; i += blockDim.x) buf[i] = kKeySentinel;
    if (threadIdx.x == 0) {
      *cnt = 0;
      *tau = kKeySentinel;
    }
    __syncthreads();
  }
  // every lane of the warp must call this (converged)
  __device__ __forceinline__ void push_warp(bool pred, unsigned long long key) {
    unsigned mask = __ballot_sync(0xffffffffu, pred);
    if (mask) {
      int lane = threadIdx.x & 31;
      int leader = __ffs(mask) - 1;
      int base = 0;
      if (lane == leader) base = atomicAdd(cnt, __popc(mask));
      base = __shfl_sync(0xffffffffu, base, leader);
      if (pred) buf[KP + base + __popc(mask & ((1u << lane) - 1u))] = key;
    }
  }
  // all threads; must be preceded by a __syncthreads() after the last push.  Small buffers are
  // sorted (bitonic, occupied prefix only); big ones go through an MSB radix select, whose cost is
  // linear in the fill.  final_sort: leave buf[0, KP) sorted ascending (the kernel's result).
  // exact: leave exactly the k best in buf[0, k) (no slack keys) -- for a final flush whose caller does not sort
  __device__ __forceinline__ void flush(bool final_sort = false, bool exact = false) {
    int c = *cnt;
    if (KP + c > kSelectMin) {
      flush_select(c, final_sort, exact);
      return;
    }
    // only the occupied prefix needs sorting: everything behind it is (made) sentinel
    int n = KP;
    while (n < KP + c) n <<= 1;
    if (n < 2 * KP && n < SORTN) n = 2 * KP;
    for (int i = KP + c + threadIdx.x; i < n; i += blockDim.x) buf[i] = kKeySentinel;
    __syncthreads();
    block_bitonic_sort(buf, n);
    if (threadIdx.x == 0) {
      *cnt = 0;
      *tau = buf[k - 1];
    }
    __syncthreads();
  }

  // above this fill the flush is a radix select (linear in the fill) instead of a bitonic sort: a 1 Ki-key sort per
  // flush dominated the instructions of a one-list scan with k = 400
  static constexpr int kSelectMin = 512;

  // Radix-select flush.  Finds the shortest byte prefix P (most significant bytes first) such that
  // between k and KP valid keys are <= P|11..1, compacts those keys to buf[0, kept) in place
  // (unordered), pads buf[kept, KP) with sentinels and sets tau = P|11..1.  That tau is >= the true
  // k-th best key and < every discarded key, so the "key < tau" admission test never loses a top-k
  // key; the up to KP - k extra keys ride along until the final sort drops them.  Stopping as soon as
  // the selected bin fits the slack (instead of descending until exactly k remain) saves most of the
  // 8 byte passes when scores share their leading bytes: with k = 400 the flushes were 40 % of a
  // one-list scan (phase A of the tensor-core filter).  Keys are unique (one vid appears once per
  // query), which bounds the loop at 8 passes.
  __device__ __forceinline__ void flush_select(int c, bool final_sort, bool exact = false) {
    __shared__ int s_hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_need, s_done, s_valid, s_pos;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
    const int n = KP + c;
    if (tid == 0) {
      s_valid = 0;
      s_pos = 0;
    }
    unsigned long long prefix = 0, tup = kKeySentinel;
    int need = k;
    bool all_valid = false;
    for (int shift = 56;; shift -= 8) {
      for (int i = tid; i < 256; i += nt) s_hist[i] = 0;
      __syncthreads();
      int myvalid = 0;
      for (int i = tid; i < n; i += nt) {
        unsigned long long key = buf[i];
        bool match;
        if (shift == 56) {
          myvalid += key != kKeySentinel;
          match = true;
        } else {
          match = (key >> (shift + 8)) == prefix;
        }
        // (a warp-aggregated add via __match_any_sync was slower than the plain shared atomics)
        if (match) atomicAdd(&s_hist[(int)(key >> shift) & 255], 1);
      }
      if (shift == 56) {
        myvalid = __reduce_add_sync(0xffffffffu, myvalid);
        if (lane == 0 && myvalid) atomicAdd(&s_valid, myvalid);
      }
      __syncthreads();
      if (shift == 56 && s_valid <= k) {
        all_valid = true;
        break;
      }
      if (tid < 32) {
        int h[8], sum = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) {
          h[j] = s_hist[lane * 8 + j];
          sum += h[j];
        }
        int incl = sum;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          int v = __shfl_up_sync(0xffffffffu, incl, off);
          if (lane >= off) incl += v;
        }
        int before = incl - sum;
        if (before < need && need <= incl) {
#pragma unroll
          for (int j = 0; j < 8; j++) {
            if (before < need && need <= before + h[j]) {
              s_prefix = (prefix << 8) | (unsigned long long)(lane * 8 + j);
              s_need = need - before;
              // keeping the whole bin leaves k - (need - before) + h[j] keys: done when that fits KP
              s_done = (h[j] - (need - before) <= (exact ? 0 : KP - k)) ? 1 : 0;
            }
            before += h[j];
          }
        }
      }
      __syncthreads();
      prefix = s_prefix;
      need = s_need;
      if (s_done || shift == 0) {
        tup = shift == 0 ? prefix : ((prefix << shift) | ((1ull << shift) - 1ull));
        break;
      }
    }
    // in-place compaction: a chunk is read, then (after the barrier) its survivors are written to
    // positions below the number of keys read so far
    for (int base = 0; base < n; base += nt) {
      int i = base + tid;
      unsigned long long key = i < n ? buf[i] : kKeySentinel;
      __syncthreads();
      bool keep = key != kKeySentinel && (all_valid || key <= tup);
      unsigned mask = __ballot_sync(0xffffffffu, keep);
      if (mask) {
        int leader = __ffs(mask) - 1, pos = 0;
        if (lane == leader) pos = atomicAdd(&s_pos, __popc(mask));
        pos = __shfl_sync(0xffffffffu, pos, leader);
        if (keep) buf[pos + __popc(mask & ((1u << lane) - 1u))] = key;
      }
    }
    __syncthreads();
    const int kept = s_pos;
    for (int i = kept + tid; i < KP; i += nt) buf[i] = kKeySentinel;
    if (tid == 0) {
      *cnt = 0;
      if (!all_valid) *tau = tup;
    }
    __syncthreads();
    if (final_sort) block_bitonic_sort(buf, KP);
  }
};

__host__ __device__ __forceinline__ int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

}  // namespace gb
