// Scalar filters on the device: one launch evaluates a request's filters over every document and writes the combined
// LSB-first bitmap with its cardinality; one scatter kernel applies a batch of staged values to a column.
#include "kernels.h"

namespace gb {

namespace {

__device__ __forceinline__ bool in_sorted(const int32_t* __restrict__ t, int n, int32_t c) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const int32_t v = __ldg(t + mid);
    if (v < c) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && __ldg(t + lo) == c;
}

template <typename T>
__device__ __forceinline__ bool cmp_hit(const FilterDesc& f, T v, T lo, T hi) {
  if (f.equal) return f.lo_ok && (f.neg ? v != lo : v == lo);
  bool hit = true;
  if (f.has_lo) hit = f.lo_ok && (v > lo || (v == lo && f.inc_lo));
  if (hit && f.has_hi) hit = f.hi_ok && (v < hi || (v == hi && f.inc_hi));
  return hit;
}

// filter f on document d (d < the request's n)
__device__ bool eval_one(const FilterDesc& f, int64_t d) {
  if (f.kind == kFilterNumeric) {
    if (d >= f.ncol || !((__ldg(f.valid + (d >> 5)) >> (d & 31)) & 1u)) return false;  // absent or invalid: no match
    if (f.is_float) {
      const double v = f.width == 4 ? (double)__ldg(static_cast<const float*>(f.col) + d)
                                    : __ldg(static_cast<const double*>(f.col) + d);
      return cmp_hit<double>(f, v, f.lo_f, f.hi_f);
    }
    int64_t v;
    if (f.width == 1) v = __ldg(static_cast<const uint8_t*>(f.col) + d);
    else if (f.width == 4) v = __ldg(static_cast<const int32_t*>(f.col) + d);
    else v = __ldg(static_cast<const long long*>(f.col) + d);
    return cmp_hit<int64_t>(f, v, f.lo_i, f.hi_i);
  }
  bool in = false;
  if (d < f.ncol) {
    if (f.kind == kFilterString) {
      in = in_sorted(f.terms, f.nterms, __ldg(f.codes + d));
    } else {
      const int64_t off = __ldg(f.arr_off + d);
      const int cnt = __ldg(f.arr_cnt + d);
      for (int j = 0; j < cnt && !in; j++) in = in_sorted(f.terms, f.nterms, __ldg(f.pool + off + j));
    }
  }
  return f.neg ? !in : in;  // NotIn: every document below n that is not in, with or without a value
}

__global__ void __launch_bounds__(256) filter_eval_kernel(const FilterDesc* __restrict__ fd, int nf, int op, int64_t n,
                                                          int64_t words, uint32_t* __restrict__ out,
                                                          unsigned long long* __restrict__ card) {
  const int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool acc = false;
  if (d < n) {
    acc = eval_one(fd[0], d);
    for (int i = 1; i < nf; i++) {
      // what the remaining filters cannot change is not evaluated
      if (op == 0 ? !acc : (op == 1 ? acc : true)) break;
      acc = eval_one(fd[i], d);
    }
  }
  const uint32_t w = __ballot_sync(0xffffffffu, acc);
  const int64_t wi = d >> 5;
  if ((threadIdx.x & 31) == 0 && wi < words) out[wi] = w;
  // one atomic per block: a counter shared by every warp of a dense result serialises on its address
  const int hits = __syncthreads_count(acc);
  if (threadIdx.x == 0 && hits) atomicAdd(card, (unsigned long long)hits);
}

__global__ void scatter_column_kernel(const int32_t* __restrict__ docs, const uint64_t* __restrict__ vals,
                                      const uint8_t* __restrict__ ok, int64_t m, int width, void* __restrict__ col,
                                      uint32_t* __restrict__ valid) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int64_t d = docs[i];
  const uint64_t v = vals[i];
  if (width == 1) static_cast<uint8_t*>(col)[d] = (uint8_t)v;
  else if (width == 4) static_cast<uint32_t*>(col)[d] = (uint32_t)v;
  else static_cast<unsigned long long*>(col)[d] = (unsigned long long)v;
  if (valid) {
    const uint32_t bit = 1u << (d & 31);
    if (ok[i]) atomicOr(valid + (d >> 5), bit);
    else atomicAnd(valid + (d >> 5), ~bit);
  }
}

}  // namespace

cudaError_t launch_filter_eval(const FilterDesc* fd, int nf, int op, int64_t n, int64_t words, uint32_t* out,
                               unsigned long long* card, cudaStream_t st) {
  if (words <= 0) return cudaSuccess;
  if (nf <= 0) return cudaErrorInvalidValue;
  const int64_t threads = words * 32;
  filter_eval_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(fd, nf, op, n, words, out, card);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_scatter_column(const int32_t* docs, const uint64_t* vals, const uint8_t* ok, int64_t m, int width,
                                  void* col, uint32_t* valid, cudaStream_t st) {
  if (m <= 0) return cudaSuccess;
  scatter_column_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(docs, vals, ok, m, width, col, valid);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
