// BINARYIVF kernels (K12): Hamming distances over packed binary rows on the CUDA cores, the ±1 expansion around the
// faiss-Clustering k-means of the coarse centroids, and the Hamming codec of the query-major list scan (list_scan.cuh).
//
// A binary row is d / 8 bytes, bit i of the vector at bit (i & 7) of byte i >> 3 (faiss's packing).  Device rows are
// kept 4-byte padded with zero bytes (the raw store pads to 16), so the distance of two rows is the popcount of the XOR
// of their 32-bit words: the pad words XOR to zero.  Distances are integers; as fp32 they are exact up to 2^24 bits.
#include "common.cuh"
#include "list_scan.cuh"

namespace gb {
namespace {

constexpr int HT_ROWS = 128;  // rows per CTA, one per thread
constexpr int HT_QB = 16;     // queries per CTA, held in shared memory
constexpr int HT_MAXW = 64;   // words of a query chunk in shared memory (256 bytes); longer rows loop over chunks

// out[q][r] = popcount(Q_q ^ R_r) over W 32-bit words.  One thread per row, HT_QB queries per CTA from shared memory:
// each row word is loaded once and XORed with every query of the tile.
__global__ void __launch_bounds__(HT_ROWS)
    hamming_tile_kernel(const uint32_t* __restrict__ Q, int64_t ldq, int nq, const uint32_t* __restrict__ R, int64_t ldr,
                        int m, int W, float* __restrict__ out, int64_t ldo, CancelPoll cancel) {
  if (cta_cancelled(cancel, kCsHammingTile)) return;
  __shared__ uint32_t qs[HT_QB][HT_MAXW];
  const int q0 = blockIdx.y * HT_QB;
  const int nqb = min(HT_QB, nq - q0);
  const int r = blockIdx.x * HT_ROWS + threadIdx.x;
  const uint32_t* row = R + (int64_t)min(r, m - 1) * ldr;
  int acc[HT_QB];
#pragma unroll
  for (int j = 0; j < HT_QB; j++) acc[j] = 0;
  for (int w0 = 0; w0 < W; w0 += HT_MAXW) {
    const int nw = min(HT_MAXW, W - w0);
    __syncthreads();
    for (int i = threadIdx.x; i < HT_QB * HT_MAXW; i += HT_ROWS) {
      const int j = i / HT_MAXW, w = i % HT_MAXW;
      qs[j][w] = (j < nqb && w < nw) ? Q[(int64_t)(q0 + j) * ldq + w0 + w] : 0u;
    }
    __syncthreads();
    for (int w = 0; w < nw; w++) {
      const uint32_t x = __ldg(row + w0 + w);
#pragma unroll
      for (int j = 0; j < HT_QB; j++) acc[j] += __popc(x ^ qs[j][w]);
    }
  }
  if (r >= m) return;
#pragma unroll
  for (int j = 0; j < HT_QB; j++)
    if (j < nqb) out[(int64_t)(q0 + j) * ldo + r] = (float)acc[j];
}

// faiss binary_to_real: out[i][j] = bit j of row i ? +1 : -1, j < d (d a multiple of 8; ldo >= d floats)
__global__ void binary_to_real_kernel(const uint8_t* __restrict__ x, int64_t ldx, int64_t n, int d, float* __restrict__ out,
                                      int64_t ldo) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  const int64_t i = t / d;
  const int j = (int)(t - i * d);
  out[i * ldo + j] = ((x[i * ldx + (j >> 3)] >> (j & 7)) & 1) ? 1.0f : -1.0f;
}

// faiss real_to_binary: byte b of row i = bits (x[i][8 b + k] > 0) << k; bytes [d / 8, ldo) are zeroed
__global__ void real_to_binary_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d, uint8_t* __restrict__ out,
                                      int64_t ldo) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * ldo) return;
  const int64_t i = t / ldo;
  const int b = (int)(t - i * ldo);
  uint32_t v = 0;
  if (b < d / 8) {
    const float* xi = x + i * ldx + 8 * b;
#pragma unroll
    for (int k = 0; k < 8; k++) v |= (xi[k] > 0.0f ? 1u : 0u) << k;
  }
  out[t] = (uint8_t)v;
}

__host__ __device__ inline int bin_tile_entries(int code_size) {  // ~16 KiB of codes, 256..1024 entries
  int e = 16384 / code_size;
  e = (e / LS_NT) * LS_NT;
  return e < LS_NT ? LS_NT : (e > 1024 ? 1024 : e);
}

// The Hamming codec of the list scan: the "table" is the query's packed words, an entry's score is the popcount of the
// XOR of its words with them (smaller is better, the list's coarse distance takes no part).  Entries are code_size bytes
// apart in the stage, so they start at any byte: each word of an entry is funnel-shifted out of the two aligned words
// holding it, and the bytes of its last word past the entry are masked off.
struct BinaryHammingCodec {
  using Entry = uint32_t;
  static constexpr bool kDis0 = false;
  static constexpr bool kCodeSum = true;
  static constexpr int kMinCtasPerSm = 0;
  const uint32_t* queries;  // [nq][ldq] words, zero padded past code_size bytes
  int64_t ldq;
  int cb;

  __host__ __device__ int words() const { return (cb + 3) / 4; }
  __host__ __device__ int code_bytes() const { return cb; }
  __host__ __device__ int table_entries() const { return (words() + 3) & ~3; }
  int tile_entries() const { return bin_tile_entries(cb); }
  __host__ __device__ static constexpr int pt(int) { return 1; }  // not used: MW = 0 only

  __device__ __forceinline__ void cta_begin(uint32_t* tab, int q, int metric) const {
    (void)metric;
    for (int i = threadIdx.x; i < table_entries(); i += LS_NT) tab[i] = i < words() ? queries[(int64_t)q * ldq + i] : 0u;
    __syncthreads();
  }
  __device__ __forceinline__ void list_begin(uint32_t*, int, int) const {}
  using Acc = int;
  __device__ __forceinline__ int start(float) const { return 0; }
  __device__ __forceinline__ float finish(int acc) const { return (float)acc; }
  __device__ __forceinline__ int code_sum(const unsigned char* code, const uint32_t* __restrict__ tab, int acc) const {
    const uintptr_t a = reinterpret_cast<uintptr_t>(code);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3) * 8;
    const int W = words();
    uint32_t lo = w[0];
    for (int i = 0; i < W; i++) {
      // the word after the entry's last byte is read only when the entry is not word aligned (sh > 0), and then lies in
      // the stage or in the launcher's 16-byte pad
      const uint32_t hi = sh ? w[i + 1] : 0u;
      uint32_t x = __funnelshift_r(lo, hi, sh);
      const int rem = cb - 4 * i;
      if (rem < 4) x &= (1u << (8 * rem)) - 1u;
      acc += __popc(x ^ tab[i]);
      lo = hi;
      if (!sh && i + 1 < W) lo = w[i + 1];
    }
    return acc;
  }
};

int64_t blocks_of(int64_t n, int nt) { return (n + nt - 1) / nt; }

}  // namespace

cudaError_t launch_hamming_tile(const uint32_t* Q, int64_t ldq, int nq, const uint32_t* R, int64_t ldr, int m, int words,
                                float* out, int64_t ldo, cudaStream_t st, CancelPoll cancel) {
  if (nq <= 0 || m <= 0) return cudaSuccess;
  static_assert(kHammingTileMaxQueries == 65535 * HT_QB, "one launch: at most 65535 query tiles");
  if (words <= 0 || nq > kHammingTileMaxQueries) return cudaErrorInvalidValue;
  dim3 grid((unsigned)blocks_of(m, HT_ROWS), (unsigned)blocks_of(nq, HT_QB));
  hamming_tile_kernel<<<grid, HT_ROWS, 0, st>>>(Q, ldq, nq, R, ldr, m, words, out, ldo, cancel);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_binary_to_real(const uint8_t* x, int64_t ldx, int64_t n, int d, float* out, int64_t ldo, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  if (d % 8 || ldo < d) return cudaErrorInvalidValue;
  binary_to_real_kernel<<<(unsigned)blocks_of(n * d, 256), 256, 0, st>>>(x, ldx, n, d, out, ldo);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_real_to_binary(const float* x, int64_t ldx, int64_t n, int d, uint8_t* out, int64_t ldo, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  if (d % 8 || ldo < d / 8) return cudaErrorInvalidValue;
  real_to_binary_kernel<<<(unsigned)blocks_of(n * ldo, 256), 256, 0, st>>>(x, ldx, n, d, out, ldo);
  note_launch();
  return cudaGetLastError();
}

int binary_scan_max_k(int code_size) {
  if (code_size <= 0) return 0;
  return list_scan_max_k(BinaryHammingCodec{nullptr, 0, code_size});
}

cudaError_t launch_binary_ivf_scan(const uint32_t* queries, int64_t ldq, int nq, const int32_t* probe_ids, int nprobe, int pg,
                                   ListDirectory dir, int code_size, int k, FilterArgs f, unsigned long long* partial,
                                   cudaStream_t st) {
  const BinaryHammingCodec c{queries, ldq, code_size};
  const ListScanArgs a{probe_ids, nullptr, nprobe, nprobe, pg, dir, k, f, nullptr, 0, nullptr, true, partial};
  return launch_list_scan<BinaryHammingCodec, kMetricL2, 0>(c, nq, a, st);
}

}  // namespace gb
