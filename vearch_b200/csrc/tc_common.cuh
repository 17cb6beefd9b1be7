// Hopper (sm_90a) tensor-core building blocks shared by the tensor-core kernels (kernels_tc.cu,
// kernels_pqtc.cu): shared-memory matrix descriptors (canonical no-swizzle K-major tiles), warpgroup
// MMA wrappers (wgmma tf32 with fp32 accumulators, int8 with exact s32 accumulators, in registers) and the exchange that hands a
// 128 x 128 accumulator, held as wgmma fragments by one warpgroup, to the same warpgroup one ROW per
// thread (thread t of the warpgroup = accumulator row t), 32 columns at a time.
#pragma once
#include "common.cuh"

namespace gb {

// wgmma matrix descriptor: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base_offset 0 |
// layout_type 0 = no swizzle [62,64).  K-major no-swizzle: LBO = stride between the core matrices of
// one row group along K, SBO = stride between 8-row groups.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

// descriptor of a no-swizzle K-major operand tile at shared address `addr` (LBO 2048, SBO 128): the
// high word is constant, the low word is linear in the address
__device__ __forceinline__ uint64_t lt_desc(uint32_t addr) {
  return ((uint64_t)0x8u << 32) | (uint64_t)((addr >> 4) | 0x800000u);
}

// one 64-row half of a 128-row operand tile lies 8 row groups (8 x SBO = 1024 bytes) further
constexpr uint64_t kDescHalfM = 1024u >> 4;

// D[64 x 128] (+)= A[64 x 8] B[128 x 8]^T, tf32 operands (K-major), fp32 accumulator in registers
__device__ __forceinline__ void wg_mma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      " .reg .pred p;\n"
      " setp.ne.b32 p, %66, 0;\n"
      " wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 128] (+)= A[64 x 32] B[128 x 32]^T, int8 operands (K-major), s32 accumulator in registers (exact)
__device__ __forceinline__ void wg_mma_s8(uint32_t (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      " .reg .pred p;\n"
      " setp.ne.b32 p, %66, 0;\n"
      " wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from touching accumulator registers across an asynchronous wgmma
__device__ __forceinline__ void wg_fence_acc(float (&acc)[2][64]) {
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+f"(acc[h][i])::"memory");
}
__device__ __forceinline__ void wg_fence_acc(uint32_t (&acc)[2][64]) {
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+r"(acc[h][i])::"memory");
}

// named barrier of the 128 threads of warpgroup 0 (warps 0-3)
__device__ __forceinline__ void wg0_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
// the same barrier, returning whether `p` holds in any of the 128 threads
__device__ __forceinline__ bool wg0_any(bool p) {
  uint32_t r;
  asm volatile(
      "{\n"
      " .reg .pred p, q;\n"
      " setp.ne.u32 p, %1, 0;\n"
      " bar.red.or.pred q, 1, 128, p;\n"
      " selp.u32 %0, 1, 0, q;\n"
      "}\n"
      : "=r"(r)
      : "r"((uint32_t)p)
      : "memory");
  return r != 0;
}

// Accumulator exchange.  A slab holds 32 columns of all 128 rows (16 KiB); float4 group g of row r is
// stored at group g ^ (r & 7), so the row-per-thread reads are conflict-free.  Callers keep two slabs
// and alternate: slab (c0 / 32) & 1 is rewritten two steps later, after the next step's barrier.
constexpr int kSlabFloats = 128 * 32;
constexpr int kSlabBytes = 2 * kSlabFloats * 4;  // both slabs

// columns [c0, c0 + 32) of the fragments of warpgroup thread `t` -> slab
__device__ __forceinline__ void acc_to_slab(const float (&acc)[2][64], int c0, float* slab) {
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int jj = 0; jj < 4; jj++)
#pragma unroll
      for (int r8 = 0; r8 < 2; r8++) {
        const int i = (c0 / 8 + jj) * 4 + r8 * 2;  // fragment index: row 16w + l/4 + 8 r8, column 8 (i/4) + 2 (l%4)
        const int row = h * 64 + w * 16 + (l >> 2) + r8 * 8;
        const int col = jj * 8 + (l & 3) * 2;
        const int g = (col >> 2) ^ (row & 7);
        *reinterpret_cast<float2*>(slab + row * 32 + g * 4 + (col & 3)) = make_float2(acc[h][i], acc[h][i + 1]);
      }
}

// this thread's row of a slab
__device__ __forceinline__ void slab_row(const float* slab, uint32_t (&v)[32]) {
  const int r = threadIdx.x & 127;
#pragma unroll
  for (int g = 0; g < 8; g++) {
    const float4 x = *reinterpret_cast<const float4*>(slab + r * 32 + ((g ^ (r & 7)) * 4));
    v[4 * g] = __float_as_uint(x.x), v[4 * g + 1] = __float_as_uint(x.y);
    v[4 * g + 2] = __float_as_uint(x.z), v[4 * g + 3] = __float_as_uint(x.w);
  }
}

// columns [c0, c0 + 32) of this thread's accumulator row (c0 must be a compile-time constant after
// unrolling: the fragments are registers).  Every thread of warpgroup 0 must call it.
__device__ __forceinline__ void acc_cols(const float (&acc)[2][64], int c0, float* slabs, uint32_t (&v)[32]) {
  float* slab = slabs + ((c0 >> 5) & 1) * kSlabFloats;
  acc_to_slab(acc, c0, slab);
  wg0_sync();
  slab_row(slab, v);
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      " .reg .pred p;\n"
      " elect.sync _|p, 0xffffffff;\n"
      " selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

}  // namespace gb
