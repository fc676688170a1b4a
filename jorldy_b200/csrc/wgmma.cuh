// Hopper warpgroup MMA (wgmma, sm_90a) building blocks for the 3xTF32 tensor-core products of csrc/tc_gemm.cu and
// csrc/ppo_fused.cu.  Operand tiles live in shared memory in the canonical K-major SWIZZLE_128B layout: one 128-byte row
// (32 fp32 of K) per tile row, eight rows per 1 KB atom, 16-byte chunk index XOR row-in-atom.  A warpgroup (128 threads)
// computes a 64-row slice of the tile; its fp32 accumulator lives in registers:
//   d[4 j + 0 / 1] = D[16 w + l / 4][8 j + 2 (l % 4) + 0 / 1],  d[4 j + 2 / 3] = the same columns of row + 8
// (w = warp in the warpgroup, l = lane).
#pragma once
#include <stdint.h>

namespace jbwg {

__device__ __forceinline__ uint32_t tile_off(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

// Shared-memory matrix descriptor (sm_90 bit layout), K-major SWIZZLE_128B.  `smem_addr` = 1 KB-aligned atom base + 32
// bytes per K = 8 step inside the 128-byte swizzle row.
__device__ __forceinline__ uint64_t desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);           // start address        bits [0,14)
  d |= (uint64_t)1 << 16;                               // leading byte offset  bits [16,30): unused for swizzled K-major
  d |= (uint64_t)(1024 >> 4) << 32;                     // stride byte offset   bits [32,46): 1 KB between 8-row atoms
  d |= (uint64_t)1 << 62;                               // layout type          bits [62,64): 1 = SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64][32] (+)= A[64][8] B[32][8]^T, tf32 operands (the tensor core ignores the low 13 mantissa bits), fp32 accumulate
__device__ __forceinline__ void mma_n32(float (&d)[16], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate));
}

// D[64][128] (+)= A[64][8] B[128][8]^T, as above
__device__ __forceinline__ void mma_n128(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}

// 3xTF32 over one 32-deep chunk (four K = 8 steps): D += a_hi b_hi + a_hi b_lo + a_lo b_hi.  a_* / b_* are the shared
// addresses of this warpgroup's A rows and of the B rows; `first` starts a fresh accumulation.
__device__ __forceinline__ void mma3_n32(float (&d)[16], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, bool first) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t ko = 32u * j;
    mma_n32(d, desc(a_hi + ko), desc(b_hi + ko), (first && j == 0) ? 0 : 1);
    mma_n32(d, desc(a_hi + ko), desc(b_lo + ko), 1);
    mma_n32(d, desc(a_lo + ko), desc(b_hi + ko), 1);
  }
}

// accumulator of an m64n32 warpgroup tile -> stage[row * ld + col] (rows 64 wg .. + 63 of the 128-row tile)
__device__ __forceinline__ void store_acc_n32(const float (&d)[16], float* stage, int ld) {
  const int t = threadIdx.x & 127, row = (threadIdx.x >> 7) * 64 + (t >> 5) * 16 + ((t & 31) >> 2), col = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    *reinterpret_cast<float2*>(&stage[row * ld + 8 * j + col]) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(&stage[(row + 8) * ld + 8 * j + col]) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

}  // namespace jbwg
