// Counter-based Philox4x32-10 generator (Salmon et al., SC'11), written from
// the published round function. Every random decision in the collect path is a
// pure function of (seed, stream id, counter), so env i at step t draws the
// same numbers whatever the grid shape or GPU count.
#pragma once
#include <stdint.h>

struct jb_philox4 { uint32_t x, y, z, w; };

__host__ __device__ __forceinline__ void jb_mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
#ifdef __CUDA_ARCH__
  hi = __umulhi(a, b);
  lo = a * b;
#else
  uint64_t p = (uint64_t)a * (uint64_t)b;
  hi = (uint32_t)(p >> 32);
  lo = (uint32_t)p;
#endif
}

// key = 64-bit seed; counter = (ctr, stream) each 64-bit.
__host__ __device__ __forceinline__ jb_philox4 jb_philox(uint64_t seed, uint64_t stream, uint64_t ctr) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32);
  uint32_t c2 = (uint32_t)stream, c3 = (uint32_t)(stream >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, lo0, hi1, lo1;
    jb_mulhilo(0xD2511F53u, c0, hi0, lo0);
    jb_mulhilo(0xCD9E8D57u, c2, hi1, lo1);
    uint32_t n0 = hi1 ^ c1 ^ k0;
    uint32_t n1 = lo1;
    uint32_t n2 = hi0 ^ c3 ^ k1;
    uint32_t n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  jb_philox4 o; o.x = c0; o.y = c1; o.z = c2; o.w = c3;
  return o;
}

// 53-bit uniform in [0,1) from two 32-bit words.
__host__ __device__ __forceinline__ double jb_u01_double(uint32_t a, uint32_t b) {
  uint64_t v = (((uint64_t)a) << 21) ^ (uint64_t)(b >> 11);   // 53 bits
  v &= ((1ull << 53) - 1);
  return (double)v * (1.0 / 9007199254740992.0);
}
// 24-bit uniform in [0,1) from one 32-bit word.
__host__ __device__ __forceinline__ float jb_u01_float(uint32_t a) {
  return (float)(a >> 8) * (1.0f / 16777216.0f);
}

// Two standard normals from one Philox draw by Box-Muller: u1 in (0,1] from x (so logf stays finite), u2 in [0,1) from y.
__device__ __forceinline__ void jb_normal_pair(uint64_t seed, uint64_t stream, uint64_t ctr, float& n0, float& n1) {
  jb_philox4 r = jb_philox(seed, stream, ctr);
  const float u1 = (float)((r.x >> 8) + 1u) * (1.0f / 16777216.0f);
  const float u2 = jb_u01_float(r.y);
  const float rad = sqrtf(-2.0f * logf(u1));
  n0 = rad * cospif(2.0f * u2);
  n1 = rad * sinpif(2.0f * u2);
}

// Per-row draw counter of the act kernels: returns base + row_ctr[m] and advances row_ctr[m], so that every launch (and
// every CUDA-graph replay) draws fresh numbers; base when there is no counter.
__device__ __forceinline__ uint64_t jb_next_row_ctr(long long* __restrict__ row_ctr, int m, uint64_t base = 0) {
  if (row_ctr) { base += (uint64_t)row_ctr[m]; row_ctr[m] += 1; }
  return base;
}
