// Large-M dense forward on the Hopper tensor cores (wgmma), fp32-grade accuracy by 3xTF32 operand splitting:
// y[M,N] = act(x[M,K] W[N,K]^T + b).
//
// Used for the products whose M is the number of env rows (act() over thousands of batched envs,
// the PPO pre-pass over N*T rows: policy_value.py:19-22 / q_network.py:17-20 second layer), where a
// 128x128 tile grid fills the 132 SMs.  The minibatch-sized products stay on the fp32 FFMA kernels
// (tile granularity M=128 would leave most SMs idle there, see DESIGN.md 4).
//
// Accuracy: wgmma .tf32 reads fp32 words from shared memory and keeps 10 mantissa bits.  Each operand is
// split a = a_hi + a_lo with a_hi = the tf32 truncation the hardware applies to the raw fp32 word and
// a_lo = a - a_hi (computed here, itself fed as tf32), and three MMAs are accumulated in fp32 registers:
// a_hi b_hi + a_hi b_lo + a_lo b_hi.  Dropped term a_lo b_lo ~ 2^-22 relative: the result matches the FFMA
// kernel to ~1e-6 (tests/test_tc_gemm_gpu.py), at 1/3 of the TF32 rate.
//
// Structure (one CTA = one 128x128 output tile, 256 threads = two warpgroups of 64 output rows each):
//   * operands staged with cp.async (16-byte chunks) straight into the canonical K-major SWIZZLE_128B
//     layout (128-byte rows, 1 KB 8-row atoms, chunk index XOR row) - coalesced global reads and
//     conflict-free shared-memory writes; the lo tiles are derived in place by the loading threads;
//   * each warpgroup issues wgmma.m64n128k8.tf32 x 4 k-steps x 3 per 32-deep stage and leaves them in
//     flight while the next stage's lo tiles are derived (3-stage ring, prefetch distance 2);
//   * epilogue: bias/ReLU on the register accumulator -> float2 stores (four lanes = one 32-byte sector).
#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 32, STAGES = 3, THREADS = 256;
constexpr int TILE_BYTES = BM * BK * 4;                 // 16 KB per operand tile (hi or lo)
constexpr int STAGE_BYTES = 4 * TILE_BYTES;             // A_hi, A_lo, B_hi, B_lo

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
using jbwg::tile_off;

// round-to-nearest tf32 (the tensor core itself truncates): removes the one-sided bias of the lo term
__device__ __forceinline__ float tf32_rn(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ void cp16(uint32_t smem_addr, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_addr), "l"(gmem) : "memory");
}

__global__ void __launch_bounds__(THREADS, 1)
tc_linear_fwd_kernel(const float* __restrict__ X, const float* __restrict__ W, const float* __restrict__ bias,
                     float* __restrict__ Y, int M, int N, int K, int relu) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);   // swizzle atoms need 1 KB alignment

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  const int nk = K / BK;
  // stage fill: A_hi / B_hi by cp.async into the canonical layout (one commit group per k-tile)
  auto issue_load = [&](int j) {
    uint8_t* st = smem + (size_t)(j % STAGES) * STAGE_BYTES;
    const int k0 = j * BK;
#pragma unroll
    for (int r = 0; r < (BM * BK / 4) / THREADS; ++r) {
      const int e = tid + r * THREADS, row = e >> 3, c = e & 7;
      cp16(smem_u32(st + tile_off(row, c)), X + (size_t)(m0 + row) * K + k0 + c * 4);
      cp16(smem_u32(st + 2 * TILE_BYTES + tile_off(row, c)), W + (size_t)(n0 + row) * K + k0 + c * 4);
    }
    asm volatile("cp.async.commit_group;\n" ::: "memory");
  };
  issue_load(0);
  if (nk > 1) issue_load(1);
  for (int kt = 0; kt < nk; ++kt) {
    uint8_t* st = smem + (size_t)(kt % STAGES) * STAGE_BYTES;
    if (kt + 1 < nk) asm volatile("cp.async.wait_group 1;\n" ::: "memory");   // this thread's chunks of tile kt landed
    else asm volatile("cp.async.wait_group 0;\n" ::: "memory");
    // ---- lo tiles: a - trunc_tf32(a), by the thread that loaded the chunk (tile kt - 1's MMAs still run) -----
#pragma unroll
    for (int r = 0; r < (BM * BK / 4) / THREADS; ++r) {
      const int e = tid + r * THREADS, row = e >> 3, c = e & 7;
      const uint32_t off = tile_off(row, c);
#pragma unroll
      for (int op = 0; op < 2; ++op) {
        const float4 v = *reinterpret_cast<const float4*>(st + op * 2 * TILE_BYTES + off);
        float4 lo;
        lo.x = tf32_rn(v.x - __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u));
        lo.y = tf32_rn(v.y - __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u));
        lo.z = tf32_rn(v.z - __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u));
        lo.w = tf32_rn(v.w - __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u));
        *reinterpret_cast<float4*>(st + op * 2 * TILE_BYTES + TILE_BYTES + off) = lo;
      }
    }
    jbwg::wait<0>();                                                   // tile kt - 1's MMAs of this warpgroup retired
    jbwg::fence_acc(acc);
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");     // generic-proxy smem writes -> async proxy (wgmma)
    __syncthreads();
    if (kt + 2 < nk) issue_load(kt + 2);       // into tile kt - 1's stage, which no MMA reads any more
    // ---- MMA issue: this warpgroup's 64 rows, 4 k-steps of 8, three products each ----------------------
    const uint32_t a_hi = smem_u32(st) + (uint32_t)wg * (64 * 128), a_lo = a_hi + TILE_BYTES;
    const uint32_t b_hi = smem_u32(st) + 2 * TILE_BYTES, b_lo = b_hi + TILE_BYTES;
    jbwg::fence();
#pragma unroll
    for (int j = 0; j < BK / 8; ++j) {
      const uint32_t ko = (uint32_t)j * 32u;                   // K = 8 tf32 = 32 bytes along the swizzled row
      jbwg::mma_n128(acc, jbwg::desc(a_hi + ko), jbwg::desc(b_hi + ko), (kt > 0 || j > 0) ? 1 : 0);
      jbwg::mma_n128(acc, jbwg::desc(a_hi + ko), jbwg::desc(b_lo + ko), 1);
      jbwg::mma_n128(acc, jbwg::desc(a_lo + ko), jbwg::desc(b_hi + ko), 1);
    }
    jbwg::commit();
  }
  jbwg::wait<0>();
  jbwg::fence_acc(acc);
  // ---- epilogue: accumulator element (row, col) of the fragment layout in csrc/wgmma.cuh ------------------
  const int row = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (lane & 3);
    const float b0 = bias ? bias[col] : 0.f, b1 = bias ? bias[col + 1] : 0.f;
    float2 o0 = make_float2(acc[4 * j] + b0, acc[4 * j + 1] + b1);
    float2 o1 = make_float2(acc[4 * j + 2] + b0, acc[4 * j + 3] + b1);
    if (relu) { o0.x = fmaxf(o0.x, 0.f); o0.y = fmaxf(o0.y, 0.f); o1.x = fmaxf(o1.x, 0.f); o1.y = fmaxf(o1.y, 0.f); }
    *reinterpret_cast<float2*>(Y + (size_t)row * N + col) = o0;
    *reinterpret_cast<float2*>(Y + (size_t)(row + 8) * N + col) = o1;
  }
}

}  // namespace

// Requirements: M % 128 == 0, N % 128 == 0, K % 32 == 0, 16-byte aligned pointers.  Returns -22 otherwise
// (callers fall back to jb_linear_fwd).
JB_API int jb_linear_fwd_tc(const float* x, const float* w, const float* b, float* y, int M, int in_f, int out_f,
                            int relu, void* stream) {
  if (!x || !w || !y || M <= 0 || in_f <= 0 || out_f <= 0) return JB_ERR_INVALID;
  if (M % BM || out_f % BN || in_f % BK) return JB_ERR_INVALID;
  if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) return JB_ERR_INVALID;
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(tc_linear_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr = true; }
  dim3 grid(out_f / BN, M / BM);
  tc_linear_fwd_kernel<<<grid, THREADS, smem, (cudaStream_t)stream>>>(x, w, b, y, M, out_f, in_f, relu);
  return jb_check_launch();
}
