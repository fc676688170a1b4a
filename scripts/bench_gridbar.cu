// Micro-benchmark of grid-barrier variants for the persistent PPO kernel (one CTA per SM, 256 threads).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/bench_gridbar scripts/bench_gridbar.cu
// Every variant runs ITER barriers with a little global-store work between them (so the release has
// something to drain) and is checked for correctness: after each barrier every CTA reads a value
// written by its neighbour before the barrier.
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;

constexpr int NT = 256;
constexpr int ITER = 2000;

struct Bar {
  unsigned int* ctr;     // single counter
  unsigned int* flags;   // [nctas * 32] (128-byte stride)
  unsigned int* grp;     // [32 * 32]
};

template <int V>
__device__ __forceinline__ void barrier(const Bar& b, unsigned int& epoch, unsigned int nctas) {
  if (V == 5) { cg::this_grid().sync(); return; }
  __syncthreads();
  epoch += 1;
  if (V == 0) {                       // red.release + ld.acquire poll (current kernel)
    if (threadIdx.x == 0) {
      const unsigned int target = epoch * nctas;
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(b.ctr) : "memory");
      unsigned int v;
      do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(b.ctr) : "memory"); } while (v < target);
      __threadfence();
    }
  } else if (V == 1) {                // threadfence + relaxed atomic + volatile poll + threadfence
    if (threadIdx.x == 0) {
      const unsigned int target = epoch * nctas;
      __threadfence();
      atomicAdd(b.ctr, 1u);
      while (*(volatile unsigned int*)b.ctr < target) {}
      __threadfence();
    }
  } else if (V == 2) {                // red.release + relaxed poll + one acquire fence
    if (threadIdx.x == 0) {
      const unsigned int target = epoch * nctas;
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(b.ctr) : "memory");
      unsigned int v;
      do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(b.ctr) : "memory"); } while (v < target);
      asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
    }
  } else if (V == 3) {                // flag per CTA, one poller per CTA (one flag each), no atomics
    if (threadIdx.x == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;\n" ::"l"(b.flags + blockIdx.x * 32), "r"(epoch) : "memory");
    if (threadIdx.x < nctas) {
      unsigned int v;
      do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(b.flags + threadIdx.x * 32) : "memory"); } while ((int)(v - epoch) < 0);
      asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
    }
  } else if (V == 4) {                // like 3 but flags packed densely (one word per CTA), one warp-wide poll per 128-byte line
    if (threadIdx.x == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;\n" ::"l"(b.flags + blockIdx.x), "r"(epoch) : "memory");
    if (threadIdx.x < nctas) {
      unsigned int v;
      do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(b.flags + threadIdx.x) : "memory"); } while ((int)(v - epoch) < 0);
      asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
    }
  } else if (V == 6) {                // two-level: 16 groups; last arriver of a group bumps the root; pollers poll the root
    if (threadIdx.x == 0) {
      const unsigned int g = blockIdx.x & 15u;
      const unsigned int gsize = (nctas >> 4) + ((nctas & 15u) > g ? 1u : 0u);
      unsigned int old;
      asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;\n" : "=r"(old) : "l"(b.grp + g * 32) : "memory");
      if (old + 1 == epoch * gsize) asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(b.ctr) : "memory");
      unsigned int v;
      const unsigned int target = epoch * 16u;
      do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(b.ctr) : "memory"); } while (v < target);
      asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
    }
  } else if (V == 7) {                // explicit fence (all threads see it after bar) + relaxed red + relaxed poll, NO trailing fence by thread 0 only
    if (threadIdx.x == 0) {
      const unsigned int target = epoch * nctas;
      asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
      asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;\n" ::"l"(b.ctr) : "memory");
      unsigned int v;
      do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(b.ctr) : "memory"); } while (v < target);
      asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
    }
  }
  __syncthreads();
}

template <int V>
__global__ void __launch_bounds__(NT, 1) k(Bar b, float* buf, int words_per_thread, int* errors) {
  extern __shared__ float sm[];
  unsigned int epoch = 0;
  const unsigned int n = gridDim.x;
  const int nb = (blockIdx.x + 1) % n;
  int bad = 0;
  for (int it = 0; it < ITER; ++it) {
    for (int w = 0; w < words_per_thread; ++w)
      buf[((size_t)blockIdx.x * words_per_thread + w) * NT + threadIdx.x] = (float)(it + w);
    barrier<V>(b, epoch, n);
    if (words_per_thread > 0) {
      const float v = __ldcg(&buf[((size_t)nb * words_per_thread + (words_per_thread - 1)) * NT + threadIdx.x]);
      if (v != (float)(it + words_per_thread - 1)) bad++;
    }
    barrier<V>(b, epoch, n);      // WAR: neighbours finished reading before the next overwrite
  }
  if (bad) atomicAdd(errors, bad);
  if (threadIdx.x == 0) sm[0] = 0.f;
}

template <int V>
float run(Bar b, float* buf, int wpt, int* errors, int ctas, size_t smem) {
  cudaFuncSetAttribute(k<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaMemset(b.ctr, 0, 4); cudaMemset(b.flags, 0, 4 * 32 * 256); cudaMemset(b.grp, 0, 4 * 32 * 32); cudaMemset(errors, 0, 4);
  void* args[] = {&b, &buf, &wpt, &errors};
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int rep = 0; rep < 3; ++rep) {
    cudaMemset(b.ctr, 0, 4); cudaMemset(b.flags, 0, 4 * 32 * 256); cudaMemset(b.grp, 0, 4 * 32 * 32);
    cudaEventRecord(e0);
    cudaError_t e = cudaLaunchCooperativeKernel((void*)k<V>, dim3(ctas), dim3(NT), args, smem, 0);
    cudaEventRecord(e1);
    if (e != cudaSuccess || cudaEventSynchronize(e1) != cudaSuccess) { printf("variant %d failed: %s\n", V, cudaGetErrorString(cudaGetLastError())); return -1.f; }
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  int herr = 0; cudaMemcpy(&herr, errors, 4, cudaMemcpyDeviceToHost);
  printf("variant %d  words/thread %d : %.3f us per barrier   errors %d\n", V, wpt, best * 1000.f / (2 * ITER), herr);
  return best;
}

int main() {
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  Bar b; cudaMalloc(&b.ctr, 128); cudaMalloc(&b.flags, 4 * 32 * 256); cudaMalloc(&b.grp, 4 * 32 * 32);
  float* buf; cudaMalloc(&buf, sizeof(float) * (size_t)sms * 16 * NT);
  int* errors; cudaMalloc(&errors, 4);
  const size_t smem = 180 * 1024;
  for (int wpt : {0, 1, 16}) {
    run<0>(b, buf, wpt, errors, sms, smem);
    run<1>(b, buf, wpt, errors, sms, smem);
    run<2>(b, buf, wpt, errors, sms, smem);
    run<3>(b, buf, wpt, errors, sms, smem);
    run<4>(b, buf, wpt, errors, sms, smem);
    run<6>(b, buf, wpt, errors, sms, smem);
    run<7>(b, buf, wpt, errors, sms, smem);
    run<5>(b, buf, wpt, errors, sms, smem);
  }
  return 0;
}
