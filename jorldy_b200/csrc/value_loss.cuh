// Pieces shared by the value-based loss kernels (dqn.cu, c51.cu, quantile.cu, r2d2.cu): the replayed action read, the
// f32 n-step target fold, the first-index argmax and the single-thread batch-statistics finalizes.  Everything here has
// internal linkage, so each of those objects keeps its own copy and the kernels compile as they did inline.  The finalize
// kernels are templates on the partials' type so that only the objects that launch them carry them.
#pragma once
#include "common.cuh"

namespace {

// action_kind: 0 int64, 1 int32, 2 float32 (the replay stores whatever dtype the env produced)
__device__ __forceinline__ int read_action(const void* act, int kind, int b) {
  if (kind == 0) return (int)((const int64_t*)act)[b];
  if (kind == 1) return ((const int32_t*)act)[b];
  return (int)((const float*)act)[b];
}

// y <- r_s + ((1 - d_s) gamma) y for s = n-1 .. 0, rounded step by step in this order (multistep.py / rainbow.py)
__device__ __forceinline__ float nstep_fold(float y, const float* rr, const float* dr, int n, float gamma) {
  for (int s = n - 1; s >= 0; --s) y = __fadd_rn(rr[s], __fmul_rn(__fmul_rn(__fadd_rn(1.f, -dr[s]), gamma), y));
  return y;
}

// index of the first maximum of x[0 .. n), like torch.argmax
__device__ __forceinline__ int first_argmax(const float* x, int n) {
  int am = 0;
  float best = x[0];
  for (int i = 1; i < n; ++i)
    if (x[i] > best) { best = x[i]; am = i; }
  return am;
}

// partial[b] = {loss_b, max_Q_b} for b < B -> stats = {sum_b loss_b / B, max_b max_Q_b}, summed in order
template <typename T>
__global__ void loss_maxq_finalize_kernel(const T* __restrict__ partial, int B, float* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  float l = 0.f, mq = -INFINITY;
  for (int b = 0; b < B; ++b) { l += partial[2 * b]; mq = fmaxf(mq, partial[2 * b + 1]); }
  stats[0] = l / (float)B;   // loss
  stats[1] = mq;             // max_Q
}

// partial[k] = {loss, max_Q, max_logit, min_logit} for k < n (one per CTA or per sample) -> stats, the loss sum over B
template <typename T>
__global__ void loss_logits_finalize_kernel(const T* __restrict__ partial, int n, int B, float* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  float l = 0.f, mq = -INFINITY, ml = -INFINITY, nl = INFINITY;
  for (int k = 0; k < n; ++k) {
    l += partial[4 * k]; mq = fmaxf(mq, partial[4 * k + 1]); ml = fmaxf(ml, partial[4 * k + 2]); nl = fminf(nl, partial[4 * k + 3]);
  }
  stats[0] = l / (float)B; stats[1] = mq; stats[2] = ml; stats[3] = nl;
}

}  // namespace
