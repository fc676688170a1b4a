// R2D2 sequence loss (Kapturowski et al., ICLR 2019): n-step double-Q targets under the invertible value rescaling
// h(x) = sign(x)(sqrt(|x| + 1) - 1) + eps x, IS-weighted squared TD over the trained steps of each replayed sequence,
// and the paper's sequence priority eta max_t |td| + (1 - eta) mean_t |td|.
//
// One CTA per sequence b; thread tid takes the steps t = tid, tid + RT, ... in a fixed assignment, so every sum below is
// formed in the same order on every launch (per-thread ascending t, then a fixed shuffle tree, then warps in order, then
// sequences in order in the single-thread finalize): bit-reproducible, no atomics.  The target of a step is formed in
// float64 (h^-1 of a value near 0 cancels in its last step), the loss partials too; dq is rounded once to fp32.
#include "common.cuh"
#include "value_loss.cuh"

namespace {

constexpr int RT = 128;
constexpr int R2D2_MAX_A = 18;
constexpr double VR_EPS = 1e-3;

__device__ __forceinline__ double sgn(double x) { return (double)((x > 0.0) - (x < 0.0)); }
__device__ __forceinline__ double value_h(double x) { return sgn(x) * (sqrt(fabs(x) + 1.0) - 1.0) + VR_EPS * x; }
__device__ __forceinline__ double value_h_inv(double x) {
  const double s = (sqrt(1.0 + 4.0 * VR_EPS * (fabs(x) + 1.0 + VR_EPS)) - 1.0) / (2.0 * VR_EPS);
  return sgn(x) * (s * s - 1.0);
}

__global__ void __launch_bounds__(RT)
r2d2_loss_kernel(const float* __restrict__ q, const float* __restrict__ q_next, const float* __restrict__ qt_next,
                 const int64_t* __restrict__ action, const float* __restrict__ reward, const float* __restrict__ done,
                 const double* __restrict__ weights, int B, int T, int A, int n, float gamma, float alpha, float eta,
                 float* __restrict__ dq, double* __restrict__ prio, double* __restrict__ partial /*[B][2]*/) {
  __shared__ double s_sq[RT / 32], s_abs[RT / 32], s_mabs[RT / 32];
  __shared__ float s_mq[RT / 32];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const double w = weights ? weights[b] : 1.0;
  const double gscale = -2.0 * w / ((double)B * (double)T);
  const float* rr = reward + (size_t)b * (T + n);
  const float* dr = done + (size_t)b * (T + n);
  double sq = 0.0, sabs = 0.0, mabs = 0.0;
  float mq = -INFINITY;
  for (int t = tid; t < T; t += RT) {
    const size_t row = ((size_t)b * T + t) * A;
    double y = value_h_inv((double)qt_next[row + first_argmax(q_next + row, A)]);
    for (int i = n - 1; i >= 0; --i) y = (double)rr[t + i] + (1.0 - (double)dr[t + i]) * (double)gamma * y;
    y = value_h(y);
    const int a_t = (int)action[(size_t)b * T + t];
    const float qa = q[row + a_t];
    const double td = y - (double)qa;
    for (int a = 0; a < A; ++a) dq[row + a] = a == a_t ? (float)(gscale * td) : 0.f;
    sq += w * td * td;
    sabs += fabs(td);
    mabs = fmax(mabs, fabs(td));
    mq = fmaxf(mq, qa);
  }
  for (int o = 16; o > 0; o >>= 1) {
    sq += __shfl_xor_sync(0xffffffffu, sq, o);
    sabs += __shfl_xor_sync(0xffffffffu, sabs, o);
    mabs = fmax(mabs, __shfl_xor_sync(0xffffffffu, mabs, o));
    mq = fmaxf(mq, __shfl_xor_sync(0xffffffffu, mq, o));
  }
  if (lane == 0) { s_sq[warp] = sq; s_abs[warp] = sabs; s_mabs[warp] = mabs; s_mq[warp] = mq; }
  __syncthreads();
  if (tid == 0) {
    for (int k = 1; k < RT / 32; ++k) {
      sq += s_sq[k]; sabs += s_abs[k]; mabs = fmax(mabs, s_mabs[k]); mq = fmaxf(mq, s_mq[k]);
    }
    if (prio) prio[b] = pow((double)eta * mabs + (1.0 - (double)eta) * (sabs / (double)T), (double)alpha);
    partial[2 * b] = sq;
    partial[2 * b + 1] = (double)mq;
  }
}

__global__ void r2d2_finalize_kernel(const double* __restrict__ partial, int B, int T, float* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  double l = 0.0;
  float mq = -INFINITY;
  for (int b = 0; b < B; ++b) { l += partial[2 * b]; mq = fmaxf(mq, (float)partial[2 * b + 1]); }
  stats[0] = (float)(l / ((double)B * (double)T));
  stats[1] = mq;
}

}  // namespace

JB_API int jb_r2d2_loss(const float* q, const float* q_next, const float* qt_next, const int64_t* action, const float* reward,
                        const float* done, const double* weights, int B, int T, int A, int n_step, float gamma, float alpha,
                        float eta, float* dq, double* prio, float* stats, double* scratch, void* stream) {
  if (!q || !q_next || !qt_next || !action || !reward || !done || !dq || !stats || !scratch) return JB_ERR_INVALID;
  if (B <= 0 || T <= 0 || A <= 0 || A > R2D2_MAX_A || n_step < 1) return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  r2d2_loss_kernel<<<B, RT, 0, s>>>(q, q_next, qt_next, action, reward, done, weights, B, T, A, n_step, gamma, alpha, eta, dq,
                                    prio, scratch);
  r2d2_finalize_kernel<<<1, 32, 0, s>>>(scratch, B, T, stats);
  return jb_check_launch();
}
