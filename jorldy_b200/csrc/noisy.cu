// NoisyNet (factorised Gaussian) layer support: noise draw + effective weights, and the
// gradient split back onto (mu, sigma).
//
// Reference: jorldy/core/network/utils.py:55-86 `noisy_l`
//   eps_i ~ N(0,1)^in, eps_j ~ N(0,1)^out;  f(e) = sign(e) sqrt|e|
//   eps_w = f(eps_i) f(eps_j)^T  (in x out),  eps_b = f(eps_j)
//   W = mu_w + sig_w * eps_w ;  b = mu_b + sig_b * eps_b ;  y = x @ W + b      (weight layout [in,out])
// Fresh noise on EVERY forward (Rainbow: 3 forwards x 4 noisy layers per learn, rainbow.py:167-182).
// The reference spends 31 % of a Rainbow learn() here (randn + outer product + 3 elementwise passes
// per layer); here one launch writes W/b (8 B/weight read, 4 B written) and the product itself is the
// shared jb_linear_io_* kernel.  Backward: dmu = dW, dsig = dW * eps_w (same for the bias).
#include "common.cuh"
#include "philox.cuh"

namespace {

// Philox counter of a drawn factor t (t < in_f: f_i[t], else f_j[t - in_f]) = draw * DRAW_STRIDE + t / 2: one Philox
// block gives two normals, so one draw owns 2 * DRAW_STRIDE normals.  A layer with in_f + out_f > 2 * DRAW_STRIDE would
// run into the next draw's counters and successive draws would share normals, so jb_noisy_make rejects it when it
// draws (injected normals have no such limit).  Widening the stride would change every existing stream.
constexpr uint64_t DRAW_STRIDE = 4096;
constexpr int MAX_DRAWN_FACTORS = 2 * (int)DRAW_STRIDE;

__device__ __forceinline__ float f_noise(float e) { return (e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f)) * sqrtf(fabsf(e)); }

// f_i[in], f_j[out] from injected normals or Philox Box-Muller (stream = layer id, ctr = draw index)
__global__ void noisy_factors_kernel(const float* __restrict__ eps_i, const float* __restrict__ eps_j, int in_f, int out_f,
                                     uint64_t seed, uint64_t stream, long long* __restrict__ ctr_ptr,
                                     float* __restrict__ f_i, float* __restrict__ f_j) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = in_f + out_f;
  if (t >= n) return;
  float e;
  const float* inj = (t < in_f) ? eps_i : eps_j;
  if (inj) e = (t < in_f) ? eps_i[t] : eps_j[t - in_f];
  else {
    const uint64_t c = ctr_ptr ? (uint64_t)(*ctr_ptr) : 0;
    float n0, n1;
    jb_normal_pair(seed, stream, c * DRAW_STRIDE + (uint64_t)(t >> 1), n0, n1);
    e = (t & 1) ? n1 : n0;
  }
  const float f = f_noise(e);
  if (t < in_f) f_i[t] = f; else f_j[t - in_f] = f;
}

__global__ void noisy_bump_kernel(long long* ctr) { if (threadIdx.x == 0 && blockIdx.x == 0) *ctr += 1; }

__global__ void noisy_weights_kernel(const float* __restrict__ mu_w, const float* __restrict__ sig_w,
                                     const float* __restrict__ mu_b, const float* __restrict__ sig_b,
                                     const float* __restrict__ f_i, const float* __restrict__ f_j, int in_f, int out_f,
                                     float* __restrict__ w_eff, float* __restrict__ b_eff) {
  const long long total = (long long)in_f * out_f;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / out_f), j = (int)(e % out_f);
    // mu + sig * (f_i * f_j): the product eps_w is formed first (torch.matmul outer product), then sig*eps, then +mu
    w_eff[e] = __fadd_rn(mu_w[e], __fmul_rn(sig_w[e], __fmul_rn(f_i[i], f_j[j])));
  }
  if (blockIdx.x == 0)
    for (int j = threadIdx.x; j < out_f; j += blockDim.x) b_eff[j] = __fadd_rn(mu_b[j], __fmul_rn(sig_b[j], f_j[j]));
}

__global__ void noisy_grad_kernel(const float* __restrict__ dw_eff, const float* __restrict__ db_eff,
                                  const float* __restrict__ f_i, const float* __restrict__ f_j, int in_f, int out_f,
                                  float* __restrict__ dmu_w, float* __restrict__ dsig_w, float* __restrict__ dmu_b,
                                  float* __restrict__ dsig_b) {
  const long long total = (long long)in_f * out_f;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / out_f), j = (int)(e % out_f);
    const float g = dw_eff[e];
    dmu_w[e] = g;
    dsig_w[e] = g * (f_i[i] * f_j[j]);
  }
  if (blockIdx.x == 0)
    for (int j = threadIdx.x; j < out_f; j += blockDim.x) { const float g = db_eff[j]; dmu_b[j] = g; dsig_b[j] = g * f_j[j]; }
}

}  // namespace

// Draws the factor vectors (eps_i/eps_j injected normals, or Philox with stream id + device draw
// counter) and materialises W [in,out], b [out].  is_train = 0 -> W = mu_w, b = mu_b (utils.py:69-71).
// Drawing (either eps pointer NULL) needs in_f + out_f <= 8192 (see DRAW_STRIDE) and bumps *draw_ctr once.
JB_API int jb_noisy_make(const float* mu_w, const float* sig_w, const float* mu_b, const float* sig_b, int in_f,
                         int out_f, const float* eps_i, const float* eps_j, uint64_t seed, uint64_t stream_id,
                         long long* draw_ctr, int is_train, float* f_i, float* f_j, float* w_eff, float* b_eff,
                         void* stream) {
  if (!mu_w || !sig_w || !mu_b || !sig_b || !f_i || !f_j || !w_eff || !b_eff || in_f <= 0 || out_f <= 0)
    return JB_ERR_INVALID;
  const bool draws = is_train && !(eps_i && eps_j);
  if (draws && (long long)in_f + out_f > MAX_DRAWN_FACTORS) return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  if (is_train) {
    noisy_factors_kernel<<<jb_div_up(in_f + out_f, 128), 128, 0, s>>>(eps_i, eps_j, in_f, out_f, seed, stream_id, draw_ctr, f_i, f_j);
    if (draw_ctr && draws) noisy_bump_kernel<<<1, 32, 0, s>>>(draw_ctr);
  } else {
    cudaMemsetAsync(f_i, 0, sizeof(float) * in_f, s);
    cudaMemsetAsync(f_j, 0, sizeof(float) * out_f, s);
  }
  noisy_weights_kernel<<<jb_grid_for((long long)in_f * out_f, 256 * 4, 4), 256, 0, s>>>(mu_w, sig_w, mu_b, sig_b, f_i, f_j, in_f, out_f, w_eff, b_eff);
  return jb_check_launch();
}

JB_API int jb_noisy_grad(const float* dw_eff, const float* db_eff, const float* f_i, const float* f_j, int in_f,
                         int out_f, float* dmu_w, float* dsig_w, float* dmu_b, float* dsig_b, void* stream) {
  if (!dw_eff || !db_eff || !f_i || !f_j || !dmu_w || !dsig_w || !dmu_b || !dsig_b || in_f <= 0 || out_f <= 0)
    return JB_ERR_INVALID;
  noisy_grad_kernel<<<jb_grid_for((long long)in_f * out_f, 256 * 4, 4), 256, 0, (cudaStream_t)stream>>>(
      dw_eff, db_eff, f_i, f_j, in_f, out_f, dmu_w, dsig_w, dmu_b, dsig_b);
  return jb_check_launch();
}
