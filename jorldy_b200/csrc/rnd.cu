// RND-PPO (Burda et al., 2018, arXiv:1810.12894, "Exploration by Random Network Distillation") on the PPO rollout path:
// the distillation loss and the two-stream advantage mix.  The two-critic PPO loss and the pre-pass of the two-value
// policy network are ppo.cu's kernels instantiated for two value columns (jb_rnd_ppo_loss, jb_rnd_prepass).  The RND
// networks' dense layers are the existing GEMMs (csrc/linear.cu), their BatchNorm + ELU and the running statistics are
// csrc/icm.cu's, and each stream's advantages are jb_gae's.
//
// No atomics anywhere; every reduction runs in a fixed order, so each entry point is bit-reproducible run to run.
#include "common.cuh"

namespace {

constexpr int RND_F = 256;        // RND feature width (8 floats per lane)
constexpr int RND_ROWS = 8;       // rows (warps) per distillation-loss CTA
constexpr int MIX_ROWS = 8;       // rows (warps) per advantage-mix CTA

// ---- distillation loss ----------------------------------------------------------------------------------------------
// One warp per row: lane l holds feature columns l + 32 j.  r_i[b] = mean_F (p - t)^2; dp = 2 (p - t) / (B F).
__global__ void __launch_bounds__(32 * RND_ROWS)
rnd_loss_kernel(const float* __restrict__ p, const float* __restrict__ target, const int32_t* __restrict__ idx, int B,
                float* __restrict__ ri, float* __restrict__ dp, float* __restrict__ stats) {
  __shared__ float sp[RND_ROWS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * RND_ROWS + warp;
  float rb = 0.f;
  if (b < B) {
    const int r = idx ? idx[b] : b;
    const float* pr = p + (size_t)b * RND_F;
    const float* tr = target + (size_t)r * RND_F;
    const float cf = 2.f / ((float)B * (float)RND_F);
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < RND_F / 32; ++j) {
      const int c = lane + 32 * j;
      const float d = pr[c] - tr[c];
      sq += d * d;
      if (dp) dp[(size_t)b * RND_F + c] = cf * d;
    }
    rb = jb_warp_sum(sq) / (float)RND_F;
    if (ri && lane == 0) ri[b] = rb;
  }
  if (!stats) return;
  if (lane == 0) sp[warp] = rb;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < RND_ROWS; ++w) t += sp[w];
    stats[1 + blockIdx.x] = t;
  }
}

// stats[0] = rnd_loss = mean_B r_i (per-CTA partials folded in CTA order); acc[0] += stats[0], acc[1] += 1
__global__ void rnd_loss_finalize_kernel(float* __restrict__ stats, int n_cta, int B, float* __restrict__ acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float s = 0.f;
  for (int k = 0; k < n_cta; ++k) s += stats[1 + k];
  stats[0] = s / (float)B;
  if (acc) { acc[0] += stats[0]; acc[1] += 1.f; }
}

// ---- advantage mix ----------------------------------------------------------------------------------------------------
// One warp per row of T steps.  adv = ext_coef adv_e + int_coef adv_i; with `standardize` each row becomes
// (adv - mean) / (std + 1e-7) with gae.cu's arithmetic: the float64 sums run over t = T-1 .. 0 in that order (lane k's
// value is broadcast in turn), the unbiased variance and the one rounding to float are the same expressions.
__global__ void __launch_bounds__(32 * MIX_ROWS)
adv_mix_kernel(const float* __restrict__ adv_e, const float* __restrict__ adv_i, int N, int T, float ext_coef,
               float int_coef, int standardize, float* __restrict__ adv) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = blockIdx.x * MIX_ROWS + warp;
  if (row >= N) return;
  const size_t base = (size_t)row * T;
  double sm = 0.0, sq = 0.0;
  for (int t0 = ((T - 1) / 32) * 32; t0 >= 0; t0 -= 32) {
    const int t = t0 + lane;
    float a = 0.f;
    if (t < T) {
      a = __fadd_rn(__fmul_rn(ext_coef, adv_e[base + t]), __fmul_rn(int_coef, adv_i[base + t]));
      adv[base + t] = a;
    }
    if (standardize) {
      for (int k = 31; k >= 0; --k) {
        const float x = __shfl_sync(0xffffffffu, a, k);
        if (t0 + k < T) { sm += (double)x; sq += (double)x * (double)x; }
      }
    }
  }
  if (!standardize) return;
  const double mean_d = sm / (double)T;
  double var_d = (sq - sm * mean_d) / (double)(T > 1 ? T - 1 : 1);
  if (var_d < 0) var_d = 0;
  const float mean = (float)mean_d;
  const float denom = __fadd_rn((float)sqrt(var_d), 1e-7f);
  for (int t = lane; t < T; t += 32) adv[base + t] = __fdiv_rn(__fadd_rn(adv[base + t], -mean), denom);
}

}  // namespace

JB_API int jb_rnd_loss(const float* p, const float* target, const int32_t* idx, int B, int F, float* ri, float* dp,
                       float* stats, float* acc, void* stream) {
  if (!p || !target || B <= 0 || F != RND_F) return JB_ERR_INVALID;
  if (dp ? !stats : !ri) return JB_ERR_INVALID;         // the minibatch step needs stats; the reward-only pass needs ri
  if (!dp) stats = nullptr;
  const int n_cta = jb_div_up(B, RND_ROWS);
  cudaStream_t s = (cudaStream_t)stream;
  rnd_loss_kernel<<<n_cta, 32 * RND_ROWS, 0, s>>>(p, target, idx, B, ri, dp, stats);
  if (stats) rnd_loss_finalize_kernel<<<1, 32, 0, s>>>(stats, n_cta, B, acc);
  return jb_check_launch();
}

JB_API int jb_adv_mix(const float* adv_e, const float* adv_i, int N, int T, float ext_coef, float int_coef,
                      int standardize, float* adv, void* stream) {
  if (!adv_e || !adv_i || !adv || N <= 0 || T <= 0) return JB_ERR_INVALID;
  adv_mix_kernel<<<jb_div_up(N, MIX_ROWS), 32 * MIX_ROWS, 0, (cudaStream_t)stream>>>(adv_e, adv_i, N, T, ext_coef,
                                                                                     int_coef, standardize, adv);
  return jb_check_launch();
}
