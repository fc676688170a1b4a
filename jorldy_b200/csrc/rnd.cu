// RND-PPO (Burda et al., 2018, arXiv:1810.12894, "Exploration by Random Network Distillation") on the PPO rollout path:
// the two-critic PPO loss, the pre-pass of a two-value policy network, the distillation loss and the two-stream
// advantage mix.  The RND networks' dense layers are the existing GEMMs (csrc/linear.cu), their BatchNorm + ELU and the
// running statistics are csrc/icm.cu's, and each stream's advantages are jb_gae's.
//
// Head output layout of the two-value policy network `out[M, nout]` (pre-activation, jb_heads_fwd_n):
//   discrete  : [logits(A) | v | v_i]                  nout = A + 2
//   continuous: [mu_raw(A) | log_std_raw(A) | v | v_i] nout = 2A + 2
// so every column PPO's row maths (ppo_rowmath.cuh) reads stays where it is.
//
// No atomics anywhere; every reduction runs in a fixed order, so each entry point is bit-reproducible run to run.
#include "common.cuh"
#include "ppo_rowmath.cuh"

namespace {

using jbppo::MAX_A;
using jbppo::MAX_A_DISC;

constexpr int RND_F = 256;        // RND feature width (8 floats per lane)
constexpr int RND_ROWS = 8;       // rows (warps) per distillation-loss CTA
constexpr int MIX_ROWS = 8;       // rows (warps) per advantage-mix CTA

// ---- pre-pass: value, intrinsic value, log_prob_old ---------------------------------------------------------------
template <bool CONT, int NA>
__global__ void rnd_prepass_kernel(const float* __restrict__ out, const void* __restrict__ action, int M, int A, int nout,
                                   float* __restrict__ value, float* __restrict__ value_i, float* __restrict__ logp_old) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float* o = out + (size_t)m * nout;
  const int npol = CONT ? 2 * A : A;
  if constexpr (CONT)
    jbppo::logp_continuous(o, A, (const float*)action + (size_t)m * A, logp_old + (size_t)m * A);
  else
    logp_old[m] = jbppo::logp_discrete<NA>(o, A, ((const int32_t*)action)[m]);
  value[m] = o[npol];
  value_i[m] = o[npol + 1];
}

// ---- two-critic PPO loss ------------------------------------------------------------------------------------------
// ppo.cu's ppo_loss_kernel with a second clipped critic on column npol + 1: pass 1 reduces all four critic means in one
// fixed-order block sum, pass 2 runs PPO's row maths (actor, entropy, extrinsic critic) and adds the intrinsic critic's
// gradient.  With ret_i = v_i = v_old_i every value this kernel writes equals ppo_loss_kernel's bit for bit.  Min-blocks 1
// for every instantiation: at ptxas's default the 8-wide discrete row spills 4 bytes.
template <bool CONT, int NA>
__global__ void __launch_bounds__(256, 1)
rnd_ppo_loss_kernel(const float* __restrict__ out, const int32_t* __restrict__ idx, const void* __restrict__ action_all,
                    const float* __restrict__ adv_all, const float* __restrict__ ret_all,
                    const float* __restrict__ vold_all, const float* __restrict__ ret_i_all,
                    const float* __restrict__ vold_i_all, const float* __restrict__ logp_old_all, int B, int A, int nout,
                    jbppo::HP hp, float* __restrict__ dout, float* __restrict__ stats /*[8 + 4*n_cta]*/) {
  __shared__ float sred[4 * 32];
  const float invB = 1.0f / (float)B;
  const int npol = CONT ? 2 * A : A;
  // ---- pass 1 (every CTA, whole minibatch, fixed order): the four critic means ---------------------------------------
  float c[4] = {0.f, 0.f, 0.f, 0.f};
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int r = idx ? idx[b] : b;
    const float v = out[(size_t)b * nout + npol];
    const float ret = ret_all[r], vold = vold_all[r];
    const float vclip = vold + fminf(fmaxf(v - vold, -hp.eps_clip), hp.eps_clip);
    const float d1 = v - ret, d2 = vclip - ret;
    c[0] += d1 * d1; c[1] += d2 * d2;
    const float vi = out[(size_t)b * nout + npol + 1];
    const float reti = ret_i_all[r], voldi = vold_i_all[r];
    const float viclip = voldi + fminf(fmaxf(vi - voldi, -hp.eps_clip), hp.eps_clip);
    const float e1 = vi - reti, e2 = viclip - reti;
    c[2] += e1 * e1; c[3] += e2 * e2;
  }
  jbppo::block_sum<4>(c, sred);
  const float c1 = c[0] * invB, c2 = c[1] * invB, c3 = c[2] * invB, c4 = c[3] * invB;
  float w1, w2, u1, u2;
  jbppo::critic_weights(c1, c2, w1, w2);
  jbppo::critic_weights(c3, c4, u1, u2);

  // ---- pass 2: this CTA's rows -------------------------------------------------------------------------------------
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float st[2] = {0.f, 0.f};
  float max_ratio = -INFINITY, min_prob = INFINITY;
  if (b < B) {
    const int r = idx ? idx[b] : b;
    jbppo::RowOutW<jbppo::width<NA>()> ro;
    const float* o = out + (size_t)b * nout;
    if constexpr (CONT) jbppo::row<true, NA>(o, A, 0, (const float*)action_all + (size_t)r * A, adv_all[r], ret_all[r],
                                             vold_all[r], logp_old_all + (size_t)r * A, hp, invB, ro);
    else jbppo::row<false, NA>(o, A, ((const int32_t*)action_all)[r], nullptr, adv_all[r], ret_all[r], vold_all[r],
                               logp_old_all + r, hp, invB, ro);
    float* g = dout + (size_t)b * nout;
#pragma unroll
    for (int a = 0; a < (CONT ? 2 * NA : NA); ++a) if (a < npol) g[a] = ro.dpol[a];
    g[npol] = w1 * ro.dv1 + w2 * ro.dv2;
    // intrinsic critic: the same clipped pair around v_old_i
    const float vi = o[npol + 1], voldi = vold_i_all[r], reti = ret_i_all[r];
    const float dvi = vi - voldi;
    const float viclip = voldi + fminf(fmaxf(dvi, -hp.eps_clip), hp.eps_clip);
    const float in_clip = (dvi >= -hp.eps_clip && dvi <= hp.eps_clip) ? 1.f : 0.f;
    const float e1 = vi - reti, e2 = viclip - reti;
    g[npol + 1] = u1 * (hp.vf_coef * invB * 2.f * e1) + u2 * (hp.vf_coef * invB * 2.f * e2 * in_clip);
    st[0] = ro.surr_min; st[1] = ro.ent;
    max_ratio = ro.ratio; min_prob = ro.pmin;
  }
  jbppo::block_sum<2>(st, sred);
  float mr = jb_warp_max(max_ratio), mp = jb_warp_min(min_prob);
  __shared__ float smax[32], smin_[32];
  if ((threadIdx.x & 31) == 0) { smax[threadIdx.x >> 5] = mr; smin_[threadIdx.x >> 5] = mp; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    for (int w = 1; w < nw; ++w) { mr = fmaxf(mr, smax[w]); mp = fminf(mp, smin_[w]); }
    float* sp = stats + 8 + 4 * blockIdx.x;
    sp[0] = st[0]; sp[1] = st[1]; sp[2] = mr; sp[3] = mp;
    if (blockIdx.x == 0) {
      const float ce = fmaxf(c1, c2), ci = fmaxf(c3, c4);
      stats[1] = ce + ci; stats[5] = ce; stats[6] = ci; stats[7] = 0.f;
    }
  }
}

__global__ void rnd_ppo_finalize_kernel(float* __restrict__ stats, int n_cta, int B, int A, int cont,
                                        float* __restrict__ acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  jbppo::fold_stats(stats, n_cta, B, A, cont, acc);
}

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

JB_API int jb_rnd_prepass(int continuous, const float* out, const void* action, int M, int A, int nout, float* value,
                          float* value_i, float* logp_old, void* stream) {
  if (!out || !action || !value || !value_i || !logp_old || M <= 0 || A <= 0) return JB_ERR_INVALID;
  if (A > (continuous ? MAX_A : MAX_A_DISC) || nout != (continuous ? 2 * A + 2 : A + 2)) return JB_ERR_INVALID;
  const dim3 grid(jb_div_up(M, 128));
  cudaStream_t s = (cudaStream_t)stream;
  if (continuous) rnd_prepass_kernel<true, MAX_A><<<grid, 128, 0, s>>>(out, action, M, A, nout, value, value_i, logp_old);
  else if (A <= MAX_A) rnd_prepass_kernel<false, MAX_A><<<grid, 128, 0, s>>>(out, action, M, A, nout, value, value_i, logp_old);
  else rnd_prepass_kernel<false, MAX_A_DISC><<<grid, 128, 0, s>>>(out, action, M, A, nout, value, value_i, logp_old);
  return jb_check_launch();
}

JB_API int jb_rnd_ppo_loss(int continuous, const float* out, const int32_t* idx, const void* action, const float* adv,
                           const float* ret, const float* value_old, const float* ret_i, const float* value_i_old,
                           const float* logp_old, int B, int A, int nout, float eps_clip, float vf_coef, float ent_coef,
                           float* dout, float* stats, float* acc, void* stream) {
  if (!out || !action || !adv || !ret || !value_old || !ret_i || !value_i_old || !logp_old || !dout || !stats)
    return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || A > (continuous ? MAX_A : MAX_A_DISC) || nout != (continuous ? 2 * A + 2 : A + 2))
    return JB_ERR_INVALID;
  jbppo::HP hp{eps_clip, vf_coef, ent_coef};
  const int n_cta = jb_div_up(B, 256);
  cudaStream_t s = (cudaStream_t)stream;
  if (continuous)
    rnd_ppo_loss_kernel<true, MAX_A><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, ret_i, value_i_old,
                                                           logp_old, B, A, nout, hp, dout, stats);
  else if (A <= MAX_A)
    rnd_ppo_loss_kernel<false, MAX_A><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, ret_i, value_i_old,
                                                            logp_old, B, A, nout, hp, dout, stats);
  else
    rnd_ppo_loss_kernel<false, MAX_A_DISC><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, ret_i,
                                                                 value_i_old, logp_old, B, A, nout, hp, dout, stats);
  rnd_ppo_finalize_kernel<<<1, 32, 0, s>>>(stats, n_cta, B, A, continuous, acc);
  return jb_check_launch();
}

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
