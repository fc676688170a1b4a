// PPO-specific row kernels: action sampling, old log-prob, and the fused clipped-surrogate /
// clipped-value / entropy loss forward + backward on the narrow head outputs.
//
// Reference: jorldy/core/agent/ppo.py
//   :54-69   act            -> jb_ppo_act_discrete / jb_ppo_act_continuous
//   :83-93   no-grad pass   -> jb_ppo_prepass_discrete / _continuous (value, log_prob_old)
//   :127-162 loss           -> jb_ppo_loss (loss terms + d loss / d head outputs)
// and the distribution maths of torch.distributions.Categorical / Normal (third-party torch,
// requirements.txt:10) restated from their definitions:
//   Categorical(probs=p): p <- p / sum(p); logits = log(clamp(p, eps, 1-eps)); log_prob = logits[a];
//                         entropy = -sum(logits * p)
//   Normal(mu, sd).log_prob(z) = -(z-mu)^2/(2 sd^2) - log(sd) - log(sqrt(2 pi));
//                         entropy = 0.5 + 0.5 log(2 pi) + log(sd)
//
// Head output layout `out[M, NOUT]` (pre-activation, produced by jb_heads_fwd):
//   discrete  : [logits(A) | v]                 policy_value.py:19-22
//   continuous: [mu_raw(A) | log_std_raw(A) | v] policy_value.py:51-57 (mu=clamp(.,-5,5), sd=exp(tanh(.)))
//
// The two scalar means inside `critic_loss = max(mse(v,ret), mse(v_clip,ret))` (ppo.py:148-154)
// are needed before any per-row gradient exists; every CTA therefore first reduces them over the
// whole minibatch in a fixed order (B*3 floats from L2 — cheaper than a second launch) and then
// produces its rows' gradients.  All reductions are fixed-order => bit-reproducible run to run.
//
// The pre-pass and loss kernels also serve RND-PPO's two-value policy network (jb_rnd_prepass, jb_rnd_ppo_loss), as
// instantiations for two value columns.
#include "common.cuh"
#include "philox.cuh"
#include "ppo_rowmath.cuh"

namespace {

using jbppo::MAX_A;
using jbppo::MAX_A_DISC;
using jbppo::log_softmax_row;
using jbppo::atanh_clamped;

// ---- act ------------------------------------------------------------------------------------
// NA: compile-time bound on A (MAX_A or MAX_A_DISC); every loop runs to NA with an `a < A` guard so lg/lsm stay in registers
template <int NA>
__global__ void ppo_act_discrete_kernel(const float* __restrict__ out, int M, int A, int nout,
                                        const float* __restrict__ u_in, uint64_t seed, uint64_t stream_base,
                                        uint64_t ctr, long long* __restrict__ row_ctr, int greedy,
                                        int64_t* __restrict__ action) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  ctr = jb_next_row_ctr(row_ctr, m, ctr);
  float lg[NA], lsm[NA];
#pragma unroll
  for (int a = 0; a < NA; ++a) lg[a] = a < A ? out[(size_t)m * nout + a] : 0.f;
  log_softmax_row<NA>(lg, A, lsm);
  int pick = 0;
  if (greedy) {
    float best = expf(lsm[0]);
#pragma unroll
    for (int a = 1; a < NA; ++a) if (a < A) { const float p = expf(lsm[a]); if (p > best) { best = p; pick = a; } }
  } else {
    float u;
    if (u_in) u = u_in[m];
    else { jb_philox4 r = jb_philox(seed, stream_base + (uint64_t)m, ctr); u = jb_u01_float(r.x); }
    // inverse CDF on pi = exp(log_softmax) (same law as torch.multinomial(pi, 1), ppo.py:64-68)
    float tot = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) if (a < A) tot += expf(lsm[a]);
    const float target = u * tot;
    float c = 0.f;
    bool found = false;
    pick = A - 1;
#pragma unroll
    for (int a = 0; a < NA; ++a) if (a < A && !found) { c += expf(lsm[a]); if (target < c) { pick = a; found = true; } }
  }
  action[m] = pick;
}

__global__ void ppo_act_continuous_kernel(const float* __restrict__ out, int M, int A, int nout,
                                          const float* __restrict__ n_in, uint64_t seed, uint64_t stream_base,
                                          uint64_t ctr, long long* __restrict__ row_ctr, int greedy,
                                          float* __restrict__ action) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  ctr = jb_next_row_ctr(row_ctr, m, ctr);
  for (int a = 0; a < A; a += 2) {
    float n0 = 0.f, n1 = 0.f;
    if (!greedy) {
      if (n_in) { n0 = n_in[(size_t)m * A + a]; if (a + 1 < A) n1 = n_in[(size_t)m * A + a + 1]; }
      else jb_normal_pair(seed, stream_base + (uint64_t)m, ctr * 8 + (uint64_t)(a >> 1), n0, n1);
    }
    for (int q = 0; q < 2 && a + q < A; ++q) {
      const float mu = fminf(fmaxf(out[(size_t)m * nout + a + q], -5.f), 5.f);
      const float sd = expf(tanhf(out[(size_t)m * nout + A + a + q]));
      const float z = greedy ? mu : fmaf(sd, q ? n1 : n0, mu);      // torch.normal(mu, std)
      action[(size_t)m * A + a + q] = tanhf(z);
    }
  }
}

// ---- pre-pass: value (and the intrinsic value) + log_prob_old -----------------------------------
// NV: value columns after the policy columns, 1 (PPO) or 2 (RND-PPO's [v | v_i]).  value_i is read only when NV == 2;
// it comes last so the one-critic instantiations keep PPO's parameter layout.
template <bool CONT, int NA, int NV>
__global__ void ppo_prepass_kernel(const float* __restrict__ out, const void* __restrict__ action, int M, int A, int nout,
                                   float* __restrict__ value, float* __restrict__ logp_old /*[M] or [M,A]*/,
                                   float* __restrict__ value_i) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float* o = out + (size_t)m * nout;
  const int npol = CONT ? 2 * A : A;
  if constexpr (CONT)
    jbppo::logp_continuous(o, A, (const float*)action + (size_t)m * A, logp_old + (size_t)m * A);
  else
    logp_old[m] = jbppo::logp_discrete<NA>(o, A, ((const int32_t*)action)[m]);
  value[m] = o[npol];
  if constexpr (NV == 2) value_i[m] = o[npol + 1];
}

// ---- loss -------------------------------------------------------------------------------------
// NA: compile-time bound on A, see jbppo::row.  NV: value columns, 1 (PPO) or 2 (RND-PPO: a second clipped critic on
// column npol + 1 learning ret_i around v_old_i, whose means join pass 1's block sum and whose gradient pass 2 adds; the
// actor, entropy and extrinsic-critic terms are the one-critic kernel's).  ret_i_all / vold_i_all are read only when
// NV == 2; they come last so the one-critic instantiations keep PPO's parameter layout.
// The 18-wide row holds ~145 live registers: min-blocks 1 lets ptxas use them instead of spilling at its default 128 (0
// leaves the 8-wide one-critic instantiations unconstrained, as before).  Two critics: min-blocks 1 for every
// instantiation, since at ptxas's default the 8-wide discrete row spills 4 bytes.
template <bool CONT, int NA, int NV>
__global__ void __launch_bounds__(256, (NV == 2 || NA > MAX_A) ? 1 : 0)
ppo_loss_kernel(const float* __restrict__ out, const int32_t* __restrict__ idx, const void* __restrict__ action_all,
                const float* __restrict__ adv_all, const float* __restrict__ ret_all,
                const float* __restrict__ vold_all, const float* __restrict__ logp_old_all, int B, int A, int nout,
                jbppo::HP hp, float* __restrict__ dout, float* __restrict__ stats /*[8 + 4*n_cta]*/,
                const float* __restrict__ ret_i_all, const float* __restrict__ vold_i_all) {
  __shared__ float sred[2 * NV * 32];
  const float invB = 1.0f / (float)B;
  // ---- pass 1 (every CTA, whole minibatch, fixed order): the two critic means per critic ------
  float c[2 * NV] = {};
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int r = idx ? idx[b] : b;
    const float v = out[(size_t)b * nout + (CONT ? 2 * A : A)];
    const float ret = ret_all[r], vold = vold_all[r];
    const float vclip = vold + fminf(fmaxf(v - vold, -hp.eps_clip), hp.eps_clip);
    const float d1 = v - ret, d2 = vclip - ret;
    c[0] += d1 * d1; c[1] += d2 * d2;
    if constexpr (NV == 2) {
      const float vi = out[(size_t)b * nout + (CONT ? 2 * A : A) + 1];
      const float reti = ret_i_all[r], voldi = vold_i_all[r];
      const float viclip = voldi + fminf(fmaxf(vi - voldi, -hp.eps_clip), hp.eps_clip);
      const float e1 = vi - reti, e2 = viclip - reti;
      c[2] += e1 * e1; c[3] += e2 * e2;
    }
  }
  jbppo::block_sum<2 * NV>(c, sred);
  const float c1 = c[0] * invB, c2 = c[1] * invB;
  float c3 = 0.f, c4 = 0.f;
  if constexpr (NV == 2) { c3 = c[2] * invB; c4 = c[3] * invB; }
  float w1, w2, u1 = 0.f, u2 = 0.f;
  jbppo::critic_weights(c1, c2, w1, w2);
  if constexpr (NV == 2) jbppo::critic_weights(c3, c4, u1, u2);

  // ---- pass 2: this CTA's rows -----------------------------------------------------------------
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float st[2] = {0.f, 0.f};
  float max_ratio = -INFINITY, min_prob = INFINITY;
  if (b < B) {
    const int r = idx ? idx[b] : b;
    jbppo::RowOutW<jbppo::width<NA>()> ro;
    const float* o = out + (size_t)b * nout;
    if constexpr (CONT) jbppo::row<true, NA>(o, A, 0, (const float*)action_all + (size_t)r * A, adv_all[r], ret_all[r], vold_all[r],
                               logp_old_all + (size_t)r * A, hp, invB, ro);
    else jbppo::row<false, NA>(o, A, ((const int32_t*)action_all)[r], nullptr, adv_all[r], ret_all[r], vold_all[r],
                           logp_old_all + r, hp, invB, ro);
    float* g = dout + (size_t)b * nout;
    const int npol = CONT ? 2 * A : A;
#pragma unroll
    for (int a = 0; a < (CONT ? 2 * NA : NA); ++a) if (a < npol) g[a] = ro.dpol[a];
    g[npol] = w1 * ro.dv1 + w2 * ro.dv2;
    if constexpr (NV == 2) {      // intrinsic critic: the same clipped pair around v_old_i
      const float vi = o[npol + 1], voldi = vold_i_all[r], reti = ret_i_all[r];
      const float dvi = vi - voldi;
      const float viclip = voldi + fminf(fmaxf(dvi, -hp.eps_clip), hp.eps_clip);
      const float in_clip = (dvi >= -hp.eps_clip && dvi <= hp.eps_clip) ? 1.f : 0.f;
      const float e1 = vi - reti, e2 = viclip - reti;
      g[npol + 1] = u1 * (hp.vf_coef * invB * 2.f * e1) + u2 * (hp.vf_coef * invB * 2.f * e2 * in_clip);
    }
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
    float* sp = stats + 8 + 4 * blockIdx.x;     // per-CTA partials after the 8 final slots
    sp[0] = st[0]; sp[1] = st[1]; sp[2] = mr; sp[3] = mp;
    if (blockIdx.x == 0) {
      if constexpr (NV == 2) {
        const float ce = fmaxf(c1, c2), ci = fmaxf(c3, c4);
        stats[1] = ce + ci; stats[5] = ce; stats[6] = ci; stats[7] = 0.f;
      } else {
        stats[1] = fmaxf(c1, c2);
      }
    }
  }
}

// folds the per-CTA partials written by ppo_loss_kernel into stats[0..4] and accumulates running
// sums for the learn()-level result dict: acc[0..2] += losses, acc[3] = max(max_ratio), acc[4] =
// min(min_prob), acc[5] += 1
__global__ void ppo_stats_finalize_kernel(float* __restrict__ stats, int n_cta, int B, int A, int cont,
                                          float* __restrict__ acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  jbppo::fold_stats(stats, n_cta, B, A, cont, acc);
}

// cur_idx[0..B) = perm[cursor*B .. cursor*B+B); cursor += 1.  Lets a captured CUDA graph of one
// minibatch step be replayed for every minibatch of an epoch (ppo.py:118-120 slicing of the
// shuffled index array) without baking the offset into the graph.
__global__ void take_minibatch_kernel(const int32_t* __restrict__ perm, long long* __restrict__ cursor, int B,
                                      int32_t* __restrict__ cur_idx) {
  const long long base = (*cursor) * (long long)B;
  for (int i = threadIdx.x; i < B; i += blockDim.x) cur_idx[i] = perm[base + i];
  __syncthreads();
  if (threadIdx.x == 0) *cursor += 1;
}

// The instantiation of each kernel for the action kind and A, for one or two value columns.
template <int NV>
void launch_prepass(int continuous, const float* out, const void* action, int M, int A, int nout, float* value,
                    float* logp_old, float* value_i, cudaStream_t s) {
  const dim3 grid(jb_div_up(M, 128));
  if (continuous) ppo_prepass_kernel<true, MAX_A, NV><<<grid, 128, 0, s>>>(out, action, M, A, nout, value, logp_old, value_i);
  else if (A <= MAX_A) ppo_prepass_kernel<false, MAX_A, NV><<<grid, 128, 0, s>>>(out, action, M, A, nout, value, logp_old, value_i);
  else ppo_prepass_kernel<false, MAX_A_DISC, NV><<<grid, 128, 0, s>>>(out, action, M, A, nout, value, logp_old, value_i);
}

template <int NV>
void launch_loss(int continuous, const float* out, const int32_t* idx, const void* action, const float* adv,
                 const float* ret, const float* value_old, const float* ret_i, const float* value_i_old,
                 const float* logp_old, int B, int A, int nout, jbppo::HP hp, float* dout, float* stats, float* acc,
                 cudaStream_t s) {
  const int n_cta = jb_div_up(B, 256);
  if (continuous)
    ppo_loss_kernel<true, MAX_A, NV><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, logp_old, B, A, nout, hp,
                                                           dout, stats, ret_i, value_i_old);
  else if (A <= MAX_A)
    ppo_loss_kernel<false, MAX_A, NV><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, logp_old, B, A, nout, hp,
                                                            dout, stats, ret_i, value_i_old);
  else
    ppo_loss_kernel<false, MAX_A_DISC, NV><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, logp_old, B, A,
                                                                 nout, hp, dout, stats, ret_i, value_i_old);
  ppo_stats_finalize_kernel<<<1, 32, 0, s>>>(stats, n_cta, B, A, continuous, acc);
}

}  // namespace

JB_API int jb_take_minibatch(const int32_t* perm, long long* cursor, int B, int32_t* cur_idx, void* stream) {
  if (!perm || !cursor || !cur_idx || B <= 0) return JB_ERR_INVALID;
  take_minibatch_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(perm, cursor, B, cur_idx);
  return jb_check_launch();
}

// Randomness: u[M] uniforms if given, else Philox(seed, stream_base + row, ctr + row_ctr[row]);
// row_ctr (device int64[M], may be NULL) is post-incremented per row so that a captured graph
// draws fresh numbers at every replay.
JB_API int jb_ppo_act_discrete(const float* out, int M, int A, int nout, const float* u, uint64_t seed,
                               uint64_t stream_base, uint64_t ctr, long long* row_ctr, int greedy, int64_t* action,
                               void* stream) {
  if (!out || !action || M <= 0 || A <= 0 || A > MAX_A_DISC || nout < A) return JB_ERR_INVALID;
  const dim3 grid(jb_div_up(M, 128));
  cudaStream_t s = (cudaStream_t)stream;
  if (A <= MAX_A) ppo_act_discrete_kernel<MAX_A><<<grid, 128, 0, s>>>(out, M, A, nout, u, seed, stream_base, ctr, row_ctr, greedy, action);
  else ppo_act_discrete_kernel<MAX_A_DISC><<<grid, 128, 0, s>>>(out, M, A, nout, u, seed, stream_base, ctr, row_ctr, greedy, action);
  return jb_check_launch();
}

JB_API int jb_ppo_act_continuous(const float* out, int M, int A, int nout, const float* normal, uint64_t seed,
                                 uint64_t stream_base, uint64_t ctr, long long* row_ctr, int greedy, float* action,
                                 void* stream) {
  if (!out || !action || M <= 0 || A <= 0 || A > MAX_A || nout < 2 * A) return JB_ERR_INVALID;
  ppo_act_continuous_kernel<<<jb_div_up(M, 128), 128, 0, (cudaStream_t)stream>>>(out, M, A, nout, normal, seed, stream_base, ctr, row_ctr, greedy, action);
  return jb_check_launch();
}

JB_API int jb_ppo_prepass_discrete(const float* out, const int32_t* action, int M, int A, int nout, float* value,
                                   float* logp_old, void* stream) {
  if (!out || !action || !value || !logp_old || M <= 0 || A <= 0 || A > MAX_A_DISC || nout != A + 1) return JB_ERR_INVALID;
  launch_prepass<1>(0, out, action, M, A, nout, value, logp_old, nullptr, (cudaStream_t)stream);
  return jb_check_launch();
}

JB_API int jb_ppo_prepass_continuous(const float* out, const float* action, int M, int A, int nout, float* value,
                                     float* logp_old, void* stream) {
  if (!out || !action || !value || !logp_old || M <= 0 || A <= 0 || A > MAX_A || nout != 2 * A + 1) return JB_ERR_INVALID;
  launch_prepass<1>(1, out, action, M, A, nout, value, logp_old, nullptr, (cudaStream_t)stream);
  return jb_check_launch();
}

// RND-PPO's two-value policy network: out[M, nout] = [logits(A) | v | v_i] (nout = A + 2) or
// [mu_raw(A) | log_std_raw(A) | v | v_i] (nout = 2A + 2), so every column PPO's row maths reads stays where it is.
JB_API int jb_rnd_prepass(int continuous, const float* out, const void* action, int M, int A, int nout, float* value,
                          float* value_i, float* logp_old, void* stream) {
  if (!out || !action || !value || !value_i || !logp_old || M <= 0 || A <= 0) return JB_ERR_INVALID;
  if (A > (continuous ? MAX_A : MAX_A_DISC) || nout != (continuous ? 2 * A + 2 : A + 2)) return JB_ERR_INVALID;
  launch_prepass<2>(continuous, out, action, M, A, nout, value, logp_old, value_i, (cudaStream_t)stream);
  return jb_check_launch();
}

// out[B,nout]: head outputs of the minibatch rows (row b <-> rollout row idx[b], or b if idx NULL).
// action/adv/ret/value_old/logp_old are the *full-rollout* arrays, gathered through idx.
// dout[B,nout] receives d loss / d out.  stats must hold 8 + 4*ceil(B/256) floats:
//   [0] actor_loss [1] critic_loss [2] entropy_loss [3] max_ratio [4] min_prob; acc (6 floats,
//   may be NULL) accumulates them across minibatches on the device (ppo.py:171-175 without .item()).
JB_API int jb_ppo_loss(int continuous, const float* out, const int32_t* idx, const void* action, const float* adv,
                       const float* ret, const float* value_old, const float* logp_old, int B, int A, int nout,
                       float eps_clip, float vf_coef, float ent_coef, float* dout, float* stats, float* acc,
                       void* stream) {
  if (!out || !action || !adv || !ret || !value_old || !logp_old || !dout || !stats) return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || A > (continuous ? MAX_A : MAX_A_DISC) || nout != (continuous ? 2 * A + 1 : A + 1)) return JB_ERR_INVALID;
  launch_loss<1>(continuous, out, idx, action, adv, ret, value_old, nullptr, nullptr, logp_old, B, A, nout,
                 jbppo::HP{eps_clip, vf_coef, ent_coef}, dout, stats, acc, (cudaStream_t)stream);
  return jb_check_launch();
}

// jb_ppo_loss for the two-value policy network (see jb_rnd_prepass): PPO's actor and entropy terms and two clipped
// critics, v against ret around value_old and v_i against ret_i around value_i_old.  stats as jb_ppo_loss's, with [1] the
// sum of the two critic losses, [5] the extrinsic one and [6] the intrinsic one.  With ret_i = v_i = value_i_old every
// value written equals jb_ppo_loss's.
JB_API int jb_rnd_ppo_loss(int continuous, const float* out, const int32_t* idx, const void* action, const float* adv,
                           const float* ret, const float* value_old, const float* ret_i, const float* value_i_old,
                           const float* logp_old, int B, int A, int nout, float eps_clip, float vf_coef, float ent_coef,
                           float* dout, float* stats, float* acc, void* stream) {
  if (!out || !action || !adv || !ret || !value_old || !ret_i || !value_i_old || !logp_old || !dout || !stats)
    return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || A > (continuous ? MAX_A : MAX_A_DISC) || nout != (continuous ? 2 * A + 2 : A + 2))
    return JB_ERR_INVALID;
  launch_loss<2>(continuous, out, idx, action, adv, ret, value_old, ret_i, value_i_old, logp_old, B, A, nout,
                 jbppo::HP{eps_clip, vf_coef, ent_coef}, dout, stats, acc, (cudaStream_t)stream);
  return jb_check_launch();
}
