// PPO-specific row kernels: action sampling, old log-prob, and the fused clipped-surrogate /
// clipped-value / entropy loss forward + backward on the narrow head outputs.
//
// Reference: jorldy/core/agent/ppo.py
//   :54-69   act            -> jb_ppo_act_discrete / jb_ppo_act_continuous
//   :83-93   no-grad pass   -> jb_ppo_prepass_discrete / _continuous (value, log_prob_old)
//   :127-162 loss           -> jb_ppo_loss_discrete / _continuous (loss terms + d loss / d head outputs)
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

// ---- pre-pass: value + log_prob_old ------------------------------------------------------------
template <int NA>
__global__ void ppo_prepass_discrete_kernel(const float* __restrict__ out, const int32_t* __restrict__ action,
                                            int M, int A, int nout, float* __restrict__ value,
                                            float* __restrict__ logp_old) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float lg[NA], lsm[NA];
#pragma unroll
  for (int a = 0; a < NA; ++a) lg[a] = a < A ? out[(size_t)m * nout + a] : 0.f;
  log_softmax_row<NA>(lg, A, lsm);
  const int a = action[m];
  float la = 0.f;                              // lsm[a] without a run-time register index
#pragma unroll
  for (int q = 0; q < NA; ++q) if (q == a) la = lsm[q];
  logp_old[m] = logf(expf(la));                // pi.gather(1, a).log(), pi = exp(log_softmax)
  value[m] = out[(size_t)m * nout + A];
}

__global__ void ppo_prepass_continuous_kernel(const float* __restrict__ out, const float* __restrict__ action,
                                              int M, int A, int nout, float* __restrict__ value,
                                              float* __restrict__ logp_old /*[M,A]*/) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float log_sqrt_2pi = 0.9189385332046727f;
  for (int a = 0; a < A; ++a) {
    const float mu = fminf(fmaxf(out[(size_t)m * nout + a], -5.f), 5.f);
    const float sd = expf(tanhf(out[(size_t)m * nout + A + a]));
    const float z = atanh_clamped(action[(size_t)m * A + a]);
    const float d = z - mu;
    logp_old[(size_t)m * A + a] = -(d * d) / (2.f * (sd * sd)) - logf(sd) - log_sqrt_2pi;
  }
  value[m] = out[(size_t)m * nout + 2 * A];
}

// ---- loss -------------------------------------------------------------------------------------
// fixed-order block reduction; result broadcast to all threads
template <int NV>
__device__ __forceinline__ void block_sum(float* v, float* smem /*[NV][32]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    float x = v[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if (lane == 0) smem[q * 32 + warp] = x;
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    float t = 0.f;
    for (int w = 0; w < nw; ++w) t += smem[q * 32 + w];
    v[q] = t;
  }
  __syncthreads();
}

// NA: compile-time bound on A, see jbppo::row.  The 18-wide row holds ~145 live registers: min-blocks 1 lets ptxas use
// them instead of spilling at its default 128 (0 leaves the 8-wide instantiations unconstrained, as before).
template <bool CONT, int NA>
__global__ void __launch_bounds__(256, NA > MAX_A ? 1 : 0)
ppo_loss_kernel(const float* __restrict__ out, const int32_t* __restrict__ idx, const void* __restrict__ action_all,
                const float* __restrict__ adv_all, const float* __restrict__ ret_all,
                const float* __restrict__ vold_all, const float* __restrict__ logp_old_all, int B, int A, int nout,
                jbppo::HP hp, float* __restrict__ dout, float* __restrict__ stats /*[8 + 4*n_cta]*/) {
  __shared__ float sred[2 * 32];
  const float invB = 1.0f / (float)B;
  // ---- pass 1 (every CTA, whole minibatch, fixed order): the two critic means -----------------
  float c[2] = {0.f, 0.f};
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int r = idx ? idx[b] : b;
    const float v = out[(size_t)b * nout + (CONT ? 2 * A : A)];
    const float ret = ret_all[r], vold = vold_all[r];
    const float vclip = vold + fminf(fmaxf(v - vold, -hp.eps_clip), hp.eps_clip);
    const float d1 = v - ret, d2 = vclip - ret;
    c[0] += d1 * d1; c[1] += d2 * d2;
  }
  block_sum<2>(c, sred);
  const float c1 = c[0] * invB, c2 = c[1] * invB;
  float w1, w2;
  jbppo::critic_weights(c1, c2, w1, w2);

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
    st[0] = ro.surr_min; st[1] = ro.ent;
    max_ratio = ro.ratio; min_prob = ro.pmin;
  }
  block_sum<2>(st, sred);
  float mr = jb_warp_max(max_ratio), mp = jb_warp_min(min_prob);
  __shared__ float smax[32], smin_[32];
  if ((threadIdx.x & 31) == 0) { smax[threadIdx.x >> 5] = mr; smin_[threadIdx.x >> 5] = mp; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    for (int w = 1; w < nw; ++w) { mr = fmaxf(mr, smax[w]); mp = fminf(mp, smin_[w]); }
    float* sp = stats + 8 + 4 * blockIdx.x;     // per-CTA partials after the 8 final slots
    sp[0] = st[0]; sp[1] = st[1]; sp[2] = mr; sp[3] = mp;
    if (blockIdx.x == 0) stats[1] = fmaxf(c1, c2);
  }
}

// folds the per-CTA partials written by ppo_loss_kernel into stats[0..4] and accumulates running
// sums for the learn()-level result dict: acc[0..2] += losses, acc[3] = max(max_ratio), acc[4] =
// min(min_prob), acc[5] += 1
__global__ void ppo_stats_finalize_kernel(float* __restrict__ stats, int n_cta, int B, int A, int cont,
                                          float* __restrict__ acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float s0 = 0.f, s1 = 0.f, mr = -INFINITY, mp = INFINITY;
  for (int k = 0; k < n_cta; ++k) {
    const float* sp = stats + 8 + 4 * k;
    s0 += sp[0]; s1 += sp[1]; mr = fmaxf(mr, sp[2]); mp = fminf(mp, sp[3]);
  }
  const float invB = 1.0f / (float)B;
  stats[0] = -s0 * invB;                                   // actor_loss
  stats[2] = -s1 * invB / (cont ? (float)A : 1.f);         // entropy_loss
  stats[3] = mr; stats[4] = mp;
  if (acc) {
    acc[0] += stats[0]; acc[1] += stats[1]; acc[2] += stats[2];
    acc[3] = fmaxf(acc[3], mr); acc[4] = fminf(acc[4], mp); acc[5] += 1.f;
  }
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
  const dim3 grid(jb_div_up(M, 128));
  cudaStream_t s = (cudaStream_t)stream;
  if (A <= MAX_A) ppo_prepass_discrete_kernel<MAX_A><<<grid, 128, 0, s>>>(out, action, M, A, nout, value, logp_old);
  else ppo_prepass_discrete_kernel<MAX_A_DISC><<<grid, 128, 0, s>>>(out, action, M, A, nout, value, logp_old);
  return jb_check_launch();
}

JB_API int jb_ppo_prepass_continuous(const float* out, const float* action, int M, int A, int nout, float* value,
                                     float* logp_old, void* stream) {
  if (!out || !action || !value || !logp_old || M <= 0 || A <= 0 || A > MAX_A || nout != 2 * A + 1) return JB_ERR_INVALID;
  ppo_prepass_continuous_kernel<<<jb_div_up(M, 128), 128, 0, (cudaStream_t)stream>>>(out, action, M, A, nout, value, logp_old);
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
  jbppo::HP hp{eps_clip, vf_coef, ent_coef};
  const int n_cta = jb_div_up(B, 256);
  cudaStream_t s = (cudaStream_t)stream;
  if (continuous) ppo_loss_kernel<true, MAX_A><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, logp_old, B, A, nout, hp, dout, stats);
  else if (A <= MAX_A) ppo_loss_kernel<false, MAX_A><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, logp_old, B, A, nout, hp, dout, stats);
  else ppo_loss_kernel<false, MAX_A_DISC><<<n_cta, 256, 0, s>>>(out, idx, action, adv, ret, value_old, logp_old, B, A, nout, hp, dout, stats);
  ppo_stats_finalize_kernel<<<1, 32, 0, s>>>(stats, n_cta, B, A, continuous, acc);
  return jb_check_launch();
}
