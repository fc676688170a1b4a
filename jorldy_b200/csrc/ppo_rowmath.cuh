// Per-row PPO loss forward + backward on the pre-activation head outputs, shared by the
// stand-alone loss kernel (ppo.cu) and the persistent minibatch-loop kernel (ppo_fused.cu) so both
// produce bit-identical values.
//
// Reference: jorldy/core/agent/ppo.py:127-162 and torch.distributions Categorical / Normal (see the
// header of ppo.cu for the restated definitions).
#pragma once
#include "common.cuh"

namespace jbppo {

constexpr int MAX_A = 8;        // continuous PPO, and every action count of the persistent kernel (ppo_fused.cu)
constexpr int MAX_A_DISC = 18;  // discrete PPO row kernels (ppo.cu): ALE's full action set
constexpr float F32_EPS = 1.1920928955078125e-07f;   // torch.finfo(float32).eps

struct HP { float eps_clip, vf_coef, ent_coef; };

// Register width of the per-action arrays of row<., NA>: MAX_A up to NA = 8, so those instantiations keep the layout the
// persistent kernel is tuned for; NA itself above that.
template <int NA> constexpr int width() { return NA > MAX_A ? NA : MAX_A; }

template <int W = MAX_A>
struct RowOutW {
  float dpol[2 * W];       // d loss / d policy head outputs: discrete [A] logits; continuous [A] mu then [A] log_std
  float dv1, dv2;          // value-head gradient if critic_loss1 / critic_loss2 is the max (already x vf_coef / B)
  float sq1, sq2;          // (v - ret)^2, (v_clip - ret)^2
  float d1, d2;            // v - ret, v_clip - ret
  float surr_min, ent;     // min(surr1, surr2), entropy (continuous: summed over dims)
  float ratio, pmin;       // ratio; exp(log_prob) (continuous: min over dims)
};
using RowOut = RowOutW<MAX_A>;

// All per-action loops run over a compile-time bound (NA, or the array width W >= NA) with an `a < A` guard: arrays stay
// in registers (a run-time trip count would index them dynamically and put them in local memory) and the arithmetic
// order is the plain ascending-a order of the restated definitions.
template <int NA = MAX_A, int W>
__device__ __forceinline__ void log_softmax_row(const float (&lg)[W], int A, float (&lsm)[W]) {
  float mx = lg[0];
#pragma unroll
  for (int a = 1; a < NA; ++a) if (a < A) mx = fmaxf(mx, lg[a]);
  float s = 0.f;
#pragma unroll
  for (int a = 0; a < NA; ++a) if (a < A) s += expf(lg[a] - mx);
  const float ls = logf(s);
#pragma unroll
  for (int a = NA; a < W; ++a) lsm[a] = 0.f;
#pragma unroll
  for (int a = 0; a < NA; ++a) lsm[a] = a < A ? (lg[a] - mx) - ls : 0.f;
}

__device__ __forceinline__ float atanh_clamped(float a) {
  const float hi = (float)(1.0 - 1e-7), lo = (float)(-1.0 + 1e-7);
  return atanhf(fminf(fmaxf(a, lo), hi));
}

__device__ __forceinline__ void surrogate(float ratio, float adv, float eps, float& smin, float& g) {
  const float s1 = ratio * adv;
  const float rc = fminf(fmaxf(ratio, 1.f - eps), 1.f + eps);
  const float s2 = rc * adv;
  const float inr = (ratio >= 1.f - eps && ratio <= 1.f + eps) ? 1.f : 0.f;
  smin = fminf(s1, s2);
  if (s1 < s2) g = adv;
  else if (s1 > s2) g = adv * inr;
  else g = 0.5f * adv + 0.5f * adv * inr;        // torch.minimum splits ties
}

// o: the row's head outputs [nout] (at least 2*MAX_A... entries readable up to index nout-1); a_disc / a_cont:
// the stored action; lpo: log_prob_old (1 or A values)
// NA: compile-time bound on A (the loops run to NA, guarded by a < A): row<., 2> costs a quarter of row<., 8>.
// Continuous rows take NA <= MAX_A, discrete rows NA <= MAX_A_DISC.
template <bool CONT, int NA = MAX_A, int W = width<NA>()>
__device__ __forceinline__ void row(const float* o, int A, int a_disc, const float* a_cont, float adv, float ret,
                                    float vold, const float* lpo, HP hp, float invB, RowOutW<W>& r) {
  static_assert(NA <= (CONT ? MAX_A : MAX_A_DISC) && W >= NA, "row: action bound out of range");
  float v = 0.f;                                   // o[CONT ? 2A : A] without a run-time register index
#pragma unroll
  for (int q = 0; q < 2 * NA + 1; ++q) if (q == (CONT ? 2 * A : A)) v = o[q];
  const float dv_raw = v - vold;
  const float vclip = vold + fminf(fmaxf(dv_raw, -hp.eps_clip), hp.eps_clip);
  const float in_clip = (dv_raw >= -hp.eps_clip && dv_raw <= hp.eps_clip) ? 1.f : 0.f;
  const float d1 = v - ret, d2 = vclip - ret;
  r.sq1 = d1 * d1; r.sq2 = d2 * d2;
  r.d1 = d1; r.d2 = d2;
  r.dv1 = hp.vf_coef * invB * 2.f * d1;
  r.dv2 = hp.vf_coef * invB * 2.f * d2 * in_clip;
#pragma unroll
  for (int q = 0; q < 2 * W; ++q) r.dpol[q] = 0.f;
  if (!CONT) {
    float lg[W], lsm[W], pi[W], p[W], lc[W], inr[W];
#pragma unroll
    for (int a = 0; a < W; ++a) lg[a] = (a < NA && a < A) ? o[a] : 0.f;
    log_softmax_row<NA>(lg, A, lsm);
    float S = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) { pi[a] = 0.f; if (a < A) { pi[a] = expf(lsm[a]); S += pi[a]; } }
    float ent = 0.f, logp = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      p[a] = 1.f; lc[a] = 0.f; inr[a] = 0.f;
      if (a < A) {
        p[a] = pi[a] / S;
        const float pc = fminf(fmaxf(p[a], F32_EPS), 1.f - F32_EPS);
        inr[a] = (p[a] >= F32_EPS && p[a] <= 1.f - F32_EPS) ? 1.f : 0.f;
        lc[a] = logf(pc);
        ent -= lc[a] * p[a];
        if (a == a_disc) logp = lc[a];
      }
    }
    const float ratio = expf(logp - lpo[0]);
    float smin, gr;
    surrogate(ratio, adv, hp.eps_clip, smin, gr);
    r.surr_min = smin; r.ent = ent; r.ratio = ratio; r.pmin = expf(logp);
    const float dlogp = -gr * ratio * invB;            // d(actor_loss)/d log_prob
    const float dent = -hp.ent_coef * invB;            // d(ent_coef * entropy_loss)/d entropy_b
    float dp[W], dot = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      dp[a] = 0.f;
      if (a < A) {
        float t = dent * (-(lc[a] + inr[a]));
        if (a == a_disc) t += dlogp * inr[a] / p[a];
        dp[a] = t;
        dot += t * pi[a];
      }
    }
    float dlsm[W], sum_dlsm = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      dlsm[a] = 0.f;
      if (a < A) {
        const float dpi = dp[a] / S - dot / (S * S);
        dlsm[a] = dpi * pi[a];
        sum_dlsm += dlsm[a];
      }
    }
#pragma unroll
    for (int a = 0; a < NA; ++a) if (a < A) r.dpol[a] = dlsm[a] - expf(lsm[a]) * sum_dlsm;
  } else {
    const float log_sqrt_2pi = 0.9189385332046727f;
    float dsum = 0.f, ent = 0.f;
    float omu[W], ols[W], mu[W], sd[W], ls[W], z[W], dmu_[W], dls_[W];
#pragma unroll
    for (int a = 0; a < NA; ++a) {                 // o[a] and o[A + a] without run-time register indices
      omu[a] = a < A ? o[a] : 0.f;
      float t = 0.f;
#pragma unroll
      for (int q = 0; q < 2 * NA; ++q) if (q == A + a && a < A) t = o[q];
      ols[a] = t;
    }
    float pmin = INFINITY;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      mu[a] = sd[a] = ls[a] = z[a] = 0.f;
      if (a < A) {
        mu[a] = fminf(fmaxf(omu[a], -5.f), 5.f);
        ls[a] = tanhf(ols[a]);
        sd[a] = expf(ls[a]);
        z[a] = atanh_clamped(a_cont[a]);
        const float d = z[a] - mu[a];
        const float logp = -(d * d) / (2.f * (sd[a] * sd[a])) - logf(sd[a]) - log_sqrt_2pi;
        dsum += logp - lpo[a];
        ent += 0.5f + 0.5f * 1.8378770664093453f + logf(sd[a]);
        pmin = fminf(pmin, expf(logp));
      }
    }
    const float ratio = expf(dsum);
    float smin, gr;
    surrogate(ratio, adv, hp.eps_clip, smin, gr);
    r.surr_min = smin; r.ent = ent; r.ratio = ratio; r.pmin = pmin;
    const float dlogp = -gr * ratio * invB;
    const float dent = -hp.ent_coef * invB / (float)A;   // entropy_loss = -mean over B*A elements
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      dmu_[a] = dls_[a] = 0.f;
      if (a < A) {
        const float d = z[a] - mu[a];
        const float var = sd[a] * sd[a];
        const float dmu = dlogp * d / var;
        const float dsd = dlogp * (d * d / (var * sd[a]) - 1.f / sd[a]) + dent / sd[a];
        const float in_mu = (omu[a] >= -5.f && omu[a] <= 5.f) ? 1.f : 0.f;
        dmu_[a] = dmu * in_mu;
        dls_[a] = dsd * sd[a] * (1.f - ls[a] * ls[a]);
      }
    }
#pragma unroll
    for (int q = 0; q < 2 * NA; ++q) {
      float t = 0.f;
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        if (a < A && q == a) t = dmu_[a];
        if (a < A && q == A + a) t = dls_[a];
      }
      r.dpol[q] = t;
    }
  }
}

// weights of the two critic means in max(c1, c2) (torch.maximum splits ties)
__device__ __forceinline__ void critic_weights(float c1, float c2, float& w1, float& w2) {
  w1 = (c1 > c2) ? 1.f : ((c1 == c2) ? 0.5f : 0.f);
  w2 = 1.f - w1;
}

// log_prob_old of one pre-pass row (ppo.py:83-93), shared by PPO's and RND-PPO's pre-pass kernels.
// Discrete: pi.gather(1, a).log() with pi = exp(log_softmax(o[0..A))).  NA: compile-time bound on A.
template <int NA>
__device__ __forceinline__ float logp_discrete(const float* o, int A, int a) {
  float lg[NA], lsm[NA];
#pragma unroll
  for (int q = 0; q < NA; ++q) lg[q] = q < A ? o[q] : 0.f;
  log_softmax_row<NA>(lg, A, lsm);
  float la = 0.f;                              // lsm[a] without a run-time register index
#pragma unroll
  for (int q = 0; q < NA; ++q) if (q == a) la = lsm[q];
  return logf(expf(la));
}

// Normal(mu, sd).log_prob(z) of one action dimension.
__device__ __forceinline__ float normal_logpdf(float z, float mu, float sd) {
  const float log_sqrt_2pi = 0.9189385332046727f;
  const float d = z - mu;
  return -(d * d) / (2.f * (sd * sd)) - logf(sd) - log_sqrt_2pi;
}

// Continuous: lp[a] = Normal(clamp(mu, +-5), exp(tanh(log_std))).log_prob(atanh(clamp(action[a], +-(1 - 1e-7)))).
__device__ __forceinline__ void logp_continuous(const float* o, int A, const float* action, float* lp) {
  for (int a = 0; a < A; ++a) {
    const float mu = fminf(fmaxf(o[a], -5.f), 5.f);
    const float sd = expf(tanhf(o[A + a]));
    const float z = atanh_clamped(action[a]);
    lp[a] = normal_logpdf(z, mu, sd);
  }
}

// fixed-order block reduction of NV values; result broadcast to all threads.  NW: the warp count when the caller's block
// size is a compile-time constant (0: read it from blockDim).
template <int NV, int NW = 0>
__device__ __forceinline__ void block_sum(float* v, float* smem /*[NV][32]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = NW ? NW : (blockDim.x + 31) >> 5;
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

// One thread folds the per-CTA partials (stats + 8 + 4 k: surr_min sum, entropy sum, max ratio, min prob) in CTA order
// into stats[0] actor_loss, stats[2] entropy_loss, stats[3] max_ratio, stats[4] min_prob; stats[1] (the critic loss) is
// the loss kernel's.  acc (may be NULL): acc[0..2] += stats[0..2], acc[3] = max, acc[4] = min, acc[5] += 1.
__device__ __forceinline__ void fold_stats(float* stats, int n_cta, int B, int A, int cont, float* acc) {
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

}  // namespace jbppo
