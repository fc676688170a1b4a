// MPO (Abdolmaleki et al., arXiv:1806.06920) on the replay path: the Retrace critic target (Munos et al.,
// arXiv:1606.02647) over stored n-step windows, and the sampled E-step / decoupled-KL M-step policy loss
// (arXiv:1812.02256) with learned Lagrange multipliers [eta, alpha_mu, alpha_sigma].  The head conventions are PPO's
// (ppo_rowmath.cuh): discrete logits; continuous raw [mu | log_std], mu = clamp(raw, +-5), sd = exp(tanh(raw)), the
// action is tanh(z) and its log-density the Normal log-pdf of atanh(clamp(a, +-(1 - 1e-7))) without a Jacobian.
//
// A learn holds B windows of n steps.  Rows of a window are laid out oldest first: the n + 1 states s_0 .. s_n of
// window b are rows b (n + 1) + t, its n steps (action, reward, done, log mu, the online critic and actor rows) are
// rows b n + t.
//
//   jb_mpo_logp           log pi(a | s) of given actions under given head outputs (the behaviour log mu at act time)
//   jb_mpo_sample         z = mu' + sd' eps and tanh(z) for K normals per state row; the critic input rows repeat
//                         each state K (+1: the taken action) times
//   jb_mpo_critic_target  V'_t, c_t, the Retrace recursion in one warp per window, dL_Q/dQ and the loss stats
//   jb_mpo_policy_loss    E-step weights from the target networks, L_eta, L_pi, the KLs, L_alpha; d / d head outputs
//                         and d / d multipliers.  Per-CTA partials are folded in CTA order by a one-thread launch.
// No atomics anywhere: a learn is bit-reproducible.
#include "common.cuh"
#include "ppo_rowmath.cuh"

namespace {

using jbppo::MAX_A;
using jbppo::MAX_A_DISC;
using jbppo::log_softmax_row;
using jbppo::atanh_clamped;
using jbppo::block_sum;

constexpr int MPO_THREADS = 256;
constexpr int MPO_TARGET_THREADS = 512;   // 16 warps, one window per warp at a time
constexpr int MPO_PARTS = 5;              // per-CTA partials of the policy loss
constexpr int MPO_MAX_N = 32;
constexpr int MPO_MAX_K = 64;
constexpr float LOG_SQRT_2PI = 0.9189385332046727f;

// log N(atanh(clamp(a)); mu, sd) summed over the A dims, from the raw head row o = [mu_raw | log_std_raw]
template <int NA>
__device__ __forceinline__ float gauss_logp(const float* __restrict__ o, const float* __restrict__ a, int A) {
  float lp = 0.f;
#pragma unroll
  for (int j = 0; j < NA; ++j) {
    if (j < A) {
      const float mu = fminf(fmaxf(o[j], -5.f), 5.f);
      const float ls = tanhf(o[A + j]);
      const float sd = expf(ls);
      const float d = atanh_clamped(a[j]) - mu;
      lp += -0.5f * (d * d) * (1.f / (sd * sd)) - ls - LOG_SQRT_2PI;
    }
  }
  return lp;
}

template <int NA>
__device__ __forceinline__ float categorical_logp(const float* __restrict__ o, int A, int a) {
  float lg[NA], lsm[NA];
#pragma unroll
  for (int j = 0; j < NA; ++j) lg[j] = j < A ? o[j] : 0.f;
  log_softmax_row<NA>(lg, A, lsm);
  float r = 0.f;
#pragma unroll
  for (int j = 0; j < NA; ++j) if (j == a) r = lsm[j];
  return r;
}

template <bool CONT, int NA>
__global__ void __launch_bounds__(MPO_THREADS)
mpo_logp_kernel(const float* __restrict__ out, int nout, const void* __restrict__ action, int M, int A, float* __restrict__ logp) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  if constexpr (CONT) logp[m] = gauss_logp<NA>(out + (size_t)m * nout, (const float*)action + (size_t)m * A, A);
  else logp[m] = categorical_logp<NA>(out + (size_t)m * nout, A, (int)((const int64_t*)action)[m]);
}

// One element per (slot, column): slot = r * KK + k over R state rows and KK = K (+1) columns per row; columns 0..D-1
// copy the state row, columns D..D+A-1 write the action (a sample for k < K, the taken action for k = K).
__global__ void __launch_bounds__(MPO_THREADS)
mpo_sample_kernel(const float* __restrict__ raw, const float* __restrict__ eps, int R, int K, int A, const float* __restrict__ x,
                  int D, const float* __restrict__ taken, int n, float* __restrict__ z, float* __restrict__ xs,
                  float* __restrict__ as) {
  const int KK = taken ? K + 1 : K;
  const long long W = (long long)D + A;
  const long long total = (long long)R * KK * W;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long slot = e / W;
    const int c = (int)(e - slot * W);
    const int r = (int)(slot / KK), k = (int)(slot - (long long)r * KK);
    if (c < D) {
      xs[slot * D + c] = x[(long long)r * D + c];
      continue;
    }
    const int j = c - D;
    float a;
    if (k < K) {
      const float* o = raw + (size_t)r * 2 * A;
      const float mu = fminf(fmaxf(o[j], -5.f), 5.f);
      const float sd = expf(tanhf(o[A + j]));
      const float zz = mu + sd * eps[((size_t)r * K + k) * A + j];
      z[((size_t)r * K + k) * A + j] = zz;
      a = tanhf(zz);
    } else {
      const int b = r / (n + 1), t = r - b * (n + 1);
      a = t < n ? taken[((size_t)b * n + t) * A + j] : 0.f;
    }
    as[slot * A + j] = a;
  }
}

// One warp per window, lane t = step t.  Lane t reads row t + 1 of the target networks: V'_{t+1}, and for t + 1 < n
// c_{t+1} and Q'(s_{t+1}, a_{t+1}).  The recursion runs from t = n - 1 down, the running Qret broadcast by shuffles.
template <bool CONT, int NA>
__global__ void __launch_bounds__(MPO_TARGET_THREADS)
mpo_critic_target_kernel(const float* __restrict__ tq, const float* __restrict__ tout, const float* __restrict__ q,
                         const void* __restrict__ action, const float* __restrict__ log_mu, const float* __restrict__ reward,
                         const float* __restrict__ done, int B, int n, int A, int K, float gamma, int retrace,
                         float* __restrict__ dq, float* __restrict__ qret, float* __restrict__ stats) {
  __shared__ float sred[2][MPO_TARGET_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int tout_ld = CONT ? 2 * A : A;
  const float inv = 1.f / (float)(B * n);
  float acc_sq = 0.f, acc_q = 0.f;
  for (int b = warp; b < B; b += nw) {
    const int t = lane;
    float v = 0.f, c = 0.f, qn = 0.f, rt = 0.f, dt = 0.f, qt = 0.f;
    int at = 0;
    if (t < n) {
      const int row = b * (n + 1) + t + 1;          // state s_{t+1}
      const float* o = tout + (size_t)row * tout_ld;
      if constexpr (CONT) {
        const float* qs = tq + (size_t)row * (K + 1);
        for (int k = 0; k < K; ++k) v += qs[k];
        v *= 1.f / (float)K;
        if (t + 1 < n) {
          qn = qs[K];
          const int s1 = b * n + t + 1;
          if (retrace) c = fminf(1.f, expf(gauss_logp<NA>(o, (const float*)action + (size_t)s1 * A, A) - log_mu[s1]));
        }
      } else {
        float lg[NA], lsm[NA];
#pragma unroll
        for (int j = 0; j < NA; ++j) lg[j] = j < A ? o[j] : 0.f;
        log_softmax_row<NA>(lg, A, lsm);
        const float* qs = tq + (size_t)row * A;
#pragma unroll
        for (int j = 0; j < NA; ++j) if (j < A) v += expf(lsm[j]) * qs[j];
        if (t + 1 < n) {
          const int s1 = b * n + t + 1;
          const int a1 = (int)((const int64_t*)action)[s1];
          float lpa = 0.f;
#pragma unroll
          for (int j = 0; j < NA; ++j) if (j == a1) lpa = lsm[j];
          qn = qs[a1];
          if (retrace) c = fminf(1.f, expf(lpa - log_mu[s1]));
        }
      }
      const int s = b * n + t;
      rt = reward[s];
      dt = done[s];
      if constexpr (CONT) qt = q[s];
      else { at = (int)((const int64_t*)action)[s]; qt = q[(size_t)s * A + at]; }
    }
    float next = 0.f, mine = 0.f;
    for (int tt = n - 1; tt >= 0; --tt) {
      const float val = rt + gamma * (1.f - dt) * (v + c * (next - qn));   // c = 0 at t = n - 1
      next = __shfl_sync(0xffffffffu, val, tt);
      if (lane == tt) mine = next;
    }
    if (t < n) {
      const int s = b * n + t;
      const float diff = qt - mine;
      qret[s] = mine;
      if constexpr (CONT) dq[s] = 2.f * diff * inv;
      else {
        for (int j = 0; j < A; ++j) dq[(size_t)s * A + j] = j == at ? 2.f * diff * inv : 0.f;
      }
      acc_sq += diff * diff;
      acc_q += mine;
    }
  }
  acc_sq = jb_warp_sum(acc_sq);
  acc_q = jb_warp_sum(acc_q);
  if (lane == 0) { sred[0][warp] = acc_sq; sred[1][warp] = acc_q; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, bq = 0.f;
    for (int w = 0; w < nw; ++w) { a += sred[0][w]; bq += sred[1][w]; }
    stats[0] = a * inv;
    stats[1] = bq * inv;
  }
}

// One thread per state row s = b n + t (target row b (n + 1) + t).  part = [eta-free log-mean-exp (discrete: the
// log-partition under pi'), its d / d eta, L_pi row, KL_mu row, KL_sigma row].
template <bool CONT, int NA>
__global__ void __launch_bounds__(MPO_THREADS, NA > MAX_A ? 1 : 0)
mpo_policy_kernel(const float* __restrict__ out, const float* __restrict__ tout, const float* __restrict__ tq,
                  const float* __restrict__ zs, int B, int n, int A, int K, const float* __restrict__ mult,
                  float* __restrict__ dout, float* __restrict__ partials) {
  __shared__ float sred[MPO_PARTS * 32];
  const int S = B * n;
  const float eta = mult[0], alpha_mu = mult[1], alpha_sigma = mult[2];
  const float invS = 1.f / (float)S;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  float part[MPO_PARTS] = {0.f, 0.f, 0.f, 0.f, 0.f};
  if (s < S) {
    const int b = s / n, t = s - b * n;
    const int row = b * (n + 1) + t;
    if constexpr (!CONT) {
      const float* o = out + (size_t)s * A;
      const float* oo = tout + (size_t)row * A;
      const float* qs = tq + (size_t)row * A;
      float lg[NA], lgo[NA], lsm[NA], lsmo[NA], x[NA];
#pragma unroll
      for (int a = 0; a < NA; ++a) { lg[a] = a < A ? o[a] : 0.f; lgo[a] = a < A ? oo[a] : 0.f; }
      log_softmax_row<NA>(lg, A, lsm);
      log_softmax_row<NA>(lgo, A, lsmo);
      float m = -INFINITY;
#pragma unroll
      for (int a = 0; a < NA; ++a) { x[a] = 0.f; if (a < A) { x[a] = lsmo[a] + qs[a] / eta; m = fmaxf(m, x[a]); } }
      float Z = 0.f, sdx = 0.f, slp = 0.f;
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        if (a < A) { const float e = expf(x[a] - m); Z += e; sdx += e * (m - x[a]); slp += e * lsmo[a]; }
      }
      const float iZ = 1.f / Z, logZ = logf(Z);
      part[0] = m + logZ;                              // log sum_a pi'(a) exp(Q'(a) / eta)
      part[1] = sdx * iZ + logZ + slp * iZ;             // d (eta part[0]) / d eta, no cancellation of ~Q'/eta terms
      float lpi = 0.f, kl = 0.f, so = 0.f, sq = 0.f;
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        if (a < A) {
          const float qa = expf(x[a] - m) * iZ;
          const float po = expf(lsmo[a]);
          lpi -= qa * lsm[a];
          kl += po * (lsmo[a] - lsm[a]);
          so += po;
          sq += qa;
        }
      }
      part[2] = lpi; part[3] = kl;
      const float ck = alpha_mu * invS;
      float* g = dout + (size_t)s * A;
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        if (a < A) {
          const float p = expf(lsm[a]);
          const float qa = expf(x[a] - m) * iZ;
          g[a] = -(qa - p * sq) * invS + ck * (p * so - expf(lsmo[a]));
        }
      }
    } else {
      const float* o = out + (size_t)s * 2 * A;
      const float* oo = tout + (size_t)row * 2 * A;
      const float* qs = tq + (size_t)row * (K + 1);
      const float* zr = zs + (size_t)row * K * A;
      float m = -INFINITY;
      for (int k = 0; k < K; ++k) m = fmaxf(m, qs[k] / eta);
      float Z = 0.f, sdx = 0.f;
      for (int k = 0; k < K; ++k) { const float x = qs[k] / eta; const float e = expf(x - m); Z += e; sdx += e * (m - x); }
      const float iZ = 1.f / Z, logZ = logf(Z), logK = logf((float)K);
      part[0] = m + logZ - logK;                       // log mean_k exp(Q'(a_k) / eta)
      part[1] = sdx * iZ + logZ - logK;
      float mu[NA], ls[NA], sd[NA], mu_o[NA], ls_o[NA], sd_o[NA], q1[NA], q2[NA], q3[NA];
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        mu[a] = ls[a] = mu_o[a] = ls_o[a] = q1[a] = q2[a] = q3[a] = 0.f; sd[a] = sd_o[a] = 1.f;
        if (a < A) {
          mu[a] = fminf(fmaxf(o[a], -5.f), 5.f); ls[a] = tanhf(o[A + a]); sd[a] = expf(ls[a]);
          mu_o[a] = fminf(fmaxf(oo[a], -5.f), 5.f); ls_o[a] = tanhf(oo[A + a]); sd_o[a] = expf(ls_o[a]);
        }
      }
      // q1 = sum_k q_k z_k, q2 = sum_k q_k (z_k - mu)^2, q3 = sum_k q_k (z_k - mu')^2 per dim
      float sq = 0.f;
      for (int k = 0; k < K; ++k) {
        const float qk = expf(qs[k] / eta - m) * iZ;
        sq += qk;
#pragma unroll
        for (int a = 0; a < NA; ++a) {
          if (a < A) {
            const float zz = zr[k * A + a];
            const float d1 = zz - mu[a], d2 = zz - mu_o[a];
            q1[a] += qk * zz; q2[a] += qk * (d1 * d1); q3[a] += qk * (d2 * d2);
          }
        }
      }
      const float cm = alpha_mu * invS, cs = alpha_sigma * invS;
      float lpi = 0.f, km = 0.f, ks = 0.f;
      float* g = dout + (size_t)s * 2 * A;
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        if (a < A) {
          const float iv = 1.f / (sd[a] * sd[a]), ivo = 1.f / (sd_o[a] * sd_o[a]), isd = 1.f / sd[a];
          // log N(z; mu, sd') + log N(z; mu', sd), weighted by q_k and summed over k
          lpi -= -0.5f * q2[a] * ivo - sq * ls_o[a] - 0.5f * q3[a] * iv - sq * ls[a] - 2.f * sq * LOG_SQRT_2PI;
          const float dm = mu[a] - mu_o[a];
          km += 0.5f * (dm * dm) * ivo;
          const float r = (sd_o[a] * sd_o[a]) * iv;
          ks += 0.5f * (r - 1.f + 2.f * (ls[a] - ls_o[a]));
          const float gmu = -(q1[a] - sq * mu[a]) * ivo * invS + cm * dm * ivo;
          const float gsd = (-(q3[a] * iv - sq) * invS + cs * (1.f - r)) * isd;
          const float in_mu = (o[a] >= -5.f && o[a] <= 5.f) ? 1.f : 0.f;
          g[a] = gmu * in_mu;
          g[A + a] = gsd * sd[a] * (1.f - ls[a] * ls[a]);
        }
      }
      part[2] = lpi; part[3] = km; part[4] = ks;
    }
  }
  block_sum<MPO_PARTS, MPO_THREADS / 32>(part, sred);
  if (threadIdx.x == 0) {
    float* p = partials + MPO_PARTS * blockIdx.x;
#pragma unroll
    for (int q = 0; q < MPO_PARTS; ++q) p[q] = part[q];
  }
}

// stats[0..4] = L_pi, L_eta, L_alpha, mean KL_mu (discrete: the KL), mean KL_sigma; dmult = d loss / d mult
__global__ void mpo_policy_finalize_kernel(const float* __restrict__ partials, int n_cta, int S, int cont,
                                           const float* __restrict__ mult, float eps_eta, float eps_alpha_mu,
                                           float eps_alpha_sigma, float* __restrict__ dmult, float* __restrict__ stats) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float p[MPO_PARTS] = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (int c = 0; c < n_cta; ++c)
    for (int q = 0; q < MPO_PARTS; ++q) p[q] += partials[MPO_PARTS * c + q];
  const float invS = 1.f / (float)S;
  const float eta = mult[0], alpha_mu = mult[1], alpha_sigma = mult[2];
  const float lme = p[0] * invS, km = p[3] * invS, ks = p[4] * invS;
  float l_alpha = alpha_mu * (eps_alpha_mu - km) + alpha_mu * km;
  if (cont) l_alpha += alpha_sigma * (eps_alpha_sigma - ks) + alpha_sigma * ks;
  dmult[0] = eps_eta + p[1] * invS;
  dmult[1] = eps_alpha_mu - km;
  dmult[2] = cont ? eps_alpha_sigma - ks : 0.f;
  stats[0] = p[2] * invS;
  stats[1] = eta * eps_eta + eta * lme;
  stats[2] = l_alpha;
  stats[3] = km;
  stats[4] = ks;
}

}  // namespace

JB_API int jb_mpo_logp(int continuous, const float* out, int nout, const void* action, int M, int A, float* logp,
                       void* stream) {
  if (!out || !action || !logp || M < 0 || A <= 0 || A > (continuous ? MAX_A : MAX_A_DISC)) return JB_ERR_INVALID;
  if (nout < (continuous ? 2 * A : A)) return JB_ERR_INVALID;
  if (M == 0) return JB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int g = jb_div_up(M, MPO_THREADS);
  if (continuous) mpo_logp_kernel<true, MAX_A><<<g, MPO_THREADS, 0, s>>>(out, nout, action, M, A, logp);
  else if (A <= MAX_A) mpo_logp_kernel<false, MAX_A><<<g, MPO_THREADS, 0, s>>>(out, nout, action, M, A, logp);
  else mpo_logp_kernel<false, MAX_A_DISC><<<g, MPO_THREADS, 0, s>>>(out, nout, action, M, A, logp);
  return jb_check_launch();
}

JB_API int jb_mpo_sample(const float* raw, const float* eps, int R, int K, int A, const float* x, int D, const float* taken,
                         int n, float* z, float* xs, float* as, void* stream) {
  if (!raw || !eps || !x || !z || !xs || !as || R <= 0 || K <= 0 || K > MPO_MAX_K || A <= 0 || A > MAX_A || D <= 0)
    return JB_ERR_INVALID;
  if (taken && (n <= 0 || R % (n + 1))) return JB_ERR_INVALID;
  const long long total = (long long)R * (K + (taken ? 1 : 0)) * (D + A);
  mpo_sample_kernel<<<jb_grid_for(total, MPO_THREADS, 8), MPO_THREADS, 0, (cudaStream_t)stream>>>(
      raw, eps, R, K, A, x, D, taken, n, z, xs, as);
  return jb_check_launch();
}

JB_API int jb_mpo_critic_target(int continuous, const float* tq, const float* tout, const float* q, const void* action,
                                const float* log_mu, const float* reward, const float* done, int B, int n, int A, int K,
                                float gamma, int retrace, float* dq, float* qret, float* stats, void* stream) {
  if (!tq || !tout || !q || !action || !log_mu || !reward || !done || !dq || !qret || !stats) return JB_ERR_INVALID;
  if (B <= 0 || n <= 0 || n > MPO_MAX_N || A <= 0 || A > (continuous ? MAX_A : MAX_A_DISC)) return JB_ERR_INVALID;
  if (continuous && (K <= 0 || K > MPO_MAX_K)) return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
#define MPO_TARGET_ARGS tq, tout, q, action, log_mu, reward, done, B, n, A, K, gamma, retrace, dq, qret, stats
  if (continuous) mpo_critic_target_kernel<true, MAX_A><<<1, MPO_TARGET_THREADS, 0, s>>>(MPO_TARGET_ARGS);
  else if (A <= MAX_A) mpo_critic_target_kernel<false, MAX_A><<<1, MPO_TARGET_THREADS, 0, s>>>(MPO_TARGET_ARGS);
  else mpo_critic_target_kernel<false, MAX_A_DISC><<<1, MPO_TARGET_THREADS, 0, s>>>(MPO_TARGET_ARGS);
#undef MPO_TARGET_ARGS
  return jb_check_launch();
}

JB_API int jb_mpo_policy_partials(int S) { return MPO_PARTS * jb_div_up(S, MPO_THREADS); }

JB_API int jb_mpo_policy_loss(int continuous, const float* out, const float* tout, const float* tq, const float* z, int B,
                              int n, int A, int K, const float* mult, float eps_eta, float eps_alpha_mu,
                              float eps_alpha_sigma, float* dout, float* dmult, float* partials, float* stats,
                              void* stream) {
  if (!out || !tout || !tq || !mult || !dout || !dmult || !partials || !stats) return JB_ERR_INVALID;
  if (B <= 0 || n <= 0 || n > MPO_MAX_N || A <= 0 || A > (continuous ? MAX_A : MAX_A_DISC)) return JB_ERR_INVALID;
  if (continuous && (!z || K <= 0 || K > MPO_MAX_K)) return JB_ERR_INVALID;
  const int S = B * n, n_cta = jb_div_up(S, MPO_THREADS);
  cudaStream_t s = (cudaStream_t)stream;
#define MPO_POLICY_ARGS out, tout, tq, z, B, n, A, K, mult, dout, partials
  if (continuous) mpo_policy_kernel<true, MAX_A><<<n_cta, MPO_THREADS, 0, s>>>(MPO_POLICY_ARGS);
  else if (A <= MAX_A) mpo_policy_kernel<false, MAX_A><<<n_cta, MPO_THREADS, 0, s>>>(MPO_POLICY_ARGS);
  else mpo_policy_kernel<false, MAX_A_DISC><<<n_cta, MPO_THREADS, 0, s>>>(MPO_POLICY_ARGS);
#undef MPO_POLICY_ARGS
  mpo_policy_finalize_kernel<<<1, 32, 0, s>>>(partials, n_cta, S, continuous, mult, eps_eta, eps_alpha_mu, eps_alpha_sigma,
                                              dmult, stats);
  return jb_check_launch();
}
