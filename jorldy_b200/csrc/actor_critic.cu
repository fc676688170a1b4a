// Row / element-wise kernels of the continuous off-policy family — jorldy/core/agent/ddpg.py, td3.py, sac.py
// (SURVEY.md 8f-4).  The dense layers are the shared jb_gemm tiles (linear.cu); what lives here is everything
// between them: soft target update, tanh policy head (+ TD3 noise), Ornstein-Uhlenbeck exploration, the TD target
// + MSE gradient for one or two critics, SAC's reparameterised sample / log-prob and its backward, and the
// entropy-temperature bookkeeping.  Reductions are single-CTA and fixed-order (B <= a few thousand rows).
#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int AC_MAX_A = 8;

// ---- t := tau * p + (1 - tau) * t  (ddpg.py:160-164, td3.py:190-196, sac.py:262-266) ---------------------------------
// torch evaluates `tau * p.data + (1 - tau) * t_p.data` as two rounded products and one rounded sum: no FMA here.
__global__ void soft_update_kernel(float* __restrict__ t, const float* __restrict__ p, long long n, float tau, float omt) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    t[i] = __fadd_rn(__fmul_rn(tau, p[i]), __fmul_rn(omt, t[i]));
}

// ---- out = clip(tanh(pre) + clip(noise * scale, +-noise_clip), +-out_clip) --------------------------------------------
// noise NULL: plain tanh head (policy.py:19-20).  noise_clip <= 0 / out_clip <= 0 disable the respective clamp.
// TD3 target smoothing (td3.py:153-156): scale = target_noise_std, noise_clip = target_noise_clip, out_clip = 1;
// TD3 act (td3.py:141-142): scale = action_noise_std, no noise clip, out_clip = 1.
__global__ void tanh_act_kernel(const float* __restrict__ pre, const float* __restrict__ noise, long long n,
                                float scale, float noise_clip, float out_clip, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a = tanhf(pre[i]);
  if (noise) {
    float z = __fmul_rn(noise[i], scale);
    if (noise_clip > 0.f) z = fminf(fmaxf(z, -noise_clip), noise_clip);
    a = __fadd_rn(a, z);
    if (out_clip > 0.f) a = fminf(fmaxf(a, -out_clip), out_clip);
  }
  out[i] = a;
}

// dpre = da * (1 - a^2)
__global__ void tanh_bwd_kernel(const float* __restrict__ da, const float* __restrict__ a, long long n,
                                float* __restrict__ dpre) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float t = a[i];
  dpre[i] = da[i] * (1.f - t * t);
}

// ---- Ornstein-Uhlenbeck exploration (agent/utils.py:8-26, ddpg.py:113-118) --------------------------------------------
// One process per env row, state X[M,A] in f64 (the reference's X turns f64 after the first sample).  The reference
// draws `randn(len(X))` with X of shape (1, A): ONE normal per step, shared by all action dimensions.
// action = tanh(pre) + clip(X, -1, 1) when training, tanh(pre) otherwise.
__global__ void ou_act_kernel(const float* __restrict__ pre, int M, int A, double* __restrict__ X,
                              const double* __restrict__ n_in, uint64_t seed, uint64_t stream_base,
                              long long* __restrict__ row_ctr, double theta, double mu, double sigma, int greedy,
                              float* __restrict__ action) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  double nz = 0.0;
  if (!greedy) {
    if (n_in) nz = n_in[m];
    else {
      const uint64_t ctr = jb_next_row_ctr(row_ctr, m);
      float n0, n1;
      jb_normal_pair(seed, stream_base + (uint64_t)m, ctr, n0, n1);
      nz = (double)n0;
    }
  }
  for (int j = 0; j < A; ++j) {
    const float t = tanhf(pre[(size_t)m * A + j]);
    if (greedy) { action[(size_t)m * A + j] = t; continue; }
    double x = X[(size_t)m * A + j];
    x = x + (theta * (mu - x) + sigma * nz);
    X[(size_t)m * A + j] = x;
    action[(size_t)m * A + j] = (float)((double)t + fmin(fmax(x, -1.0), 1.0));
  }
}

// ---- fills: standard normals / uniforms [lo, hi) from Philox ------------------------------------------------------------
__global__ void philox_fill_kernel(float* __restrict__ out, long long n, int kind, float lo, float hi, uint64_t seed,
                                   uint64_t stream, const long long* __restrict__ ctr_dev, uint64_t ctr) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // pair index
  if (2 * p >= n) return;
  if (ctr_dev) ctr += (uint64_t)ctr_dev[0];
  float v0, v1;
  if (kind == 0) jb_normal_pair(seed, stream + (uint64_t)p, ctr, v0, v1);
  else {
    jb_philox4 r = jb_philox(seed, stream + (uint64_t)p, ctr);
    v0 = lo + (hi - lo) * jb_u01_float(r.x);
    v1 = lo + (hi - lo) * jb_u01_float(r.y);
  }
  out[2 * p] = v0;
  if (2 * p + 1 < n) out[2 * p + 1] = v1;
}
__global__ void bump_kernel(long long* c) { c[0] += 1; }

// block-wide sum / max over 256 threads in a fixed order
__device__ __forceinline__ float block_sum256(float v, float* sm) {
  v = jb_warp_sum(v);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x < 32) {
    t = threadIdx.x < 8 ? sm[threadIdx.x] : 0.f;
    t = jb_warp_sum(t);
    if (threadIdx.x == 0) sm[8] = t;
  }
  __syncthreads();
  t = sm[8];
  __syncthreads();
  return t;
}
__device__ __forceinline__ float block_max256(float v, float* sm) {
  v = jb_warp_max(v);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
  if (threadIdx.x < 32) {
    t = threadIdx.x < 8 ? sm[threadIdx.x] : -INFINITY;
    t = jb_warp_max(t);
    if (threadIdx.x == 0) sm[8] = t;
  }
  __syncthreads();
  t = sm[8];
  __syncthreads();
  return t;
}

// ---- TD target + MSE for one or two critics -----------------------------------------------------------------------------
// y = r + ((1 - d) * gamma) * (min(nq1, nq2) + alpha * (-next_logp))        (ddpg.py:133-135, td3.py:157-160, sac.py:186-190)
// loss_i = mean((q_i - y)^2); dq_i = 2 (q_i - y) / B; stats = {loss1, loss2, max_b y}.
__global__ void __launch_bounds__(256) critic_loss_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                                          const float* __restrict__ nq1, const float* __restrict__ nq2,
                                                          const float* __restrict__ alpha, const float* __restrict__ next_logp,
                                                          const float* __restrict__ reward, const float* __restrict__ done,
                                                          int B, float gamma, float* __restrict__ dq1,
                                                          float* __restrict__ dq2, float* __restrict__ stats) {
  __shared__ float sm[9];
  float s1 = 0.f, s2 = 0.f, mx = -INFINITY;
  const float inv = 1.f / (float)B;
  const float al = (alpha && next_logp) ? alpha[0] : 0.f;
  for (int b = threadIdx.x; b < B; b += 256) {
    float nq = nq1[b];
    if (nq2) nq = fminf(nq, nq2[b]);
    if (alpha && next_logp) nq = __fadd_rn(nq, __fmul_rn(al, -next_logp[b]));
    const float y = __fadd_rn(reward[b], __fmul_rn(__fmul_rn(1.f - done[b], gamma), nq));
    mx = fmaxf(mx, y);
    const float e1 = q1[b] - y;
    s1 += e1 * e1;
    dq1[b] = 2.f * e1 * inv;
    if (q2) {
      const float e2 = q2[b] - y;
      s2 += e2 * e2;
      dq2[b] = 2.f * e2 * inv;
    }
  }
  s1 = block_sum256(s1, sm);
  s2 = block_sum256(s2, sm);
  mx = block_max256(mx, sm);
  if (threadIdx.x == 0) { stats[0] = s1 * inv; stats[1] = s2 * inv; stats[2] = mx; }
}

// ---- deterministic-policy actor loss: L = -mean(q)  (ddpg.py:143-144, td3.py:176-177): dq = -1/B ----------------------
__global__ void __launch_bounds__(256) neg_mean_kernel(const float* __restrict__ q, int B, float* __restrict__ dq,
                                                       float* __restrict__ stat) {
  __shared__ float sm[9];
  float s = 0.f;
  const float inv = 1.f / (float)B;
  for (int b = threadIdx.x; b < B; b += 256) { s += q[b]; dq[b] = -inv; }
  s = block_sum256(s, sm);
  if (threadIdx.x == 0) stat[0] = -s * inv;
}

// ---- SAC: a = tanh(mu + std * eps), log pi(a) with the tanh correction (sac.py:151-160, policy.py:50-56) ---------------
__global__ void sac_sample_kernel(const float* __restrict__ raw, int nout, const float* __restrict__ eps, int M, int A,
                                  float* __restrict__ action, float* __restrict__ logp) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float lp = 0.f;
  for (int j = 0; j < A; ++j) {
    const float mu = fminf(fmaxf(raw[(size_t)m * nout + j], -5.f), 5.f);
    const float sd = expf(tanhf(raw[(size_t)m * nout + A + j]));
    const float z = __fadd_rn(mu, __fmul_rn(eps[(size_t)m * A + j], sd));        // Normal.rsample: loc + eps * scale
    const float a = tanhf(z);
    action[(size_t)m * A + j] = a;
    const float dz = z - mu;
    float l = -(dz * dz) / (2.f * (sd * sd)) - logf(sd) - 0.91893853320467274178f;   // Normal.log_prob
    l -= logf(1.f - a * a + 1e-7f);
    lp += l;
  }
  logp[m] = lp;
}

// ---- SAC actor objective L = mean(alpha * logp - min(q1, q2))  (sac.py:222-236) -----------------------------------------
// dq_i = -(1/B) where q_i is the smaller one (1/2 each on ties: torch.minimum's backward).
// stats = {actor_loss, mean min_q, mean entropy (= -logp), mean(entropy - target_entropy)}.
__global__ void __launch_bounds__(256) sac_minq_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                                       const float* __restrict__ logp, const float* __restrict__ alpha,
                                                       float target_entropy, int B, float* __restrict__ dq1,
                                                       float* __restrict__ dq2, float* __restrict__ stats) {
  __shared__ float sm[9];
  float sl = 0.f, sq = 0.f, se = 0.f;
  const float inv = 1.f / (float)B, al = alpha[0];
  for (int b = threadIdx.x; b < B; b += 256) {
    const float a = q1[b], c = q2[b];
    const float mn = fminf(a, c);
    dq1[b] = a < c ? -inv : (a == c ? -0.5f * inv : 0.f);
    dq2[b] = c < a ? -inv : (a == c ? -0.5f * inv : 0.f);
    const float ent = -logp[b];
    sl += al * ent + mn;
    sq += mn;
    se += ent;
  }
  sl = block_sum256(sl, sm);
  sq = block_sum256(sq, sm);
  se = block_sum256(se, sm);
  if (threadIdx.x == 0) {
    stats[0] = -sl * inv;
    stats[1] = sq * inv;
    stats[2] = se * inv;
    stats[3] = se * inv - target_entropy;
  }
}

// d L / d(raw mu, raw log_std) from d L / d action (critic path, already carrying -1/B) and the alpha * logp term.
//   z = mu + std eps, a = tanh z, logp_j = -eps^2/2 - log std - c - log(1 - a^2 + 1e-7)
//   dL/dz   = da (1 - a^2) + (alpha/B) 2a (1 - a^2) / (1 - a^2 + 1e-7)
//   dL/dmu  = dL/dz [|raw_mu| <= 5];  dL/dstd = dL/dz eps - (alpha/B) / std;  dL/draw_ls = dL/dstd std (1 - tanh^2 raw_ls)
__global__ void sac_actor_bwd_kernel(const float* __restrict__ raw, int nout, const float* __restrict__ eps,
                                     const float* __restrict__ action, const float* __restrict__ da,
                                     const float* __restrict__ alpha, int B, int A, float* __restrict__ dout) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * A) return;
  const int m = i / A, j = i % A;
  const float ab = alpha[0] / (float)B;
  const float rmu = raw[(size_t)m * nout + j];
  const float t = tanhf(raw[(size_t)m * nout + A + j]);
  const float sd = expf(t);
  const float a = action[i];
  const float om = 1.f - a * a;
  const float gz = da[i] * om + ab * (2.f * a * om / (om + 1e-7f));
  dout[(size_t)m * nout + j] = (rmu >= -5.f && rmu <= 5.f) ? gz : 0.f;
  const float gs = gz * eps[i] - ab / sd;
  dout[(size_t)m * nout + A + j] = gs * sd * (1.f - t * t);
}

// ---- entropy temperature (sac.py:238-246): alpha := exp(log_alpha) BEFORE this learn's optimiser step ------------------
// alpha_loss = log_alpha * mean(entropy - target_entropy); d/dlog_alpha = that mean.
__global__ void sac_alpha_kernel(const float* __restrict__ log_alpha, const float* __restrict__ stats4,
                                 float* __restrict__ alpha, float* __restrict__ grad, float* __restrict__ alpha_loss) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const float la = log_alpha[0];
    alpha_loss[0] = la * stats4[3];
    alpha[0] = expf(la);
    if (grad) grad[0] = stats4[3];
  }
}

// ---- discrete-action SAC (SAC-Discrete, Christodoulou 2019, arXiv:1910.07207) --------------------------------------------
// One row of A <= SACD_MAX_A logits per thread, held in registers: every loop over actions is fully unrolled and guarded
// by `a < A`, so no per-thread array is indexed dynamically.  logpi = log_softmax(z) exactly (z - max - log sum exp),
// pi = exp(logpi).
constexpr int SACD_MAX_A = 18;   // the full Atari action set

__device__ __forceinline__ void sacd_log_softmax(const float* __restrict__ z, int A, float (&lp)[SACD_MAX_A]) {
  float mx = -INFINITY;
#pragma unroll
  for (int a = 0; a < SACD_MAX_A; ++a) if (a < A) { lp[a] = z[a]; mx = fmaxf(mx, lp[a]); }
  float s = 0.f;
#pragma unroll
  for (int a = 0; a < SACD_MAX_A; ++a) if (a < A) s += expf(lp[a] - mx);
  const float lse = mx + logf(s);
#pragma unroll
  for (int a = 0; a < SACD_MAX_A; ++a) if (a < A) lp[a] = lp[a] - lse;
}

// act: a ~ Categorical(pi) by inverse CDF on one uniform per row (u_in, or Philox(seed, stream_base + m, row_ctr[m]) with
// the row's counter advanced, so CUDA-graph replays draw fresh numbers); greedy: argmax pi, first index on ties.
__global__ void sacd_act_kernel(const float* __restrict__ z, int M, int A, const float* __restrict__ u_in, uint64_t seed,
                                uint64_t stream_base, long long* __restrict__ row_ctr, int greedy,
                                int64_t* __restrict__ action) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float lp[SACD_MAX_A];
  sacd_log_softmax(z + (size_t)m * A, A, lp);
  int pick = 0;
  if (greedy) {
    float best = -1.f;
#pragma unroll
    for (int a = 0; a < SACD_MAX_A; ++a)
      if (a < A) { const float p = expf(lp[a]); if (p > best) { best = p; pick = a; } }
  } else {
    float u;
    if (u_in) u = u_in[m];
    else u = jb_u01_float(jb_philox(seed, stream_base + (uint64_t)m, jb_next_row_ctr(row_ctr, m)).x);
    float tot = 0.f;
#pragma unroll
    for (int a = 0; a < SACD_MAX_A; ++a) if (a < A) tot += expf(lp[a]);
    const float target = u * tot;
    float c = 0.f;
    pick = A - 1;
    bool found = false;
#pragma unroll
    for (int a = 0; a < SACD_MAX_A; ++a)
      if (a < A && !found) { c += expf(lp[a]); if (target < c) { pick = a; found = true; } }
  }
  action[m] = pick;
}

// critics: V' = sum_a pi'(a) [min(nq1, nq2)(a) - alpha logpi'(a)]   (pi' from the actor on s', nq_i the target critics)
//          y = r + ((1 - d) gamma) V';  q_i = Q_i(s)[a_b];  loss_i = mean (q_i - y)^2
//          dq_i[b,k] = 2 (q_i - y) / B at k = a_b, 0 elsewhere;  stats = {loss1, loss2, max_b y}
__global__ void __launch_bounds__(256) sacd_critic_loss_kernel(
    const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ nq1, const float* __restrict__ nq2,
    const float* __restrict__ nz, const int64_t* __restrict__ action, const float* __restrict__ reward,
    const float* __restrict__ done, const float* __restrict__ alpha, int B, int A, float gamma, float* __restrict__ dq1,
    float* __restrict__ dq2, float* __restrict__ stats) {
  __shared__ float sm[9];
  float s1 = 0.f, s2 = 0.f, mx = -INFINITY;
  const float inv = 1.f / (float)B, al = alpha[0];
  for (int b = threadIdx.x; b < B; b += 256) {
    const size_t o = (size_t)b * A;
    float lp[SACD_MAX_A];
    sacd_log_softmax(nz + o, A, lp);
    float v = 0.f;
#pragma unroll
    for (int a = 0; a < SACD_MAX_A; ++a)
      if (a < A) v += expf(lp[a]) * (fminf(nq1[o + a], nq2[o + a]) - al * lp[a]);
    const float y = __fadd_rn(reward[b], __fmul_rn(__fmul_rn(1.f - done[b], gamma), v));
    mx = fmaxf(mx, y);
    const int k = (int)action[b];
    const float e1 = q1[o + k] - y, e2 = q2[o + k] - y;
    s1 += e1 * e1;
    s2 += e2 * e2;
    for (int a = 0; a < A; ++a) {
      dq1[o + a] = a == k ? 2.f * e1 * inv : 0.f;
      dq2[o + a] = a == k ? 2.f * e2 * inv : 0.f;
    }
  }
  s1 = block_sum256(s1, sm);
  s2 = block_sum256(s2, sm);
  mx = block_max256(mx, sm);
  if (threadIdx.x == 0) { stats[0] = s1 * inv; stats[1] = s2 * inv; stats[2] = mx; }
}

// actor, through the updated critics: m = min(q1, q2) over [B,A], f = alpha logpi - m, L_b = sum_a pi f,
// actor_loss = mean_b L_b, dz[b,k] = pi_k (f_k - L_b) / B.  H_b = -sum_a pi logpi.
// stats = {actor_loss, mean_b sum_a pi m, mean H, mean H - target_entropy}.
__global__ void __launch_bounds__(256) sacd_actor_kernel(const float* __restrict__ z, const float* __restrict__ q1,
                                                         const float* __restrict__ q2, const float* __restrict__ alpha,
                                                         float target_entropy, int B, int A, float* __restrict__ dz,
                                                         float* __restrict__ stats) {
  __shared__ float sm[9];
  float sl = 0.f, sq = 0.f, se = 0.f;
  const float inv = 1.f / (float)B, al = alpha[0];
  for (int b = threadIdx.x; b < B; b += 256) {
    const size_t o = (size_t)b * A;
    float lp[SACD_MAX_A], f[SACD_MAX_A];
    sacd_log_softmax(z + o, A, lp);
    float L = 0.f, mq = 0.f, H = 0.f;
#pragma unroll
    for (int a = 0; a < SACD_MAX_A; ++a)
      if (a < A) {
        const float p = expf(lp[a]), m = fminf(q1[o + a], q2[o + a]);
        f[a] = al * lp[a] - m;
        L += p * f[a];
        mq += p * m;
        H -= p * lp[a];
      }
#pragma unroll
    for (int a = 0; a < SACD_MAX_A; ++a)
      if (a < A) dz[o + a] = expf(lp[a]) * (f[a] - L) * inv;
    sl += L;
    sq += mq;
    se += H;
  }
  sl = block_sum256(sl, sm);
  sq = block_sum256(sq, sm);
  se = block_sum256(se, sm);
  if (threadIdx.x == 0) {
    stats[0] = sl * inv;
    stats[1] = sq * inv;
    stats[2] = se * inv;
    stats[3] = se * inv - target_entropy;
  }
}

}  // namespace

JB_API int jb_soft_update(float* target, const float* online, int64_t n, double tau, void* stream) {
  if (!target || !online || n <= 0) return JB_ERR_INVALID;
  soft_update_kernel<<<jb_grid_for(n, 1024), 256, 0, (cudaStream_t)stream>>>(target, online, (long long)n, (float)tau,
                                                                            (float)(1.0 - tau));
  return jb_check_launch();
}

JB_API int jb_tanh_act(const float* pre, const float* noise, int64_t n, float scale, float noise_clip, float out_clip,
                       float* out, void* stream) {
  if (!pre || !out || n <= 0) return JB_ERR_INVALID;
  tanh_act_kernel<<<jb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(pre, noise, (long long)n, scale, noise_clip, out_clip, out);
  return jb_check_launch();
}

JB_API int jb_tanh_bwd(const float* da, const float* a, int64_t n, float* dpre, void* stream) {
  if (!da || !a || !dpre || n <= 0) return JB_ERR_INVALID;
  tanh_bwd_kernel<<<jb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(da, a, (long long)n, dpre);
  return jb_check_launch();
}

JB_API int jb_ou_act(const float* pre, int M, int A, double* X, const double* normal, uint64_t seed, uint64_t stream_base,
                     long long* row_ctr, double theta, double mu, double sigma, int greedy, float* action, void* stream) {
  if (!pre || !action || M <= 0 || A <= 0 || (!greedy && !X)) return JB_ERR_INVALID;
  ou_act_kernel<<<jb_div_up(M, 128), 128, 0, (cudaStream_t)stream>>>(pre, M, A, X, normal, seed, stream_base, row_ctr, theta,
                                                                     mu, sigma, greedy, action);
  return jb_check_launch();
}

// kind 0: standard normals; kind 1: uniforms in [lo, hi).  Element pair p uses Philox(seed, stream + p, ctr + ctr_dev[0]);
// ctr_dev (device int64[1], may be NULL) is incremented afterwards so that a captured graph draws fresh numbers.
JB_API int jb_philox_fill(float* out, int64_t n, int kind, float lo, float hi, uint64_t seed, uint64_t stream_base,
                          uint64_t ctr, long long* ctr_dev, void* stream) {
  if (!out || n <= 0 || kind < 0 || kind > 1) return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  philox_fill_kernel<<<jb_div_up((n + 1) / 2, 256), 256, 0, s>>>(out, (long long)n, kind, lo, hi, seed, stream_base, ctr_dev, ctr);
  if (ctr_dev) bump_kernel<<<1, 1, 0, s>>>(ctr_dev);
  return jb_check_launch();
}

JB_API int jb_ac_critic_loss(const float* q1, const float* q2, const float* nq1, const float* nq2, const float* alpha,
                             const float* next_logp, const float* reward, const float* done, int B, float gamma,
                             float* dq1, float* dq2, float* stats, void* stream) {
  if (!q1 || !nq1 || !reward || !done || !dq1 || !stats || B <= 0 || (q2 && !dq2)) return JB_ERR_INVALID;
  critic_loss_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q1, q2, nq1, nq2, alpha, next_logp, reward, done, B, gamma, dq1, dq2, stats);
  return jb_check_launch();
}

JB_API int jb_ac_neg_mean(const float* q, int B, float* dq, float* stat, void* stream) {
  if (!q || !dq || !stat || B <= 0) return JB_ERR_INVALID;
  neg_mean_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q, B, dq, stat);
  return jb_check_launch();
}

JB_API int jb_sac_sample(const float* raw, int nout, const float* eps, int M, int A, float* action, float* logp,
                         void* stream) {
  if (!raw || !eps || !action || !logp || M <= 0 || A <= 0 || A > AC_MAX_A || nout < 2 * A) return JB_ERR_INVALID;
  sac_sample_kernel<<<jb_div_up(M, 128), 128, 0, (cudaStream_t)stream>>>(raw, nout, eps, M, A, action, logp);
  return jb_check_launch();
}

JB_API int jb_sac_minq(const float* q1, const float* q2, const float* logp, const float* alpha, float target_entropy,
                       int B, float* dq1, float* dq2, float* stats, void* stream) {
  if (!q1 || !q2 || !logp || !alpha || !dq1 || !dq2 || !stats || B <= 0) return JB_ERR_INVALID;
  sac_minq_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q1, q2, logp, alpha, target_entropy, B, dq1, dq2, stats);
  return jb_check_launch();
}

JB_API int jb_sac_actor_bwd(const float* raw, int nout, const float* eps, const float* action, const float* da,
                            const float* alpha, int B, int A, float* dout, void* stream) {
  if (!raw || !eps || !action || !da || !alpha || !dout || B <= 0 || A <= 0 || A > AC_MAX_A || nout != 2 * A)
    return JB_ERR_INVALID;
  sac_actor_bwd_kernel<<<jb_div_up((long long)B * A, 256), 256, 0, (cudaStream_t)stream>>>(raw, nout, eps, action, da, alpha, B, A, dout);
  return jb_check_launch();
}

JB_API int jb_sac_alpha(const float* log_alpha, const float* stats4, float* alpha, float* grad, float* alpha_loss,
                        void* stream) {
  if (!log_alpha || !stats4 || !alpha || !alpha_loss) return JB_ERR_INVALID;
  sac_alpha_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(log_alpha, stats4, alpha, grad, alpha_loss);
  return jb_check_launch();
}

JB_API int jb_sacd_act(const float* logits, int M, int A, const float* u, uint64_t seed, uint64_t stream_base,
                       long long* row_ctr, int greedy, int64_t* action, void* stream) {
  if (!logits || !action || M <= 0 || A <= 0 || A > SACD_MAX_A) return JB_ERR_INVALID;
  sacd_act_kernel<<<jb_div_up(M, 128), 128, 0, (cudaStream_t)stream>>>(logits, M, A, u, seed, stream_base, row_ctr, greedy,
                                                                       action);
  return jb_check_launch();
}

JB_API int jb_sacd_critic_loss(const float* q1, const float* q2, const float* nq1, const float* nq2, const float* next_logits,
                               const int64_t* action, const float* reward, const float* done, const float* alpha, int B,
                               int A, float gamma, float* dq1, float* dq2, float* stats, void* stream) {
  if (!q1 || !q2 || !nq1 || !nq2 || !next_logits || !action || !reward || !done || !alpha || !dq1 || !dq2 || !stats ||
      B <= 0 || A <= 0 || A > SACD_MAX_A)
    return JB_ERR_INVALID;
  sacd_critic_loss_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q1, q2, nq1, nq2, next_logits, action, reward, done, alpha, B,
                                                               A, gamma, dq1, dq2, stats);
  return jb_check_launch();
}

JB_API int jb_sacd_actor(const float* logits, const float* q1, const float* q2, const float* alpha, float target_entropy,
                         int B, int A, float* dlogits, float* stats4, void* stream) {
  if (!logits || !q1 || !q2 || !alpha || !dlogits || !stats4 || B <= 0 || A <= 0 || A > SACD_MAX_A) return JB_ERR_INVALID;
  sacd_actor_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(logits, q1, q2, alpha, target_entropy, B, A, dlogits, stats4);
  return jb_check_launch();
}
