// V-MPO minibatch loss (Song et al., ICLR 2020, arXiv:1909.12238) on the PPO rollout path: top-half advantage
// selection, temperature (eta) loss, psi-weighted policy loss, the decoupled KL trust regions with learned Lagrange
// multipliers (arXiv:1812.02256 for the Gaussian split) and the critic MSE, forward and backward on the narrow head
// outputs.  The row conventions (head layout, mu = clamp(mu_raw, -5, 5), sd = exp(tanh(log_std_raw)), atanh of the
// stored action) are PPO's, see ppo.cu / ppo_rowmath.cuh.
//
// Per minibatch of B rows (row b <-> rollout row idx[b]):
//   m      = lower median of adv (torch.median: element (B-1)//2 of the sorted values)
//   T      = {b : adv_b > m}, n = |T|;  z_b = adv_b / eta, M = max_T z, S = sum_T exp(z - M)
//   psi_b  = exp(z_b - M) / S                                    (detached)
//   L_pi   = -sum_T psi_b log pi(a_b | s_b)
//   L_eta  = eta eps_eta + eta (M + log S - log n)               (max-shifted log-mean-exp: no overflow at small eta)
//   L_alpha= sum_k mean_b[alpha_k (eps_k - sg KL_kb) + sg(alpha_k) KL_kb]   k = mu (discrete: the whole KL), sigma
//   L_v    = mean_b (v_b - ret_b)^2
// n = 0 (every advantage equals the median) gives L_pi = L_eta = 0 and zero gradients for them.
//
// Every CTA first reduces the minibatch-wide scalars (m by an exact radix select on order-preserving uint32 keys,
// then M, n, S, sum psi*(M - z)) over all B rows in a fixed order, then produces its own rows' gradients; a one-thread
// launch folds the per-CTA partials in CTA order.  No atomics: bit-reproducible run to run, for any B.
#include "common.cuh"
#include "ppo_rowmath.cuh"

namespace {

using jbppo::MAX_A;
using jbppo::MAX_A_DISC;
using jbppo::log_softmax_row;
using jbppo::atanh_clamped;
using jbppo::block_sum;

constexpr int VMPO_THREADS = 256;
constexpr int VMPO_SCALARS = 8;        // stats[8..15]: the minibatch scalars CTA 0 publishes for the finalize launch
constexpr int VMPO_PARTIALS = 16;      // stats[16 + 4*cta ..]: per-CTA partial sums

// float -> uint32 with the same order (negative floats reversed, sign bit flipped for the rest)
__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__device__ __forceinline__ float row_adv(const float* __restrict__ adv, const int32_t* __restrict__ idx, int b) {
  return adv[idx ? idx[b] : b];
}

// Exact k-th smallest (0-based) of the B advantages: four-bit radix select from the top digit down.  Each pass counts,
// per warp and per digit, the candidates (keys matching the digits chosen so far) by ballot; thread d < 16 sums digit d
// over the warps and thread 0 walks the 16 totals to the digit that holds rank k.
__device__ uint32_t select_key(const float* __restrict__ adv, const int32_t* __restrict__ idx, int B, int k,
                               int* s_cnt /*[32*16]*/, int* s_tot /*[16]*/, uint32_t* s_sel /*[3]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  uint32_t prefix = 0u, mask = 0u;
  for (int shift = 28; shift >= 0; shift -= 4) {
    int cnt = 0;
    for (int base = warp * 32; base < B; base += blockDim.x) {      // warp-uniform trip count: ballots stay convergent
      const int b = base + lane;
      const uint32_t key = b < B ? order_key(row_adv(adv, idx, b)) : 0u;
      const bool cand = b < B && (key & mask) == prefix;
      const uint32_t dig = (key >> shift) & 15u;
#pragma unroll
      for (uint32_t d = 0; d < 16; ++d) {
        const int c = __popc(__ballot_sync(0xffffffffu, cand && dig == d));
        if (lane == (int)d) cnt += c;
      }
    }
    if (lane < 16) s_cnt[warp * 16 + lane] = cnt;
    __syncthreads();
    if (threadIdx.x < 16) {
      int t = 0;
      for (int w = 0; w < nw; ++w) t += s_cnt[w * 16 + threadIdx.x];
      s_tot[threadIdx.x] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int d = 0;
      while (d < 15 && k >= s_tot[d]) { k -= s_tot[d]; ++d; }
      s_sel[0] = prefix | ((uint32_t)d << shift);
      s_sel[1] = (uint32_t)k;
    }
    __syncthreads();
    prefix = s_sel[0];
    k = (int)s_sel[1];
    mask |= 15u << shift;
    __syncthreads();                   // s_sel is rewritten by the next pass
  }
  return prefix;
}

struct Mult { float eta, alpha_mu, alpha_sigma; };

// Per-row forward + backward.  w: the row's psi (0 outside the top set).  Writes d loss / d out into g[0..nout) and
// returns the row's log pi, KL_mu (discrete: the KL), KL_sigma and (v - ret)^2.
template <bool CONT, int NA>
__device__ __forceinline__ void vmpo_row(const float* __restrict__ o, const float* __restrict__ oo, int A, int a_disc,
                                         const float* __restrict__ a_cont, float ret, float w, Mult mu_, float invB,
                                         float* __restrict__ g, float& logpi, float& kl_mu, float& kl_sigma, float& sq) {
  const float v = o[CONT ? 2 * A : A];
  const float dv = v - ret;
  sq = dv * dv;
  g[CONT ? 2 * A : A] = 2.f * dv * invB;
  kl_sigma = 0.f;
  if constexpr (!CONT) {
    float lg[NA], lgo[NA], lsm[NA], lsmo[NA];
#pragma unroll
    for (int a = 0; a < NA; ++a) { lg[a] = a < A ? o[a] : 0.f; lgo[a] = a < A ? oo[a] : 0.f; }
    log_softmax_row<NA>(lg, A, lsm);
    log_softmax_row<NA>(lgo, A, lsmo);
    float la = 0.f, kl = 0.f, so = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      if (a < A) {
        if (a == a_disc) la = lsm[a];
        const float po = expf(lsmo[a]);
        kl += po * (lsmo[a] - lsm[a]);
        so += po;
      }
    }
    logpi = la;
    kl_mu = kl;
    const float ck = mu_.alpha_mu * invB;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      if (a < A) {
        const float p = expf(lsm[a]);
        const float dpi = -w * ((a == a_disc ? 1.f : 0.f) - p);         // d(-w log softmax_a) / d logit
        const float dkl = p * so - expf(lsmo[a]);                       // d KL / d logit
        g[a] = dpi + ck * dkl;
      }
    }
  } else {
    const float log_sqrt_2pi = 0.9189385332046727f;
    const float cm = mu_.alpha_mu * invB, cs = mu_.alpha_sigma * invB;
    float lp = 0.f, km = 0.f, ks = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      if (a < A) {
        const float omu = o[a], ols = o[A + a];
        const float mu = fminf(fmaxf(omu, -5.f), 5.f);
        const float ls = tanhf(ols);
        const float sd = expf(ls);
        const float mu_o = fminf(fmaxf(oo[a], -5.f), 5.f);
        const float ls_o = tanhf(oo[A + a]);
        const float sd_o = expf(ls_o);
        const float z = atanh_clamped(a_cont[a]);
        const float d = z - mu;
        // three reciprocals instead of a division per term: the IEEE divide's slow-path call would spill here
        const float iv = 1.f / (sd * sd), ivo = 1.f / (sd_o * sd_o), isd = 1.f / sd;
        lp += -0.5f * (d * d) * iv - ls - log_sqrt_2pi;                  // log sd = tanh(log_std_raw)
        const float dm = mu - mu_o;
        km += 0.5f * (dm * dm) * ivo;
        const float r = (sd_o * sd_o) * iv;                               // sd_old^2 / sd^2
        ks += 0.5f * (r - 1.f + 2.f * (ls - ls_o));
        // d/dmu and d/dsd of  -w log pi + alpha_mu/B KL_mu + alpha_sigma/B KL_sigma
        const float gmu = -w * d * iv + cm * dm * ivo;
        const float gsd = (-w * (d * d * iv - 1.f) + cs * (1.f - r)) * isd;
        const float in_mu = (omu >= -5.f && omu <= 5.f) ? 1.f : 0.f;
        g[a] = gmu * in_mu;
        g[A + a] = gsd * sd * (1.f - ls * ls);
      }
    }
    logpi = lp;
    kl_mu = km;
    kl_sigma = ks;
  }
}

// NA: compile-time bound on A, as in ppo_loss_kernel (min-blocks 1 for the 18-wide discrete rows).
template <bool CONT, int NA>
__global__ void __launch_bounds__(VMPO_THREADS, NA > MAX_A ? 1 : 0)
vmpo_loss_kernel(const float* __restrict__ out, const float* __restrict__ out_old, const int32_t* __restrict__ idx,
                 const void* __restrict__ action_all, const float* __restrict__ adv_all, const float* __restrict__ ret_all,
                 int B, int A, int nout, const float* __restrict__ mult, float* __restrict__ dout,
                 float* __restrict__ stats) {
  __shared__ int s_cnt[32 * 16];
  __shared__ int s_tot[16];
  __shared__ uint32_t s_sel[2];
  __shared__ float sred[4 * 32];
  const Mult ml{mult[0], mult[1], mult[2]};
  const float eta = ml.eta;

  // ---- phase 1 (every CTA, whole minibatch): the lower median -------------------------------------------------
  const float m = key_value(select_key(adv_all, idx, B, (B - 1) / 2, s_cnt, s_tot, s_sel));

  // ---- phase 2: M and n, then S and sum exp(z - M) (M - z), in a fixed order ---------------------------------
  float zmax = -INFINITY, cnt[1] = {0.f};
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const float a = row_adv(adv_all, idx, b);
    if (a > m) { zmax = fmaxf(zmax, a / eta); cnt[0] += 1.f; }
  }
  zmax = jb_warp_max(zmax);
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = zmax;
  __syncthreads();
  float M = sred[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) M = fmaxf(M, sred[w]);
  __syncthreads();
  block_sum<1, VMPO_THREADS / 32>(cnt, sred);
  const float n = cnt[0];
  float es[2] = {0.f, 0.f};
  if (n > 0.f) {
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
      const float a = row_adv(adv_all, idx, b);
      if (a > m) { const float z = a / eta; const float e = expf(z - M); es[0] += e; es[1] += e * (M - z); }
    }
  }
  block_sum<2, VMPO_THREADS / 32>(es, sred);
  const float S = es[0];

  // ---- phase 3: this CTA's rows ---------------------------------------------------------------------------------
  const float invB = 1.0f / (float)B;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float part[4] = {0.f, 0.f, 0.f, 0.f};       // sum psi log pi, sum KL_mu, sum KL_sigma, sum (v - ret)^2
  if (b < B) {
    const int r = idx ? idx[b] : b;
    const float a = adv_all[r];
    const float w = a > m ? expf(a / eta - M) / S : 0.f;
    float logpi, km, ks, sq;
    if constexpr (CONT)
      vmpo_row<true, NA>(out + (size_t)b * nout, out_old + (size_t)r * nout, A, 0, (const float*)action_all + (size_t)r * A,
                         ret_all[r], w, ml, invB, dout + (size_t)b * nout, logpi, km, ks, sq);
    else
      vmpo_row<false, NA>(out + (size_t)b * nout, out_old + (size_t)r * nout, A, ((const int32_t*)action_all)[r], nullptr,
                          ret_all[r], w, ml, invB, dout + (size_t)b * nout, logpi, km, ks, sq);
    part[0] = w > 0.f ? w * logpi : 0.f;
    part[1] = km; part[2] = ks; part[3] = sq;
  }
  block_sum<4, VMPO_THREADS / 32>(part, sred);
  if (threadIdx.x == 0) {
    float* sp = stats + VMPO_PARTIALS + 4 * blockIdx.x;
    sp[0] = part[0]; sp[1] = part[1]; sp[2] = part[2]; sp[3] = part[3];
    if (blockIdx.x == 0) {
      float* sc = stats + VMPO_SCALARS;
      sc[0] = m; sc[1] = n; sc[2] = M; sc[3] = S; sc[4] = es[1];
    }
  }
}

// Folds the per-CTA partials in CTA order into the losses, the multiplier gradients and the stats:
//   stats[0..7] = L_pi, L_v, L_eta, L_alpha, mean KL_mu, mean KL_sigma, n, m
//   dmult[0..2] = d loss / d (eta, alpha_mu, alpha_sigma);  acc[0..3] += L_pi, L_v, L_eta, L_alpha;  acc[4] += 1
__global__ void vmpo_finalize_kernel(float* __restrict__ stats, int n_cta, int B, int cont, const float* __restrict__ mult,
                                     float eps_eta, float eps_alpha_mu, float eps_alpha_sigma, float* __restrict__ dmult,
                                     float* __restrict__ acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float wl = 0.f, km = 0.f, ks = 0.f, sq = 0.f;
  for (int k = 0; k < n_cta; ++k) {
    const float* sp = stats + VMPO_PARTIALS + 4 * k;
    wl += sp[0]; km += sp[1]; ks += sp[2]; sq += sp[3];
  }
  const float invB = 1.0f / (float)B;
  const float* sc = stats + VMPO_SCALARS;
  const float m = sc[0], n = sc[1], M = sc[2], S = sc[3], sdz = sc[4];
  const float eta = mult[0], alpha_mu = mult[1], alpha_sigma = mult[2];
  km *= invB; ks *= invB;
  float l_eta = 0.f, d_eta = 0.f;
  if (n > 0.f) {
    const float lme = M + logf(S) - logf(n);          // log mean_T exp(adv / eta)
    l_eta = eta * eps_eta + eta * lme;
    // lme - sum psi adv / eta = log S - log n + sum psi (M - z): no cancellation of two ~M-sized terms at small eta
    d_eta = eps_eta + (logf(S) - logf(n)) + sdz / S;
  }
  float l_alpha = alpha_mu * (eps_alpha_mu - km) + alpha_mu * km;
  if (cont) l_alpha += alpha_sigma * (eps_alpha_sigma - ks) + alpha_sigma * ks;
  dmult[0] = d_eta;
  dmult[1] = eps_alpha_mu - km;
  dmult[2] = cont ? eps_alpha_sigma - ks : 0.f;
  stats[0] = -wl;
  stats[1] = sq * invB;
  stats[2] = l_eta;
  stats[3] = l_alpha;
  stats[4] = km; stats[5] = ks; stats[6] = n; stats[7] = m;
  if (acc) {
    acc[0] += stats[0]; acc[1] += stats[1]; acc[2] += stats[2]; acc[3] += stats[3]; acc[4] += 1.f;
  }
}

__global__ void vmpo_clamp_kernel(float* __restrict__ mult, float min_eta, float min_alpha_mu, float min_alpha_sigma) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    mult[0] = fmaxf(mult[0], min_eta);
    mult[1] = fmaxf(mult[1], min_alpha_mu);
    mult[2] = fmaxf(mult[2], min_alpha_sigma);
  }
}

}  // namespace

JB_API int jb_vmpo_loss(int continuous, const float* out, const float* out_old, const int32_t* idx, const void* action,
                        const float* adv, const float* ret, int B, int A, int nout, const float* mult, float eps_eta,
                        float eps_alpha_mu, float eps_alpha_sigma, float* dout, float* dmult, float* stats, float* acc,
                        void* stream) {
  if (!out || !out_old || !action || !adv || !ret || !mult || !dout || !dmult || !stats) return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || A > (continuous ? MAX_A : MAX_A_DISC) || nout != (continuous ? 2 * A + 1 : A + 1)) return JB_ERR_INVALID;
  const int n_cta = jb_div_up(B, VMPO_THREADS);
  cudaStream_t s = (cudaStream_t)stream;
  if (continuous) vmpo_loss_kernel<true, MAX_A><<<n_cta, VMPO_THREADS, 0, s>>>(out, out_old, idx, action, adv, ret, B, A, nout, mult, dout, stats);
  else if (A <= MAX_A) vmpo_loss_kernel<false, MAX_A><<<n_cta, VMPO_THREADS, 0, s>>>(out, out_old, idx, action, adv, ret, B, A, nout, mult, dout, stats);
  else vmpo_loss_kernel<false, MAX_A_DISC><<<n_cta, VMPO_THREADS, 0, s>>>(out, out_old, idx, action, adv, ret, B, A, nout, mult, dout, stats);
  vmpo_finalize_kernel<<<1, 32, 0, s>>>(stats, n_cta, B, continuous, mult, eps_eta, eps_alpha_mu, eps_alpha_sigma, dmult, acc);
  return jb_check_launch();
}

JB_API int jb_vmpo_clamp(float* mult, float min_eta, float min_alpha_mu, float min_alpha_sigma, void* stream) {
  if (!mult) return JB_ERR_INVALID;
  vmpo_clamp_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(mult, min_eta, min_alpha_mu, min_alpha_sigma);
  return jb_check_launch();
}
