// Quantile-regression learners (QR-DQN, arXiv:1710.10044; IQN, arXiv:1806.06923): the quantile Huber loss with
// its closed-form gradient, the per-action quantile means, and IQN's sampled-fraction embedding.
//
// Layouts.  A quantile tensor holds, per sample, A actions x N quantiles at element offset b*A*N + a*sa + i*sq:
// QR-DQN's [B, A, K] head output is (sa, sq) = (K, 1), IQN's [B, N, A] output is (1, A).
//
// Loss (kappa = 1), with y_j = r + ((1 - d) gamma) theta'_j(s', a*) and u_ij = y_j - theta_i(s, a):
//   rho_ij = |tau_i - 1{u_ij < 0}| h(u_ij),  h = smooth_l1,  loss = (1/B) sum_b (1/N') sum_j sum_i rho_ij
//   d loss / d theta_i = -(1/(B N')) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -1, 1)  (0 on non-taken actions)
// a* = argmax_a mean_j theta'_j(s', a), first index on ties.  Every sum runs in a fixed order (no atomics), and the
// batch statistics are folded by one thread, so a learn() is bit-reproducible.  M-IQN's loss (arXiv:2007.14430) runs the
// same per-sample Huber loop on Munchausen targets (munchausen.cuh), and Rainbow-IQN's (arXiv:1908.04683) on double-Q
// n-step targets with per-sample importance weights and new priorities.
#include "common.cuh"
#include "munchausen.cuh"
#include "philox.cuh"
#include "value_loss.cuh"

namespace {

constexpr int QMAXN = 256;     // quantiles per pass (N, N')
constexpr int QMAXA = 18;      // ALE's full action set
constexpr int QT = 256;        // threads per CTA of the loss kernel: one predicted quantile each
static_assert(QMAXA == MUNCHAUSEN_MAX_A, "M-IQN's pi' / tau logpi' rows hold every action");

// mean of x[0], x[sq], ..., x[(n-1) sq] over one warp: lane-strided partial sums, then the butterfly.  The loss kernel
// and jb_quantile_mean share it, so a* / max_Q and act()'s greedy action come from bit-identical means.
__device__ __forceinline__ float warp_mean(const float* __restrict__ x, int sq, int n, int lane) {
  float s = 0.f;
  for (int j = lane; j < n; j += 32) s += x[(size_t)j * sq];
  return jb_warp_sum(s) / (float)n;
}

// The quantile Huber loss of one sample, given its targets s_y[0, Np) and fractions s_tau[0, N) in shared memory: thread
// i < N owns predicted quantile i of the taken action a_t and sums over j in order.  Writes the sample's dpred row db (0 on
// every other action) and returns (1/Np) sum_j sum_i rho_ij on thread 0 (a fixed-order tree over the warps).
__device__ __forceinline__ float quantile_huber(const float* __restrict__ pb, int p_sa, int p_sq, const float* s_y,
                                                const float* s_tau, float* s_red, int A, int N, int Np, int a_t, float gcoef,
                                                float* __restrict__ db) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float li = 0.f;
  if (tid < N) {
    const float th = pb[(size_t)a_t * p_sa + (size_t)tid * p_sq];
    const float t = s_tau[tid], tc = 1.f - t;
    float g = 0.f;
    for (int j = 0; j < Np; ++j) {
      const float u = s_y[j] - th, au = fabsf(u);
      const float w = u < 0.f ? tc : t;
      li += w * (au < 1.f ? 0.5f * u * u : au - 0.5f);
      g += w * fminf(fmaxf(u, -1.f), 1.f);
    }
    db[(size_t)a_t * p_sa + (size_t)tid * p_sq] = -g * gcoef;
  }
  for (int e = tid; e < A * N; e += QT) {
    const int a = e / N, i = e - a * N;
    if (a != a_t) db[(size_t)a * p_sa + (size_t)i * p_sq] = 0.f;
  }
  li = jb_warp_sum(li);
  if (lane == 0) s_red[warp] = li;
  __syncthreads();
  float s = 0.f;
  if (tid == 0)
    for (int w = 0; w < QT / 32; ++w) s += s_red[w];
  return s / (float)Np;
}

__global__ void __launch_bounds__(QT)
quantile_loss_kernel(const float* __restrict__ pred, int p_sa, int p_sq, const float* __restrict__ nxt, int t_sa, int t_sq,
                     const float* __restrict__ tau, int tau_stride, const void* __restrict__ action, int action_kind,
                     const float* __restrict__ reward, const float* __restrict__ done, int A, int N, int Np, float gamma,
                     float gcoef, float* __restrict__ dpred, float* __restrict__ loss_out, int32_t* __restrict__ a_star_out,
                     float* __restrict__ partial /*[B][2]*/) {
  __shared__ float s_y[QMAXN], s_tau[QMAXN], s_qt[QMAXA], s_qo[QMAXA], s_red[QT / 32];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* pb = pred + (size_t)b * A * N;
  const float* tb = nxt + (size_t)b * A * Np;
  for (int a = warp; a < A; a += QT / 32) {
    const float qt = warp_mean(tb + (size_t)a * t_sa, t_sq, Np, lane);
    const float qo = warp_mean(pb + (size_t)a * p_sa, p_sq, N, lane);
    if (lane == 0) { s_qt[a] = qt; s_qo[a] = qo; }
  }
  for (int i = tid; i < N; i += QT) s_tau[i] = tau[(size_t)b * tau_stride + i];
  __syncthreads();
  int a_star = 0;
  float best = s_qt[0], maxq = s_qo[0];
  for (int a = 1; a < A; ++a) {
    if (s_qt[a] > best) { best = s_qt[a]; a_star = a; }
    maxq = fmaxf(maxq, s_qo[a]);
  }
  const float r = reward[b], nd = __fmul_rn(__fadd_rn(1.f, -done[b]), gamma);
  for (int j = tid; j < Np; j += QT) s_y[j] = __fadd_rn(r, __fmul_rn(nd, tb[(size_t)a_star * t_sa + (size_t)j * t_sq]));
  const int a_t = read_action(action, action_kind, b);
  __syncthreads();
  const float lb = quantile_huber(pb, p_sa, p_sq, s_y, s_tau, s_red, A, N, Np, a_t, gcoef, dpred + (size_t)b * A * N);
  if (tid == 0) {
    loss_out[b] = lb;
    if (a_star_out) a_star_out[b] = a_star;
    partial[2 * b] = lb;
    partial[2 * b + 1] = maxq;
  }
}

// M-IQN (arXiv:2007.14430) on the [B, N, A] layout: q'(s, .) and q'(s', .) are the per-action means of the target
// network's quantiles on s (Nc fractions) and on s' (Np fractions); thread 0 forms the Munchausen scalars (munchausen.cuh)
// and y_j = (r + bonus) + ((1 - d) gamma) sum_a pi'(a) (theta'_j(s', a) - tau logpi'(a|s')), actions ascending.  The loss is
// quantile_huber's, unchanged.
__global__ void __launch_bounds__(QT)
munchausen_quantile_loss_kernel(const float* __restrict__ pred, const float* __restrict__ nxt, const float* __restrict__ cur,
                                const float* __restrict__ tau, int tau_stride, const void* __restrict__ action,
                                int action_kind, const float* __restrict__ reward, const float* __restrict__ done, int A,
                                int N, int Np, int Nc, float gamma, float m_alpha, float m_tau, float l0, float gcoef,
                                float* __restrict__ dpred, float* __restrict__ partial /*[B][2]*/) {
  __shared__ float s_y[QMAXN], s_tau[QMAXN], s_q[3][QMAXA], s_pi[QMAXA], s_tlp[QMAXA], s_red[QT / 32], s_bonus;
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* pb = pred + (size_t)b * A * N;
  const float* tb = nxt + (size_t)b * A * Np;
  // s_q rows: the online mean on s (for max_Q), the target means on s' and on s
  for (int e = warp; e < 3 * A; e += QT / 32) {
    const int k = e / A, a = e - k * A;
    const int n = k == 0 ? N : (k == 1 ? Np : Nc);
    const float* x = k == 0 ? pb : (k == 1 ? tb : cur + (size_t)b * A * Nc);
    const float v = warp_mean(x + a, A, n, lane);
    if (lane == 0) s_q[k][a] = v;
  }
  for (int i = tid; i < N; i += QT) s_tau[i] = tau[(size_t)b * tau_stride + i];
  const int a_t = read_action(action, action_kind, b);
  __syncthreads();
  if (tid == 0) s_bonus = munchausen_row(s_q[2], s_q[1], A, a_t, m_tau, m_alpha, l0, s_pi, s_tlp);
  __syncthreads();
  const float base = __fadd_rn(reward[b], s_bonus), nd = __fmul_rn(__fadd_rn(1.f, -done[b]), gamma);
  for (int j = tid; j < Np; j += QT) {
    const float* tj = tb + (size_t)j * A;
    float v = 0.f;
    for (int a = 0; a < A; ++a) v += s_pi[a] * (tj[a] - s_tlp[a]);
    s_y[j] = __fadd_rn(base, __fmul_rn(nd, v));
  }
  __syncthreads();
  const float lb = quantile_huber(pb, 1, A, s_y, s_tau, s_red, A, N, Np, a_t, gcoef, dpred + (size_t)b * A * N);
  if (tid == 0) {
    float maxq = s_q[0][0];
    for (int a = 1; a < A; ++a) maxq = fmaxf(maxq, s_q[0][a]);
    partial[2 * b] = lb;
    partial[2 * b + 1] = maxq;
  }
}

// Rainbow-IQN (arXiv:1908.04683) on the [B, N, A] layout: a* = argmax_a mean_j next_online[b, j, a] (double-Q, first index
// on ties), the n-step target y_j = fold_{s = n-1 .. 0} (r_s + ((1 - d_s) gamma) y) from y = next_target[b, j, a*] in c51.cu's
// float order, and quantile_huber, unchanged, with the sample's own IS weight in gcoef = w_b / (B Np).  loss_out holds the
// unweighted L_b, prio L_b^alpha; partial[b] = {w_b L_b, max_a mean_i pred, max pred, min pred}.
__global__ void __launch_bounds__(QT)
rainbow_iqn_loss_kernel(const float* __restrict__ pred, const float* __restrict__ next_online,
                        const float* __restrict__ next_target, const float* __restrict__ tau, const void* __restrict__ action,
                        int action_kind, const float* __restrict__ reward, const float* __restrict__ done,
                        const double* __restrict__ weights, int B, int A, int N, int Nn, int Np, int n_step, float gamma,
                        float alpha, float* __restrict__ dpred, float* __restrict__ loss_out, double* __restrict__ prio,
                        int32_t* __restrict__ a_star_out, float* __restrict__ partial /*[B][4]*/) {
  __shared__ float s_y[QMAXN], s_tau[QMAXN], s_qn[QMAXA], s_qo[QMAXA], s_red[QT / 32], s_mx[QT / 32], s_mn[QT / 32];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* pb = pred + (size_t)b * A * N;
  const float* ob = next_online + (size_t)b * A * Nn;
  const float* tb = next_target + (size_t)b * A * Np;
  // rows 0 .. A-1: the online means on s (max_Q); rows A .. 2A-1: the online means on s' (a*)
  for (int e = warp; e < 2 * A; e += QT / 32) {
    const int k = e / A, a = e - k * A;
    const float v = k == 0 ? warp_mean(pb + a, A, N, lane) : warp_mean(ob + a, A, Nn, lane);
    if (lane == 0) (k == 0 ? s_qo : s_qn)[a] = v;
  }
  float mx = -INFINITY, mn = INFINITY;
  for (int e = tid; e < A * N; e += QT) { const float v = pb[e]; mx = fmaxf(mx, v); mn = fminf(mn, v); }
  mx = jb_warp_max(mx);
  mn = jb_warp_min(mn);
  if (lane == 0) { s_mx[warp] = mx; s_mn[warp] = mn; }
  for (int i = tid; i < N; i += QT) s_tau[i] = tau[(size_t)b * N + i];
  __syncthreads();
  const int a_star = first_argmax(s_qn, A);
  const float* rr = reward + (size_t)b * n_step;
  const float* dr = done + (size_t)b * n_step;
  for (int j = tid; j < Np; j += QT) s_y[j] = nstep_fold(tb[(size_t)j * A + a_star], rr, dr, n_step, gamma);
  const int a_t = read_action(action, action_kind, b);
  const double w = weights ? weights[b] : 1.0;
  const float gcoef = (float)(w / ((double)B * (double)Np));
  __syncthreads();
  const float lb = quantile_huber(pb, 1, A, s_y, s_tau, s_red, A, N, Np, a_t, gcoef, dpred + (size_t)b * A * N);
  if (tid == 0) {
    float maxq = s_qo[0];
    for (int a = 1; a < A; ++a) maxq = fmaxf(maxq, s_qo[a]);
    for (int k = 1; k < QT / 32; ++k) { mx = fmaxf(mx, s_mx[k]); mn = fminf(mn, s_mn[k]); }
    loss_out[b] = lb;
    if (prio) prio[b] = pow((double)lb, (double)alpha);
    if (a_star_out) a_star_out[b] = a_star;
    partial[4 * b] = (float)(w * (double)lb);
    partial[4 * b + 1] = maxq;
    partial[4 * b + 2] = mx;
    partial[4 * b + 3] = mn;
  }
}

__global__ void quantile_mean_kernel(const float* __restrict__ x, int sa, int sq, int M, int A, int N, float* __restrict__ q) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= (long long)M * A) return;
  const long long m = row / A;
  const int a = (int)(row - m * A);
  const float v = warp_mean(x + (size_t)m * A * N + (size_t)a * sa, sq, N, lane);
  if (lane == 0) q[row] = v;
}

}  // namespace

JB_API int jb_quantile_loss(const float* pred, int p_sa, int p_sq, const float* next_target, int t_sa, int t_sq,
                            const float* tau, int tau_stride, const void* action, int action_kind, const float* reward,
                            const float* done, int B, int A, int N, int Np, float gamma, float* dpred, float* loss,
                            int32_t* a_star, float* stats, float* scratch, void* stream) {
  if (!pred || !next_target || !tau || !action || !reward || !done || !dpred || !loss || !stats || !scratch)
    return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || A > QMAXA || N <= 0 || N > QMAXN || Np <= 0 || Np > QMAXN || tau_stride < 0 ||
      action_kind < 0 || action_kind > 2)
    return JB_ERR_INVALID;
  const float gcoef = (float)(1.0 / ((double)B * (double)Np));
  cudaStream_t s = (cudaStream_t)stream;
  quantile_loss_kernel<<<B, QT, 0, s>>>(pred, p_sa, p_sq, next_target, t_sa, t_sq, tau, tau_stride, action, action_kind,
                                        reward, done, A, N, Np, gamma, gcoef, dpred, loss, a_star, scratch);
  loss_maxq_finalize_kernel<<<1, 32, 0, s>>>(scratch, B, stats);
  return jb_check_launch();
}

JB_API int jb_munchausen_quantile_loss(const float* pred, const float* next_target, const float* cur_target, const float* tau,
                                       int tau_stride, const void* action, int action_kind, const float* reward,
                                       const float* done, int B, int A, int N, int Np, int Nc, float gamma, float m_alpha,
                                       float m_tau, float l0, float* dpred, float* stats, float* scratch, void* stream) {
  if (!pred || !next_target || !cur_target || !tau || !action || !reward || !done || !dpred || !stats || !scratch)
    return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || A > QMAXA || N <= 0 || N > QMAXN || Np <= 0 || Np > QMAXN || Nc <= 0 || Nc > QMAXN ||
      tau_stride < 0 || action_kind < 0 || action_kind > 2 || !(m_tau > 0.f) || !(l0 <= 0.f))
    return JB_ERR_INVALID;
  const float gcoef = (float)(1.0 / ((double)B * (double)Np));
  cudaStream_t s = (cudaStream_t)stream;
  munchausen_quantile_loss_kernel<<<B, QT, 0, s>>>(pred, next_target, cur_target, tau, tau_stride, action, action_kind,
                                                   reward, done, A, N, Np, Nc, gamma, m_alpha, m_tau, l0, gcoef, dpred,
                                                   scratch);
  loss_maxq_finalize_kernel<<<1, 32, 0, s>>>(scratch, B, stats);
  return jb_check_launch();
}

JB_API int jb_rainbow_iqn_loss(const float* pred, const float* next_online, const float* next_target, const float* tau,
                               const void* action, int action_kind, const float* reward, const float* done,
                               const double* weights, int B, int A, int N, int Nn, int Np, int n_step, float gamma,
                               float alpha, float* dpred, float* loss, double* prio, int32_t* a_star, float* stats,
                               float* scratch, void* stream) {
  if (!pred || !next_online || !next_target || !tau || !action || !reward || !done || !dpred || !loss || !stats || !scratch)
    return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || A > QMAXA || N <= 0 || N > QMAXN || Nn <= 0 || Nn > QMAXN || Np <= 0 || Np > QMAXN ||
      n_step < 1 || action_kind < 0 || action_kind > 2)
    return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  rainbow_iqn_loss_kernel<<<B, QT, 0, s>>>(pred, next_online, next_target, tau, action, action_kind, reward, done, weights, B,
                                           A, N, Nn, Np, n_step, gamma, alpha, dpred, loss, prio, a_star, scratch);
  loss_logits_finalize_kernel<<<1, 32, 0, s>>>(scratch, B, B, stats);
  return jb_check_launch();
}

JB_API int jb_quantile_mean(const float* x, int sa, int sq, int M, int A, int N, float* q, void* stream) {
  if (!x || !q || M <= 0 || A <= 0 || N <= 0) return JB_ERR_INVALID;
  quantile_mean_kernel<<<jb_div_up((long long)M * A * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, sa, sq, M, A, N, q);
  return jb_check_launch();
}

// ------------------------------------------------------------------------------------------------ IQN embedding --
namespace {

// tau[e] = lo + (hi - lo) u_e for e < n, u from Philox(seed, stream_id, ctr[0] + e / 4) word e % 4; the counter is
// read here and advanced by tau_advance_kernel after every element has been drawn.
__global__ void iqn_tau_kernel(float* __restrict__ tau, long long n, float lo, float hi, uint64_t seed, uint64_t stream_id,
                               const long long* __restrict__ ctr) {
  const long long blk = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (blk * 4 >= n) return;
  const jb_philox4 r = jb_philox(seed, stream_id, (uint64_t)ctr[0] + (uint64_t)blk);
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  const float span = hi - lo;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const long long e = blk * 4 + k;
    if (e < n) {
      float v = lo + span * jb_u01_float(w[k]);
      if (v >= hi) v = nextafterf(hi, lo);          // keep the half-open range when span * u rounds up to span
      tau[e] = v;
    }
  }
}

__global__ void tau_advance_kernel(long long* __restrict__ ctr, long long blocks) { ctr[0] += blocks; }

// c[r, i] = cos(pi i tau[r]) for i < E
__global__ void iqn_cos_kernel(const float* __restrict__ tau, long long rows, int E, float* __restrict__ c) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows * E) return;
  const long long r = e / E;
  const int i = (int)(e - r * E);
  c[e] = cospif((float)i * tau[r]);
}

// z[b, n, :] = psi[b, :] * phi[b, n, :]
__global__ void iqn_mul_fwd_kernel(const float* __restrict__ psi, const float* __restrict__ phi, int N, int D,
                                   long long total, float* __restrict__ z) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long row = e / D;
    const int d = (int)(e - row * D);
    z[e] = psi[(row / N) * D + d] * phi[e];
  }
}

// One thread per (b, d): dpsi[b, d] = 1{psi > 0} sum_n dz[b, n, d] phi[b, n, d] (n ascending) and
// dpre[b, n, d] = dz[b, n, d] psi[b, d] 1{phi[b, n, d] > 0}.
__global__ void iqn_mul_bwd_kernel(const float* __restrict__ dz, const float* __restrict__ psi, const float* __restrict__ phi,
                                   int B, int N, int D, float* __restrict__ dpsi, float* __restrict__ dpre) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)B * D) return;
  const long long b = e / D;
  const int d = (int)(e - b * D);
  const float p = psi[e];
  float acc = 0.f;
  for (int n = 0; n < N; ++n) {
    const size_t o = ((size_t)b * N + n) * D + d;
    const float g = dz[o], f = phi[o];
    acc += g * f;
    dpre[o] = f > 0.f ? g * p : 0.f;
  }
  dpsi[e] = p > 0.f ? acc : 0.f;
}

}  // namespace

JB_API int jb_iqn_tau(float* tau, int rows, int N, float lo, float hi, uint64_t seed, uint64_t stream_id, long long* ctr,
                      void* stream) {
  if (!tau || !ctr || rows <= 0 || N <= 0 || !(hi > lo)) return JB_ERR_INVALID;
  const long long n = (long long)rows * N, blocks = (n + 3) / 4;
  cudaStream_t s = (cudaStream_t)stream;
  iqn_tau_kernel<<<jb_div_up(blocks, 256), 256, 0, s>>>(tau, n, lo, hi, seed, stream_id, ctr);
  tau_advance_kernel<<<1, 1, 0, s>>>(ctr, blocks);
  return jb_check_launch();
}

JB_API int jb_iqn_cos(const float* tau, int rows, int E, float* c, void* stream) {
  if (!tau || !c || rows <= 0 || E <= 0) return JB_ERR_INVALID;
  iqn_cos_kernel<<<jb_div_up((long long)rows * E, 256), 256, 0, (cudaStream_t)stream>>>(tau, rows, E, c);
  return jb_check_launch();
}

JB_API int jb_iqn_mul_fwd(const float* psi, const float* phi, int B, int N, int D, float* z, void* stream) {
  if (!psi || !phi || !z || B <= 0 || N <= 0 || D <= 0) return JB_ERR_INVALID;
  const long long total = (long long)B * N * D;
  iqn_mul_fwd_kernel<<<jb_grid_for(total, 256, 8), 256, 0, (cudaStream_t)stream>>>(psi, phi, N, D, total, z);
  return jb_check_launch();
}

JB_API int jb_iqn_mul_bwd(const float* dz, const float* psi, const float* phi, int B, int N, int D, float* dpsi, float* dpre,
                          void* stream) {
  if (!dz || !psi || !phi || !dpsi || !dpre || B <= 0 || N <= 0 || D <= 0) return JB_ERR_INVALID;
  iqn_mul_bwd_kernel<<<jb_div_up((long long)B * D, 128), 128, 0, (cudaStream_t)stream>>>(dz, psi, phi, B, N, D, dpsi, dpre);
  return jb_check_launch();
}
