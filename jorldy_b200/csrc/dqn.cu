// Value-based learner kernels: epsilon-greedy action selection, dueling combine, and the fused
// TD-target + loss + gradient + new-priority kernel shared by DQN / Double / Multistep / PER / Ape-X.
//
// Reference (jorldy/core/agent/):
//   dqn.py:99-115     act: epsilon-greedy over argmax Q
//   dqn.py:128-138    q = sum(Q(s)*onehot(a)); y = r + (1-d)*gamma*max_a' Qt(s'); smooth_l1_loss
//   double.py:25-41   a* = argmax Q(s'); y = r + Qt(s')[a*] * (gamma*(1-d))
//   multistep.py:41-50 / ape_x.py:96-106   y <- r_i + (1-d_i)*gamma*y for i = n-1..0
//   per.py:50-77, ape_x.py:108-116   td = |y-q|; priority = td^alpha; loss = mean(w * td^2)
//   network/dueling.py:21-35   Q = V + A - mean_a A   (rainbow.py network: per atom)
// The reference builds one-hot matrices and ~15 small ATen launches per learn and then issues B
// `.item()` device->host syncs to write priorities one by one; here it is one launch, with the
// new priorities left in device memory (f64, as the sum-tree wants them).
#include "common.cuh"
#include "munchausen.cuh"
#include "philox.cuh"
#include "value_loss.cuh"

namespace {

constexpr int MAX_ACT = 32;

// ---- epsilon-greedy ----------------------------------------------------------------------------
// One draw per ROW decides random-vs-greedy (the reference draws once per act() call of one actor,
// dqn.py:104; a row here is an actor).  eps_rows (may be NULL) gives per-actor epsilons (Ape-X,
// ape_x.py:166-172), else the scalar eps.  q_sel (may be NULL) receives Q(s)[a] (ape_x.py:76).
__global__ void q_act_kernel(const float* __restrict__ q, int M, int A, float eps, const float* __restrict__ eps_rows,
                             const float* __restrict__ u_in /*[M,2] or NULL*/, uint64_t seed, uint64_t stream_base,
                             long long* __restrict__ row_ctr, int64_t* __restrict__ action, float* __restrict__ q_sel) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float u0, u1;
  if (u_in) { u0 = u_in[2 * m]; u1 = u_in[2 * m + 1]; }
  else {
    const uint64_t c = jb_next_row_ctr(row_ctr, m);
    jb_philox4 r = jb_philox(seed, stream_base + (uint64_t)m, c);
    u0 = jb_u01_float(r.x); u1 = jb_u01_float(r.y);
  }
  const float e = eps_rows ? eps_rows[m] : eps;
  const float* qr = q + (size_t)m * A;
  int pick;
  if (u0 < e) {
    pick = (int)(u1 * (float)A);
    if (pick >= A) pick = A - 1;
  } else {
    pick = 0;
    float best = qr[0];
    for (int a = 1; a < A; ++a) if (qr[a] > best) { best = qr[a]; pick = a; }   // first max, like torch.argmax
  }
  action[m] = pick;
  if (q_sel) q_sel[m] = qr[pick];
}

// ---- dueling combine: out[b,a,k] = v[b,k] + a[b,a,k] - mean_a a[b,:,k]  (K = 1 for scalar Q) -------
__global__ void dueling_fwd_kernel(const float* __restrict__ adv, const float* __restrict__ val, int B, int A, int K,
                                   float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // over B*K
  if (i >= B * K) return;
  const int b = i / K, k = i % K;
  float s = 0.f;
  for (int a = 0; a < A; ++a) s += adv[((size_t)b * A + a) * K + k];
  const float mean = s / (float)A;
  const float v = val[(size_t)b * K + k];
  for (int a = 0; a < A; ++a) {
    const size_t o = ((size_t)b * A + a) * K + k;
    out[o] = (adv[o] - mean) + v;             // x_a - mean, then + x_v (dueling.py:27-34)
  }
}
__global__ void dueling_bwd_kernel(const float* __restrict__ dout, int B, int A, int K, float* __restrict__ dadv,
                                   float* __restrict__ dval) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * K) return;
  const int b = i / K, k = i % K;
  float s = 0.f;
  for (int a = 0; a < A; ++a) s += dout[((size_t)b * A + a) * K + k];
  const float mean = s / (float)A;
  for (int a = 0; a < A; ++a) {
    const size_t o = ((size_t)b * A + a) * K + k;
    dadv[o] = dout[o] - mean;
  }
  dval[(size_t)b * K + k] = s;
}

// ---- fused TD loss --------------------------------------------------------------------------------
struct TdHP {
  float gamma, alpha;
  int n_step, double_q, loss_kind /*0 smooth_l1, 1 weighted mse*/, order /*0 dqn, 1 double/per, 2 n-step loop*/;
};

__global__ void __launch_bounds__(1024)
td_loss_kernel(const float* __restrict__ q, const float* __restrict__ q_next, const float* __restrict__ qt_next,
               const void* __restrict__ action, int action_kind, const float* __restrict__ reward,
               const float* __restrict__ done, const double* __restrict__ weights, int B, int A, TdHP hp,
               float* __restrict__ dq, double* __restrict__ prio, float* __restrict__ stats) {
  __shared__ float s_loss[32], s_max[32];
  const int b = threadIdx.x;
  float q_b = -INFINITY, loss_b = 0.f;
  if (b < B) {
    const int a = read_action(action, action_kind, b);
    const float* qr = q + (size_t)b * A;
    const float* tr = qt_next + (size_t)b * A;
    q_b = qr[a];
    // bootstrap value
    float y;
    if (hp.double_q) {
      y = tr[first_argmax(q_next + (size_t)b * A, A)];
    } else {
      y = tr[0];
      for (int i = 1; i < A; ++i) y = fmaxf(y, tr[i]);
    }
    const float* rr = reward + (size_t)b * hp.n_step;
    const float* dr = done + (size_t)b * hp.n_step;
    if (hp.order == 0)       y = __fadd_rn(rr[0], __fmul_rn(__fmul_rn(__fadd_rn(1.f, -dr[0]), hp.gamma), y));
    else if (hp.order == 1)  y = __fadd_rn(rr[0], __fmul_rn(y, __fmul_rn(hp.gamma, __fadd_rn(1.f, -dr[0]))));
    else                     y = nstep_fold(y, rr, dr, hp.n_step, hp.gamma);
    const float diff = q_b - y;
    float g;
    if (hp.loss_kind == 0) {                    // F.smooth_l1_loss(q, y), beta = 1, mean
      const float ad = fabsf(diff);
      loss_b = ad < 1.f ? 0.5f * diff * diff : ad - 0.5f;
      g = ad < 1.f ? diff : (diff > 0.f ? 1.f : -1.f);
    } else {                                    // (w * td^2).mean(), td = |y - q|
      const float w = weights ? (float)weights[b] : 1.f;
      const float td = fabsf(y - q_b);
      loss_b = w * (td * td);
      g = w * 2.f * diff;
    }
    for (int i = 0; i < A; ++i) dq[(size_t)b * A + i] = 0.f;
    dq[(size_t)b * A + a] = g / (float)B;
    if (prio) prio[b] = (double)powf(fabsf(y - q_b), hp.alpha);    // torch.pow(td_error, alpha) in f32, then .item()
  }
  // block reductions (fixed order)
  float l = loss_b, mx = q_b;
  for (int o = 16; o > 0; o >>= 1) { l += __shfl_down_sync(0xffffffffu, l, o); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
  if ((threadIdx.x & 31) == 0) { s_loss[threadIdx.x >> 5] = l; s_max[threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f, m = -INFINITY;
    for (int w = 0; w < (blockDim.x + 31) / 32; ++w) { t += s_loss[w]; m = fmaxf(m, s_max[w]); }
    stats[0] = t / (float)B;   // loss
    stats[1] = m;              // max_Q = max over the batch of Q(s)[a]
  }
}

// ---- Munchausen DQN loss (arXiv:2007.14430) ------------------------------------------------------
// One warp per sample; lane 0 forms the target in a fixed order (munchausen.cuh), the warp writes the sample's dq row.
// The per-sample loss and Q(s)[a_t] go to partial[2b], partial[2b + 1] and one thread folds them (loss_maxq_finalize_kernel).
constexpr int MDQN_WARPS = 4;

__global__ void __launch_bounds__(MDQN_WARPS * 32)
mdqn_loss_kernel(const float* __restrict__ q, const float* __restrict__ qt_s, const float* __restrict__ qt_next,
                 const void* __restrict__ action, int action_kind, const float* __restrict__ reward,
                 const float* __restrict__ done, int B, int A, float gamma, float m_alpha, float m_tau, float l0,
                 float* __restrict__ dq, float* __restrict__ partial /*[B][2]*/) {
  __shared__ float s_pi[MDQN_WARPS][MUNCHAUSEN_MAX_A], s_tlp[MDQN_WARPS][MUNCHAUSEN_MAX_A];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * MDQN_WARPS + warp;
  if (b >= B) return;
  const int a_t = read_action(action, action_kind, b);
  float g = 0.f;
  if (lane == 0) {
    const float* qn = qt_next + (size_t)b * A;
    const float bonus = munchausen_row(qt_s + (size_t)b * A, qn, A, a_t, m_tau, m_alpha, l0, s_pi[warp], s_tlp[warp]);
    float v = 0.f;
    for (int a = 0; a < A; ++a) v += s_pi[warp][a] * (qn[a] - s_tlp[warp][a]);
    const float nd = __fmul_rn(__fadd_rn(1.f, -done[b]), gamma);
    const float y = __fadd_rn(__fadd_rn(reward[b], bonus), __fmul_rn(nd, v));
    const float q_b = q[(size_t)b * A + a_t];
    const float diff = q_b - y, ad = fabsf(diff);                 // F.smooth_l1_loss(q, y), beta = 1, as td_loss_kernel
    g = ad < 1.f ? diff : (diff > 0.f ? 1.f : -1.f);
    partial[2 * b] = ad < 1.f ? 0.5f * diff * diff : ad - 0.5f;
    partial[2 * b + 1] = q_b;
  }
  g = __shfl_sync(0xffffffffu, g, 0) / (float)B;
  for (int a = lane; a < A; a += 32) dq[(size_t)b * A + a] = a == a_t ? g : 0.f;
}

}  // namespace

JB_API int jb_q_act(const float* q, int M, int A, float eps, const float* eps_rows, const float* u, uint64_t seed,
                    uint64_t stream_base, long long* row_ctr, int64_t* action, float* q_sel, void* stream) {
  if (!q || !action || M <= 0 || A <= 0) return JB_ERR_INVALID;
  q_act_kernel<<<jb_div_up(M, 128), 128, 0, (cudaStream_t)stream>>>(q, M, A, eps, eps_rows, u, seed, stream_base, row_ctr, action, q_sel);
  return jb_check_launch();
}

JB_API int jb_dueling_fwd(const float* adv, const float* val, int B, int A, int K, float* out, void* stream) {
  if (!adv || !val || !out || B <= 0 || A <= 0 || K <= 0) return JB_ERR_INVALID;
  dueling_fwd_kernel<<<jb_div_up((long long)B * K, 128), 128, 0, (cudaStream_t)stream>>>(adv, val, B, A, K, out);
  return jb_check_launch();
}

JB_API int jb_dueling_bwd(const float* dout, int B, int A, int K, float* dadv, float* dval, void* stream) {
  if (!dout || !dadv || !dval || B <= 0 || A <= 0 || K <= 0) return JB_ERR_INVALID;
  dueling_bwd_kernel<<<jb_div_up((long long)B * K, 128), 128, 0, (cudaStream_t)stream>>>(dout, B, A, K, dadv, dval);
  return jb_check_launch();
}

// q[B,A] online Q(s); q_next[B,A] online Q(s') (double_q only, else NULL); qt_next[B,A] target Q(s').
// action_kind: 0 int64, 1 int32, 2 float32.  reward/done: [B,n_step] f32.  weights: f64 [B] IS weights
// or NULL.  order: 0 dqn.py:133-136, 1 double.py/per.py product order, 2 n-step backward loop.
// Outputs: dq[B,A] = d loss/d q, prio[B] f64 = |td|^alpha (may be NULL), stats[2] = {loss, max_Q}.
JB_API int jb_td_loss(const float* q, const float* q_next, const float* qt_next, const void* action, int action_kind,
                      const float* reward, const float* done, const double* weights, int B, int A, float gamma,
                      float alpha, int n_step, int double_q, int loss_kind, int order, float* dq, double* prio,
                      float* stats, void* stream) {
  if (!q || !qt_next || !action || !reward || !done || !dq || !stats) return JB_ERR_INVALID;
  if (B <= 0 || B > 1024 || A <= 0 || n_step <= 0 || (double_q && !q_next)) return JB_ERR_INVALID;
  TdHP hp{gamma, alpha, n_step, double_q, loss_kind, order};
  const int threads = ((B + 31) / 32) * 32;
  td_loss_kernel<<<1, threads, 0, (cudaStream_t)stream>>>(q, q_next, qt_next, action, action_kind, reward, done, weights,
                                                         B, A, hp, dq, prio, stats);
  return jb_check_launch();
}

// M-DQN: q[B,A] online Q(s); qt_s[B,A] target Q(s); qt_next[B,A] target Q(s'); reward/done [B] f32.
// y = r + alpha clip(tau logpi(a|s), l0, 0) + ((1-d) gamma) sum_a pi'(a) (qt_next[a] - tau logpi'(a|s')) (munchausen.cuh);
// dq[b, a_b] = smooth_l1'(q - y)/B, 0 elsewhere; stats[2] = {loss, max_Q}; scratch: 2*B floats.
JB_API int jb_mdqn_loss(const float* q, const float* qt_s, const float* qt_next, const void* action, int action_kind,
                        const float* reward, const float* done, int B, int A, float gamma, float m_alpha, float m_tau,
                        float l0, float* dq, float* stats, float* scratch, void* stream) {
  if (!q || !qt_s || !qt_next || !action || !reward || !done || !dq || !stats || !scratch) return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || A > MUNCHAUSEN_MAX_A || action_kind < 0 || action_kind > 2 || !(m_tau > 0.f) || !(l0 <= 0.f))
    return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  mdqn_loss_kernel<<<jb_div_up(B, MDQN_WARPS), MDQN_WARPS * 32, 0, s>>>(q, qt_s, qt_next, action, action_kind, reward, done,
                                                                       B, A, gamma, m_alpha, m_tau, l0, dq, scratch);
  loss_maxq_finalize_kernel<<<1, 32, 0, s>>>(scratch, B, stats);
  return jb_check_launch();
}
