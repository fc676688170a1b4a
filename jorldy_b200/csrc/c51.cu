// Distributional (C51 / Rainbow) learner kernel: softmax over atoms, expected-Q argmax,
// n-step Bellman shift of the support, categorical projection, KL loss, gradient w.r.t. the
// logits and the new PER priorities — one launch, one warp per sampled transition.
//
// Reference:
//   jorldy/core/agent/rainbow.py:167-235 (learn, parts 1+2), :285-292 (logits2Q, no max-subtraction)
//   jorldy/core/agent/c51.py:62-111 (learn), :124-135 (logits2Q with max-subtraction)
// which run ~25 small ATen kernels and materialise two dense one-hot tensors [B,K,K] per learn.
//
// Quirks reproduced on purpose (SURVEY.md §8a rows R5 / C1):
//   * weights (u-b) -> l and (b-l) -> u: when b is an integer (always for atoms clamped to
//     v_min/v_max) l == u and BOTH weights are 0, so that atom's mass is dropped; the row is then
//     renormalised by clamp(sum, 1e-8);
//   * rows whose FIRST step is terminal use mean_i(onehot_l*onehot_u + lluu) instead;
//   * Rainbow picks a* with the ONLINE net on s' (double), C51 with the TARGET net;
//   * Rainbow's IS weighting: `weights` is unsqueezed to [B,1] while KL is [B] (rainbow.py:233-235), so
//     `(weights * KL).mean()` broadcasts to a [B,B] outer product and the loss is mean(w) * mean(KL):
//     every sample's gradient is scaled by the batch-mean weight, not by its own.  Found by the
//     golden-vector comparison; reproduced here (PER / Ape-X, whose td_error is [B,1], weight per sample).
// The projection gathers contributions per output atom j in a fixed order over i (no atomics), so
// results are bit-reproducible.
#include "common.cuh"
#include "value_loss.cuh"

namespace {

constexpr int MAXK = 64;
constexpr int WARPS = 8;      // samples per CTA

struct C51HP {
  float gamma, v_min, v_max, delta_z, alpha;
  int n_step, variant /*0 c51, 1 rainbow*/;
};

// lane holds atoms k0 = lane and k1 = lane + 32.  Returns probabilities exp(log_softmax(x)).
__device__ __forceinline__ void warp_softmax(const float* __restrict__ x, int K, int lane, float& p0, float& p1,
                                             float& xmax, float& xmin) {
  const float x0 = lane < K ? x[lane] : -INFINITY;
  const float x1 = lane + 32 < K ? x[lane + 32] : -INFINITY;
  float mx = jb_warp_max(fmaxf(x0, x1));
  const float e0 = lane < K ? expf(x0 - mx) : 0.f;
  const float e1 = lane + 32 < K ? expf(x1 - mx) : 0.f;
  const float s = jb_warp_sum(e0 + e1);
  const float ls = logf(s);
  p0 = lane < K ? expf((x0 - mx) - ls) : 0.f;
  p1 = lane + 32 < K ? expf((x1 - mx) - ls) : 0.f;
  xmax = mx;
  const float m0 = lane < K ? x0 : INFINITY, m1 = lane + 32 < K ? x1 : INFINITY;
  xmin = jb_warp_min(fminf(m0, m1));
}

__global__ void __launch_bounds__(32 * WARPS)
c51_loss_kernel(const float* __restrict__ logits, const float* __restrict__ next_online, const float* __restrict__ next_target,
                const void* __restrict__ action, int action_kind, const float* __restrict__ reward,
                const float* __restrict__ done, const double* __restrict__ weights, const float* __restrict__ z,
                int B, int A, int K, C51HP hp, float* __restrict__ dlogits, float* __restrict__ kl_out,
                double* __restrict__ prio, float* __restrict__ partial /*[n_cta][4]*/) {
  __shared__ float s_l[WARPS][MAXK], s_u[WARPS][MAXK], s_wl[WARPS][MAXK], s_wu[WARPS][MAXK], s_tp[WARPS][MAXK];
  __shared__ float s_red[WARPS][4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * WARPS + warp;
  float st_loss = 0.f, st_maxq = -INFINITY, st_maxl = -INFINITY, st_minl = INFINITY;
  if (b < B) {
    const float z0 = lane < K ? z[lane] : 0.f, z1 = lane + 32 < K ? z[lane + 32] : 0.f;
    const int a_t = read_action(action, action_kind, b);
    // ---- online net on s: p for every action (stats) and for the taken action ------------------
    float pa0 = 0.f, pa1 = 0.f;
    for (int a = 0; a < A; ++a) {
      float p0, p1, mx, mn;
      warp_softmax(logits + ((size_t)b * A + a) * K, K, lane, p0, p1, mx, mn);
      const float qa = jb_warp_sum(z0 * p0 + z1 * p1);
      st_maxq = fmaxf(st_maxq, qa); st_maxl = fmaxf(st_maxl, mx); st_minl = fminf(st_minl, mn);
      if (a == a_t) { pa0 = p0; pa1 = p1; }
    }
    // ---- target action a* ---------------------------------------------------------------------
    const float* sel_src = hp.variant == 1 ? next_online : next_target;
    int a_star = 0; float best = -INFINITY;
    for (int a = 0; a < A; ++a) {
      float p0, p1, mx, mn;
      warp_softmax(sel_src + ((size_t)b * A + a) * K, K, lane, p0, p1, mx, mn);
      const float qa = jb_warp_sum(z0 * p0 + z1 * p1);
      if (qa > best) { best = qa; a_star = a; }
    }
    float tp0, tp1, mx_, mn_;
    warp_softmax(next_target + ((size_t)b * A + a_star) * K, K, lane, tp0, tp1, mx_, mn_);
    // ---- Bellman shift + projection weights per source atom i ----------------------------------
    const float* rr = reward + (size_t)b * hp.n_step;
    const float* dr = done + (size_t)b * hp.n_step;
    const float vrange = hp.v_max - hp.v_min;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = lane + 32 * h;
      if (i < K) {
        const float tz = nstep_fold(h ? z1 : z0, rr, dr, hp.n_step, hp.gamma);
        const float bb = fminf(fmaxf(tz - hp.v_min, 0.f), vrange) / hp.delta_z;
        const float l = floorf(bb), u = ceilf(bb);
        s_l[warp][i] = l; s_u[warp][i] = u; s_wl[warp][i] = u - bb; s_wu[warp][i] = bb - l;
        s_tp[warp][i] = h ? tp1 : tp0;
      }
    }
    __syncwarp();
    const bool term = dr[0] > 0.5f;
    float t0 = 0.f, t1 = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = lane + 32 * h;
      if (j < K) {
        float acc = 0.f;
        const float fj = (float)j;
        for (int i = 0; i < K; ++i) {
          const float il = (s_l[warp][i] == fj) ? 1.f : 0.f, iu = (s_u[warp][i] == fj) ? 1.f : 0.f;
          const float lluu = il * s_wl[warp][i] + iu * s_wu[warp][i];
          acc += term ? (il * iu + lluu) : s_tp[warp][i] * lluu;
        }
        if (term) acc = acc / (float)K;       // torch.mean over the source-atom axis
        if (h) t1 = acc; else t0 = acc;
      }
    }
    const float tsum = fmaxf(jb_warp_sum(t0 + t1), 1e-8f);
    t0 /= tsum; t1 /= tsum;
    // ---- KL, gradient, priority ----------------------------------------------------------------
    const float g0 = (lane < K && pa0 >= 1e-8f) ? 1.f : 0.f, g1 = (lane + 32 < K && pa1 >= 1e-8f) ? 1.f : 0.f;
    const float lp0 = lane < K ? logf(fmaxf(pa0, 1e-8f)) : 0.f, lp1 = lane + 32 < K ? logf(fmaxf(pa1, 1e-8f)) : 0.f;
    const float kl = -jb_warp_sum(t0 * lp0 + t1 * lp1);
    float w = 1.f;                               // batch-mean IS weight (see header: [B,1] x [B] broadcast)
    if (hp.variant == 1 && weights) {
      float ws = 0.f;
      for (int i = lane; i < B; i += 32) ws += (float)weights[i];
      w = jb_warp_sum(ws) / (float)B;
    }
    const float coef = w / (float)B;
    const float S = jb_warp_sum(t0 * g0 + t1 * g1);
    for (int a = 0; a < A; ++a) {
      float* d = dlogits + ((size_t)b * A + a) * K;
      if (lane < K) d[lane] = (a == a_t) ? coef * (pa0 * S - t0 * g0) : 0.f;
      if (lane + 32 < K) d[lane + 32] = (a == a_t) ? coef * (pa1 * S - t1 * g1) : 0.f;
    }
    if (lane == 0) {
      kl_out[b] = kl;
      if (prio) prio[b] = (double)powf(kl, hp.alpha);
    }
    st_loss = w * kl;
  }
  if (lane == 0) { s_red[warp][0] = st_loss; s_red[warp][1] = st_maxq; s_red[warp][2] = st_maxl; s_red[warp][3] = st_minl; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float l = 0.f, mq = -INFINITY, ml = -INFINITY, nl = INFINITY;
    for (int w = 0; w < WARPS; ++w) { l += s_red[w][0]; mq = fmaxf(mq, s_red[w][1]); ml = fmaxf(ml, s_red[w][2]); nl = fminf(nl, s_red[w][3]); }
    float* p = partial + 4 * blockIdx.x;
    p[0] = l; p[1] = mq; p[2] = ml; p[3] = nl;
  }
}

}  // namespace

// logits / next_online / next_target: [B, A, K] f32 (next_online may be NULL for variant 0).
// z: [K] support (torch.linspace(v_min, v_max, K) values).  reward/done: [B, n_step].
// Outputs: dlogits [B,A,K], kl [B], prio [B] f64 = KL^alpha (may be NULL),
// stats[4] = {loss, max_Q, max_logit, min_logit}; scratch: 4*ceil(B/8) floats.
JB_API int jb_c51_loss(const float* logits, const float* next_online, const float* next_target, const void* action,
                       int action_kind, const float* reward, const float* done, const double* weights, const float* z,
                       int B, int A, int K, float gamma, float v_min, float v_max, float alpha, int n_step, int variant,
                       float* dlogits, float* kl, double* prio, float* stats, float* scratch, void* stream) {
  if (!logits || !next_target || !action || !reward || !done || !z || !dlogits || !kl || !stats || !scratch)
    return JB_ERR_INVALID;
  if (B <= 0 || A <= 0 || K <= 1 || K > MAXK || n_step <= 0 || (variant == 1 && !next_online)) return JB_ERR_INVALID;
  C51HP hp{gamma, v_min, v_max, (float)(((double)v_max - (double)v_min) / (double)(K - 1)), alpha, n_step, variant};
  const int n_cta = jb_div_up(B, WARPS);
  cudaStream_t s = (cudaStream_t)stream;
  c51_loss_kernel<<<n_cta, 32 * WARPS, 0, s>>>(logits, next_online, next_target, action, action_kind, reward, done, weights, z,
                                              B, A, K, hp, dlogits, kl, prio, scratch);
  loss_logits_finalize_kernel<<<1, 32, 0, s>>>(scratch, n_cta, B, stats);
  return jb_check_launch();
}

namespace {
// expected Q per action from logits: q[b,a] = sum_k z_k softmax(logits[b,a,:])_k  (act path)
__global__ void c51_q_kernel(const float* __restrict__ logits, const float* __restrict__ z, int M, int A, int K,
                             float* __restrict__ q) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= M * A) return;
  float p0, p1, mx, mn;
  warp_softmax(logits + (size_t)row * K, K, lane, p0, p1, mx, mn);
  const float z0 = lane < K ? z[lane] : 0.f, z1 = lane + 32 < K ? z[lane + 32] : 0.f;
  const float qa = jb_warp_sum(z0 * p0 + z1 * p1);
  if (lane == 0) q[row] = qa;
}
}  // namespace

JB_API int jb_c51_q(const float* logits, const float* z, int M, int A, int K, float* q, void* stream) {
  if (!logits || !z || !q || M <= 0 || A <= 0 || K <= 1 || K > MAXK) return JB_ERR_INVALID;
  c51_q_kernel<<<jb_div_up((long long)M * A * 32, 256), 256, 0, (cudaStream_t)stream>>>(logits, z, M, A, K, q);
  return jb_check_launch();
}
