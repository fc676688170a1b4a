// MuZero (Schrittwieser et al., arXiv:1911.08265) on flat observations: the categorical value transform, the latent
// min-max scaling, a batched Monte-Carlo tree search with one tree per env in global memory, and the K-step unrolled
// loss.  The networks' dense layers are the existing GEMMs (csrc/linear.cu, csrc/heads.cu).
//
// Every reduction runs in a fixed order with no atomics, so each entry point is bit-reproducible run to run:
//   - the tree kernels give each env one warp; lanes cover the actions (A <= 18) or a row's columns, and every sum is a
//     fixed xor-shuffle tree or a per-lane loop in ascending index;
//   - the loss gives each (window, position) one warp and folds the per-warp partials with one thread in row order.
//
// Tree layout (index e = (env * (S + 1) + node) * A + action):
//   edge_n int32, edge_w / edge_p / edge_r f32, edge_child int32 (-1: not expanded)
//   latent [N, S + 1, Hs], count int32 [N] (nodes in use), bounds f32 [N, 2] (min, max of the backed-up Q values)
//   path int32 [N, S + 1] (edges root -> leaf as node * A + action), path_len int32 [N]
#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int MZ_MAX_A = 18;
constexpr int MZ_MAX_HS = 256;         // scaling: 8 columns per lane
constexpr int MZ_MAX_SUPPORT = 300;    // 2V + 1 <= 601 atoms
constexpr double VR_EPS = 1e-3;
constexpr float SCALE_MIN_RANGE = 1e-5f;
constexpr float PB_C_BASE = 19652.f, PB_C_INIT = 1.25f;
constexpr int WARPS = 8;

__device__ __forceinline__ double sgn(double x) { return (double)((x > 0.0) - (x < 0.0)); }
__device__ __forceinline__ double value_h(double x) { return sgn(x) * (sqrt(fabs(x) + 1.0) - 1.0) + VR_EPS * x; }
__device__ __forceinline__ double value_h_inv(double x) {
  const double s = (sqrt(1.0 + 4.0 * VR_EPS * (fabs(x) + 1.0 + VR_EPS)) - 1.0) / (2.0 * VR_EPS);
  return sgn(x) * (s * s - 1.0);
}

// expectation of softmax(logits) over the atoms -V..V, then h^-1; every lane returns it
__device__ __forceinline__ double support_expect(const float* __restrict__ z, int V, int lane) {
  const int n = 2 * V + 1;
  float m = -INFINITY;
  for (int i = lane; i < n; i += 32) m = fmaxf(m, z[i]);
  m = jb_warp_max(m);
  double se = 0.0, sx = 0.0;
  for (int i = lane; i < n; i += 32) {
    const double e = exp((double)z[i] - (double)m);
    se += e;
    sx += e * (double)(i - V);
  }
  se = jb_warp_sum_d(se);
  sx = jb_warp_sum_d(sx);
  return value_h_inv(sx / se);
}

// two-hot of h(x) clamped to [-V, V]: (lower atom index, weight of the upper atom)
__device__ __forceinline__ void two_hot(double x, int V, int& lo, double& up) {
  double y = fmin(fmax(value_h(x), -(double)V), (double)V);
  const double f = floor(y);
  lo = (int)f + V;
  up = y - f;
  if (lo >= 2 * V) { lo = 2 * V; up = 0.0; }
}

__device__ __forceinline__ double two_hot_at(int i, int lo, double up) {
  return i == lo ? 1.0 - up : (i == lo + 1 ? up : 0.0);
}

// argmax over the lanes' (score, index) with ties to the lowest index; lanes with valid = false never win
__device__ __forceinline__ int warp_argmax(float s, int idx) {
  for (int o = 16; o > 0; o >>= 1) {
    const float so = __shfl_xor_sync(0xffffffffu, s, o);
    const int io = __shfl_xor_sync(0xffffffffu, idx, o);
    if (so > s || (so == s && io < idx)) { s = so; idx = io; }
  }
  return idx;
}

// ---- scaling -------------------------------------------------------------------------------------------------------
// one warp per row; lowest index wins ties for both the min and the max
__device__ __forceinline__ void row_minmax(const float* __restrict__ x, int H, int lane, float& mn, float& mx, int& imn,
                                           int& imx) {
  mn = INFINITY; mx = -INFINITY; imn = H; imx = H;
  for (int j = lane; j < H; j += 32) {
    const float v = x[j];
    if (v < mn) { mn = v; imn = j; }
    if (v > mx) { mx = v; imx = j; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float a = __shfl_xor_sync(0xffffffffu, mn, o), b = __shfl_xor_sync(0xffffffffu, mx, o);
    const int ia = __shfl_xor_sync(0xffffffffu, imn, o), ib = __shfl_xor_sync(0xffffffffu, imx, o);
    if (a < mn || (a == mn && ia < imn)) { mn = a; imn = ia; }
    if (b > mx || (b == mx && ib < imx)) { mx = b; imx = ib; }
  }
}

__global__ void __launch_bounds__(WARPS * 32)
scale_fwd_kernel(const float* __restrict__ x, int M, int H, float* __restrict__ y, float* __restrict__ y2, int ld2) {
  const int row = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (size_t)row * H;
  float mn, mx; int imn, imx;
  row_minmax(xr, H, lane, mn, mx, imn, imx);
  const float s = fmaxf(mx - mn, SCALE_MIN_RANGE);
  for (int j = lane; j < H; j += 32) {
    const float v = (xr[j] - mn) / s;
    y[(size_t)row * H + j] = v;
    if (y2) y2[(size_t)row * ld2 + j] = v;
  }
}

// dx_j = dy_j / s, plus d min at the argmin and d max at the argmax (the range is a constant when it is clamped)
__global__ void __launch_bounds__(WARPS * 32)
scale_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, int M, int H, float* __restrict__ dx) {
  const int row = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (size_t)row * H;
  const float* gr = dy + (size_t)row * H;
  float mn, mx; int imn, imx;
  row_minmax(xr, H, lane, mn, mx, imn, imx);
  const bool clamped = !(mx - mn >= SCALE_MIN_RANGE);
  const float s = clamped ? SCALE_MIN_RANGE : mx - mn;
  float dmn = 0.f, dmx = 0.f;
  for (int j = lane; j < H; j += 32) {
    const float yj = (xr[j] - mn) / s;
    dmn += gr[j] * (clamped ? -1.f : yj - 1.f);
    dmx += gr[j] * (clamped ? 0.f : -yj);
  }
  dmn = jb_warp_sum(dmn) / s;
  dmx = jb_warp_sum(dmx) / s;
  for (int j = lane; j < H; j += 32)
    dx[(size_t)row * H + j] = gr[j] / s + (j == imn ? dmn : 0.f) + (j == imx ? dmx : 0.f);
}

// ---- value transform ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(WARPS * 32)
support_to_scalar_kernel(const float* __restrict__ logits, int M, int V, float* __restrict__ out) {
  const int row = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const double v = support_expect(logits + (size_t)row * (2 * V + 1), V, lane);
  if (lane == 0) out[row] = (float)v;
}

__global__ void scalar_to_support_kernel(const float* __restrict__ x, int M, int V, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int n = 2 * V + 1;
  if (i >= (long long)M * n) return;
  const int m = (int)(i / n), k = (int)(i % n);
  int lo; double up;
  two_hot((double)x[m], V, lo, up);
  out[i] = (float)two_hot_at(k, lo, up);
}

// ---- search ---------------------------------------------------------------------------------------------------------
struct Tree {
  int* n; float* w; float* p; float* r; int* child; float* latent; int* count; float* bounds; int* path; int* path_len;
};

// the env's draw counter, advanced once by lane 0 and broadcast to the warp
__device__ __forceinline__ uint64_t lane_ctr(long long* __restrict__ row_ctr, int env, int lane) {
  unsigned long long c = 0;
  if (lane == 0) c = jb_next_row_ctr(row_ctr, env);
  return __shfl_sync(0xffffffffu, c, 0);
}

// softmax over the A logits of this lane's action (lanes >= A return 0); every lane gets the same max and sum
__device__ __forceinline__ float lane_softmax(const float* __restrict__ z, int A, int lane) {
  const float v = lane < A ? z[lane] : -INFINITY;
  const float m = jb_warp_max(v);
  const float e = lane < A ? expf(v - m) : 0.f;
  return e / jb_warp_sum(e);
}

// Gamma(alpha) = Gamma(alpha + 1) U^(1/alpha), Gamma(alpha + 1) by Marsaglia-Tsang; draw i of this subsequence is
// Philox counter (ctr << 16) + i, so the rejection loop only consumes its own subsequence
__device__ __forceinline__ double gamma_draw(uint64_t seed, uint64_t stream, uint64_t ctr, double alpha) {
  const double d = alpha + 1.0 - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
  const jb_philox4 r0 = jb_philox(seed, stream, ctr << 16);
  const double u_boost = 1.0 - jb_u01_double(r0.x, r0.y);           // (0, 1]
  double g = d;
  for (uint64_t i = 1; i < 65536; ++i) {
    const jb_philox4 r = jb_philox(seed, stream, (ctr << 16) + i);
    const double u1 = 1.0 - jb_u01_double(r.x, r.y), u2 = jb_u01_double(r.z, 0u);
    const double x = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
    double v = 1.0 + c * x;
    if (v <= 0.0) continue;
    v = v * v * v;
    const double u = 1.0 - jb_u01_double(r.w, 0u);          // (0, 1], from r.w alone
    if (log(u) < 0.5 * x * x + d - d * v + d * log(v)) { g = d * v; break; }
  }
  return g * pow(u_boost, 1.0 / alpha);
}

__global__ void __launch_bounds__(WARPS * 32)
mcts_root_kernel(const float* __restrict__ pi_logits, const float* __restrict__ v_logits, const float* __restrict__ latent0,
                 int N, int A, int S, int Hs, int V, int training, float dir_alpha, float frac,
                 const double* __restrict__ gamma_in, uint64_t seed, long long* __restrict__ row_ctr, Tree t,
                 float* __restrict__ root_value) {
  const int env = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (env >= N) return;
  float prior = lane_softmax(pi_logits + (size_t)env * A, A, lane);
  if (training) {
    const uint64_t ctr = lane_ctr(row_ctr, env, lane);
    double g = 0.0;
    if (lane < A)
      g = gamma_in ? gamma_in[(size_t)env * A + lane]
                   : gamma_draw(seed, ((uint64_t)env << 8) | (uint64_t)lane, ctr, (double)dir_alpha);
    const double sum = jb_warp_sum_d(g);
    if (lane < A) prior = (float)((1.0 - (double)frac) * (double)prior + (double)frac * (g / sum));
  }
  const double v = support_expect(v_logits + (size_t)env * (2 * V + 1), V, lane);
  const size_t nodes = (size_t)env * (S + 1);
  for (int e = lane; e < (S + 1) * A; e += 32) {
    const size_t k = nodes * A + e;
    t.n[k] = 0; t.w[k] = 0.f; t.r[k] = 0.f; t.p[k] = 0.f; t.child[k] = -1;
  }
  __syncwarp();
  if (lane < A) t.p[nodes * A + lane] = prior;
  for (int j = lane; j < Hs; j += 32) t.latent[nodes * Hs + j] = latent0[(size_t)env * Hs + j];
  if (lane == 0) {
    t.count[env] = 1;
    t.bounds[2 * env] = INFINITY;
    t.bounds[2 * env + 1] = -INFINITY;
    t.path_len[env] = 0;
    if (root_value) root_value[env] = (float)v;
  }
}

__global__ void __launch_bounds__(WARPS * 32)
mcts_select_kernel(int N, int A, int S, int Hs, float gamma, Tree t, int* __restrict__ leaf_node,
                   int* __restrict__ leaf_action, float* __restrict__ dyn_in) {
  const int env = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (env >= N) return;
  const size_t nodes = (size_t)env * (S + 1);
  const float qmin = t.bounds[2 * env], qmax = t.bounds[2 * env + 1];
  int node = 0, depth = 0, a = 0;
  int parent_n = 0;
  {
    const int n0 = lane < A ? t.n[nodes * A + lane] : 0;
    parent_n = (int)jb_warp_sum((float)n0);
  }
  while (true) {
    const size_t base = (nodes + node) * A;
    float score = -INFINITY;
    if (lane < A) {
      const int n = t.n[base + lane];
      float q = 0.f;
      if (n > 0) {
        q = t.r[base + lane] + gamma * __fdividef(t.w[base + lane], (float)n);
        if (qmax > qmin) q = (q - qmin) / (qmax - qmin);
      }
      const float pb = (logf(((float)parent_n + PB_C_BASE + 1.f) / PB_C_BASE) + PB_C_INIT) * sqrtf((float)parent_n) /
                       (float)(n + 1);
      score = q + pb * t.p[base + lane];
    }
    a = warp_argmax(score, lane < A ? lane : 32);
    if (lane == 0) t.path[nodes + depth] = node * A + a;
    ++depth;
    const int c = t.child[base + a];
    if (c < 0 || depth > S) break;
    parent_n = t.n[base + a];
    node = c;
  }
  if (lane == 0) { t.path_len[env] = depth; leaf_node[env] = node; leaf_action[env] = a; }
  const float* src = t.latent + (nodes + node) * Hs;
  float* dst = dyn_in + (size_t)env * (Hs + A);
  for (int j = lane; j < Hs; j += 32) dst[j] = src[j];
  if (lane < A) dst[Hs + lane] = lane == a ? 1.f : 0.f;
}

__global__ void __launch_bounds__(WARPS * 32)
mcts_expand_backup_kernel(const float* __restrict__ latent, const float* __restrict__ pi_logits,
                          const float* __restrict__ v_logits, const float* __restrict__ r_logits, int N, int A, int S,
                          int Hs, int V, int R, float gamma, const int* __restrict__ leaf_node,
                          const int* __restrict__ leaf_action, Tree t) {
  const int env = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (env >= N) return;
  const size_t nodes = (size_t)env * (S + 1);
  const int nn = t.count[env];
  const double v = support_expect(v_logits + (size_t)env * (2 * V + 1), V, lane);
  const double r = support_expect(r_logits + (size_t)env * (2 * R + 1), R, lane);
  const float prior = lane_softmax(pi_logits + (size_t)env * A, A, lane);
  if (nn > S) return;        // full tree: only reachable with more simulations than nodes
  for (int j = lane; j < Hs; j += 32) t.latent[(nodes + nn) * Hs + j] = latent[(size_t)env * Hs + j];
  if (lane < A) t.p[(nodes + nn) * A + lane] = prior;
  if (lane != 0) return;
  const size_t leaf = (nodes + leaf_node[env]) * A + leaf_action[env];
  t.child[leaf] = nn;
  t.r[leaf] = (float)r;
  t.count[env] = nn + 1;
  float qmin = t.bounds[2 * env], qmax = t.bounds[2 * env + 1];
  float g = (float)v;
  for (int d = t.path_len[env] - 1; d >= 0; --d) {
    const size_t e = nodes * A + t.path[nodes + d];
    const float w = t.w[e] + g;
    const int n = t.n[e] + 1;
    t.w[e] = w;
    t.n[e] = n;
    const float q = t.r[e] + gamma * __fdividef(w, (float)n);
    qmin = fminf(qmin, q);
    qmax = fmaxf(qmax, q);
    g = t.r[e] + gamma * g;
  }
  t.bounds[2 * env] = qmin;
  t.bounds[2 * env + 1] = qmax;
}

__global__ void __launch_bounds__(WARPS * 32)
mcts_act_kernel(int N, int A, int S, float gamma, int training, const float* __restrict__ temperature,
                const double* __restrict__ u_in, uint64_t seed, long long* __restrict__ row_ctr, Tree t,
                int64_t* __restrict__ action, float* __restrict__ pi, float* __restrict__ root_value) {
  const int env = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (env >= N) return;
  const size_t base = (size_t)env * (S + 1) * A;
  const int n = lane < A ? t.n[base + lane] : 0;
  const float tot = jb_warp_sum((float)n);
  const float num = lane < A ? (float)n * t.r[base + lane] + gamma * t.w[base + lane] : 0.f;
  const float vsum = jb_warp_sum(num);
  if (lane < A) pi[(size_t)env * A + lane] = tot > 0.f ? (float)n / tot : 0.f;
  int a;
  if (training) {
    const uint64_t ctr = lane_ctr(row_ctr, env, lane);
    double u = 0.0;
    if (lane == 0) {
      if (u_in) u = u_in[env];
      else { const jb_philox4 q = jb_philox(seed, (1ull << 40) | (uint64_t)env, ctr); u = jb_u01_double(q.x, q.y); }
    }
    u = __shfl_sync(0xffffffffu, u, 0);
    const double inv_t = 1.0 / (double)temperature[0];
    const double wl = lane < A ? pow((double)n, inv_t) : 0.0;
    // inclusive prefix sum over the lanes (ascending action order)
    double c = wl;
    for (int o = 1; o < 32; o <<= 1) {
      const double x = __shfl_up_sync(0xffffffffu, c, o);
      if (lane >= o) c += x;
    }
    const double total = __shfl_sync(0xffffffffu, c, 31);
    const bool hit = lane < A && wl > 0.0 && u * total < c;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    a = m ? __ffs(m) - 1 : 0;
  } else {
    a = warp_argmax(lane < A ? (float)n : -INFINITY, lane < A ? lane : 32);
  }
  if (lane == 0) {
    action[env] = a;
    if (root_value) root_value[env] = tot > 0.f ? vsum / tot : 0.f;
  }
}

// ---- loss -----------------------------------------------------------------------------------------------------------
// softmax cross-entropy of one row against a target given by tgt(i); writes d = scale (softmax - target) and returns
// the row's loss (every lane)
template <class Tgt>
__device__ __forceinline__ double ce_row(const float* __restrict__ z, int n, double scale, float* __restrict__ dz, int lane, Tgt tgt) {
  float m = -INFINITY;
  for (int i = lane; i < n; i += 32) m = fmaxf(m, z[i]);
  m = jb_warp_max(m);
  double se = 0.0;
  for (int i = lane; i < n; i += 32) se += exp((double)z[i] - (double)m);
  se = jb_warp_sum_d(se);
  const double lse = (double)m + log(se);
  double l = 0.0;
  for (int i = lane; i < n; i += 32) {
    const double y = tgt(i), lp = (double)z[i] - lse;
    l -= y * lp;
    if (dz) dz[i] = (float)(scale * (exp(lp) - y));
  }
  return jb_warp_sum_d(l);
}

__global__ void __launch_bounds__(WARPS * 32)
muzero_loss_kernel(const float* __restrict__ pi_logits, const float* __restrict__ v_logits,
                   const float* __restrict__ r_logits, const float* __restrict__ reward, const float* __restrict__ done,
                   const float* __restrict__ root_value, const float* __restrict__ policy, const double* __restrict__ weights,
                   int B, int K, int n_step, int A, int V, int R, float gamma, float value_coef, float alpha,
                   double inv_b, double inv_k, float* __restrict__ d_pi, float* __restrict__ d_v, float* __restrict__ d_r, double* __restrict__ prio,
                   double* __restrict__ partial /*[B (K + 1)][3]*/) {
  const int row = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= B * (K + 1)) return;
  const int k = row / B, b = row % B, L = K + n_step + 1, nv = 2 * V + 1, nr = 2 * R + 1;
  const float* rr = reward + (size_t)b * L;
  const float* dr = done + (size_t)b * L;
  const double w = weights ? weights[b] : 1.0;
  const double f = (k == 0 ? 1.0 : inv_k) * w, scale = f * inv_b;
  bool absorbing = false, prev_absorbing = false;         // a done before position k / before position k - 1
  for (int j = 0; j < k; ++j) {
    prev_absorbing = absorbing;
    if (dr[j] != 0.f) absorbing = true;
  }
  double z = 0.0;
  if (!absorbing) {
    z = (double)root_value[(size_t)b * L + k + n_step];
    for (int i = n_step - 1; i >= 0; --i) z = (double)rr[k + i] + (1.0 - (double)dr[k + i]) * (double)gamma * z;
  }
  const size_t kb = (size_t)k * B + b;
  int lo; double up;
  two_hot(z, V, lo, up);
  const double lv = ce_row(v_logits + kb * nv, nv, scale * (double)value_coef, d_v + kb * nv, lane,
                           [=](int i) { return two_hot_at(i, lo, up); });
  double lr = 0.0;
  if (k > 0) {
    const double u = prev_absorbing ? 0.0 : (double)rr[k - 1];
    int rlo; double rup;
    two_hot(u, R, rlo, rup);
    const size_t rb = (size_t)(k - 1) * B + b;
    lr = ce_row(r_logits + rb * nr, nr, scale, d_r + rb * nr, lane, [=](int i) { return two_hot_at(i, rlo, rup); });
  }
  const float* tp = policy + ((size_t)b * L + k) * A;
  const double lp = ce_row(pi_logits + kb * A, A, absorbing ? 0.0 : scale, d_pi + kb * A, lane,
                           [=](int i) { return absorbing ? 0.0 : (double)tp[i]; });
  if (k == 0 && prio) {
    const double v0 = support_expect(v_logits + kb * nv, V, lane);
    if (lane == 0) prio[b] = pow(fabs(v0 - z), (double)alpha);
  }
  if (lane == 0) {
    partial[3 * row] = f * (double)value_coef * lv;
    partial[3 * row + 1] = f * lr;
    partial[3 * row + 2] = f * lp;
  }
}

// stats = {loss, value_loss, reward_loss, policy_loss}, each a sum over rows in row order divided by B
__global__ void muzero_finalize_kernel(const double* __restrict__ partial, int rows, int B, float* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  double s[3] = {0.0, 0.0, 0.0};
  for (int i = 0; i < rows; ++i)
    for (int q = 0; q < 3; ++q) s[q] += partial[3 * i + q];
  stats[1] = (float)(s[0] / B);
  stats[2] = (float)(s[1] / B);
  stats[3] = (float)(s[2] / B);
  stats[0] = (float)((s[0] + s[1] + s[2]) / B);
}

inline int warp_grid(long long rows) { return jb_div_up(rows, WARPS); }

inline bool tree_ok(const Tree& t) {
  return t.n && t.w && t.p && t.r && t.child && t.latent && t.count && t.bounds && t.path && t.path_len;
}

}  // namespace

JB_API int jb_muzero_scale_fwd(const float* x, int M, int H, float* y, float* y2, int ld2, void* stream) {
  if (!x || !y || M <= 0 || H <= 0 || H > MZ_MAX_HS || (y2 && ld2 < H)) return JB_ERR_INVALID;
  scale_fwd_kernel<<<warp_grid(M), WARPS * 32, 0, (cudaStream_t)stream>>>(x, M, H, y, y2, ld2);
  return jb_check_launch();
}

JB_API int jb_muzero_scale_bwd(const float* x, const float* dy, int M, int H, float* dx, void* stream) {
  if (!x || !dy || !dx || M <= 0 || H <= 0 || H > MZ_MAX_HS) return JB_ERR_INVALID;
  scale_bwd_kernel<<<warp_grid(M), WARPS * 32, 0, (cudaStream_t)stream>>>(x, dy, M, H, dx);
  return jb_check_launch();
}

JB_API int jb_muzero_support_to_scalar(const float* logits, int M, int V, float* out, void* stream) {
  if (!logits || !out || M <= 0 || V < 1 || V > MZ_MAX_SUPPORT) return JB_ERR_INVALID;
  support_to_scalar_kernel<<<warp_grid(M), WARPS * 32, 0, (cudaStream_t)stream>>>(logits, M, V, out);
  return jb_check_launch();
}

JB_API int jb_muzero_scalar_to_support(const float* x, int M, int V, float* out, void* stream) {
  if (!x || !out || M <= 0 || V < 1 || V > MZ_MAX_SUPPORT) return JB_ERR_INVALID;
  scalar_to_support_kernel<<<jb_div_up((long long)M * (2 * V + 1), 256), 256, 0, (cudaStream_t)stream>>>(x, M, V, out);
  return jb_check_launch();
}

JB_API int jb_mcts_root(const float* pi_logits, const float* v_logits, const float* latent0, int N, int A, int S, int Hs,
                        int V, int training, float dir_alpha, float frac, const double* gamma_in, uint64_t seed,
                        long long* row_ctr, int* edge_n, float* edge_w, float* edge_p, float* edge_r, int* edge_child,
                        float* latent, int* count, float* bounds, int* path, int* path_len, float* root_value,
                        void* stream) {
  const Tree t{edge_n, edge_w, edge_p, edge_r, edge_child, latent, count, bounds, path, path_len};
  if (!pi_logits || !v_logits || !latent0 || !tree_ok(t) || N <= 0 || A < 1 || A > MZ_MAX_A || S < 1 || Hs <= 0 ||
      V < 1 || V > MZ_MAX_SUPPORT || (training && !(dir_alpha > 0.f)))
    return JB_ERR_INVALID;
  mcts_root_kernel<<<warp_grid(N), WARPS * 32, 0, (cudaStream_t)stream>>>(pi_logits, v_logits, latent0, N, A, S, Hs, V,
                                                                           training, dir_alpha, frac, gamma_in, seed,
                                                                           row_ctr, t, root_value);
  return jb_check_launch();
}

JB_API int jb_mcts_select(int N, int A, int S, int Hs, float gamma, int* edge_n, float* edge_w, float* edge_p,
                          float* edge_r, int* edge_child, float* latent, int* count, float* bounds, int* path,
                          int* path_len, int* leaf_node, int* leaf_action, float* dyn_in, void* stream) {
  const Tree t{edge_n, edge_w, edge_p, edge_r, edge_child, latent, count, bounds, path, path_len};
  if (!tree_ok(t) || !leaf_node || !leaf_action || !dyn_in || N <= 0 || A < 1 || A > MZ_MAX_A || S < 1 || Hs <= 0)
    return JB_ERR_INVALID;
  mcts_select_kernel<<<warp_grid(N), WARPS * 32, 0, (cudaStream_t)stream>>>(N, A, S, Hs, gamma, t, leaf_node, leaf_action,
                                                                             dyn_in);
  return jb_check_launch();
}

JB_API int jb_mcts_expand_backup(const float* latent_new, const float* pi_logits, const float* v_logits,
                                 const float* r_logits, int N, int A, int S, int Hs, int V, int R, float gamma,
                                 const int* leaf_node, const int* leaf_action, int* edge_n, float* edge_w, float* edge_p,
                                 float* edge_r, int* edge_child, float* latent, int* count, float* bounds, int* path,
                                 int* path_len, void* stream) {
  const Tree t{edge_n, edge_w, edge_p, edge_r, edge_child, latent, count, bounds, path, path_len};
  if (!latent_new || !pi_logits || !v_logits || !r_logits || !leaf_node || !leaf_action || !tree_ok(t) || N <= 0 ||
      A < 1 || A > MZ_MAX_A || S < 1 || Hs <= 0 || V < 1 || V > MZ_MAX_SUPPORT || R < 1 || R > MZ_MAX_SUPPORT)
    return JB_ERR_INVALID;
  mcts_expand_backup_kernel<<<warp_grid(N), WARPS * 32, 0, (cudaStream_t)stream>>>(
      latent_new, pi_logits, v_logits, r_logits, N, A, S, Hs, V, R, gamma, leaf_node, leaf_action, t);
  return jb_check_launch();
}

JB_API int jb_mcts_act(int N, int A, int S, float gamma, int training, const float* temperature, const double* u_in,
                       uint64_t seed, long long* row_ctr, const int* edge_n, const float* edge_w, const float* edge_r,
                       int64_t* action, float* pi, float* root_value, void* stream) {
  if (!edge_n || !edge_w || !edge_r || !action || !pi || N <= 0 || A < 1 || A > MZ_MAX_A || S < 1 ||
      (training && !temperature))
    return JB_ERR_INVALID;
  Tree t{};
  t.n = const_cast<int*>(edge_n); t.w = const_cast<float*>(edge_w); t.r = const_cast<float*>(edge_r);
  mcts_act_kernel<<<warp_grid(N), WARPS * 32, 0, (cudaStream_t)stream>>>(N, A, S, gamma, training, temperature, u_in, seed,
                                                                          row_ctr, t, action, pi, root_value);
  return jb_check_launch();
}

JB_API int jb_muzero_loss(const float* pi_logits, const float* v_logits, const float* r_logits, const float* reward,
                          const float* done, const float* root_value, const float* policy, const double* weights, int B,
                          int K, int n_step, int A, int V, int R, float gamma, float value_coef, float alpha, float* d_pi,
                          float* d_v, float* d_r, double* prio, float* stats, double* scratch, void* stream) {
  if (!pi_logits || !v_logits || !r_logits || !reward || !done || !root_value || !policy || !d_pi || !d_v || !d_r ||
      !stats || !scratch || B <= 0 || K < 1 || n_step < 1 || A < 1 || A > MZ_MAX_A || V < 1 || V > MZ_MAX_SUPPORT ||
      R < 1 || R > MZ_MAX_SUPPORT)
    return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const int rows = B * (K + 1);
  muzero_loss_kernel<<<warp_grid(rows), WARPS * 32, 0, s>>>(pi_logits, v_logits, r_logits, reward, done, root_value, policy,
                                                            weights, B, K, n_step, A, V, R, gamma, value_coef, alpha,
                                                            1.0 / B, 1.0 / K, d_pi, d_v, d_r, prio, scratch);
  muzero_finalize_kernel<<<1, 32, 0, s>>>(scratch, rows, B, stats);
  return jb_check_launch();
}
