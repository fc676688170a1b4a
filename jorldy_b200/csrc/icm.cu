// ICM-PPO (Pathak et al., ICML 2017, "Curiosity-driven Exploration by Self-supervised Prediction") on the PPO rollout
// path: the fused ICM loss, training-mode BatchNorm1d + ELU, and the running statistics that normalise the observations
// and the intrinsic reward.  The ICM's dense layers are the existing GEMMs (csrc/linear.cu).
//
// Every reduction runs in a fixed order with no atomics, so each entry point is bit-reproducible run to run:
//   - column reductions (BatchNorm batch moments and their backward sums, RunningMeanStd batch moments) are split into
//     chunks of COL_ROWS rows; a CTA writes one chunk's float64 partial sums per column and a fold kernel adds the chunks
//     in chunk order, so the same code serves a 2-row minibatch and the 524 288-row rollout of the pre-pass;
//   - the ICM loss gives each row one warp (xor-shuffle sums), each CTA ICM_ROWS rows, and folds the per-CTA partials
//     with one thread in CTA order.
#include "common.cuh"

namespace {

constexpr int COL_ROWS = 256;      // rows per column-reduction chunk
constexpr int ICM_F = 256;         // ICM feature width (8 floats per lane)
constexpr int ICM_ROWS = 8;        // rows (warps) per ICM loss CTA
constexpr int ICM_MAX_A_DISC = 18;
constexpr int ICM_MAX_A_CONT = 8;

__device__ __forceinline__ float elu(float u) { return u > 0.f ? u : expm1f(u); }
// ELU'(u) from y = ELU(u): 1 for u > 0, exp(u) = y + 1 otherwise
__device__ __forceinline__ float elu_grad_from_y(float y) { return y > 0.f ? 1.f : y + 1.f; }

// ---- column reductions ---------------------------------------------------------------------------------------------
// part[(chunk * 2 + q) * N + c], q = 0: sum_r a(r, c), q = 1: sum_r a(r, c) * b(r, c) over the chunk's rows; b NULL
// means b = a (sum of squares).  Block (32, 8): 32 columns, 8 row lanes folded in lane order.
__global__ void __launch_bounds__(256)
colsum2_partial_kernel(const float* __restrict__ a, int lda, const float* __restrict__ b, int ldb, int M, int N,
                       double* __restrict__ part) {
  __shared__ double s[2][8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int r0 = blockIdx.y * COL_ROWS, r1 = min(M, r0 + COL_ROWS);
  double s0 = 0.0, s1 = 0.0;
  if (c < N) {
    for (int r = r0 + threadIdx.y; r < r1; r += 8) {
      const double x = a[(size_t)r * lda + c];
      s0 += x;
      s1 += x * (b ? (double)b[(size_t)r * ldb + c] : x);
    }
  }
  s[0][threadIdx.y][threadIdx.x] = s0;
  s[1][threadIdx.y][threadIdx.x] = s1;
  __syncthreads();
  if (threadIdx.y < 2 && c < N) {
    double t = 0.0;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += s[threadIdx.y][y][threadIdx.x];
    part[((size_t)blockIdx.y * 2 + threadIdx.y) * N + c] = t;
  }
}

__device__ __forceinline__ void fold_chunks(const double* __restrict__ part, int n_chunks, int N, int c, double& s0,
                                            double& s1) {
  s0 = 0.0; s1 = 0.0;
  for (int k = 0; k < n_chunks; ++k) {
    s0 += part[((size_t)k * 2) * N + c];
    s1 += part[((size_t)k * 2 + 1) * N + c];
  }
}

// ---- BatchNorm1d (training mode) + ELU -------------------------------------------------------------------------------
// Batch mean / biased variance per column, the running buffers updated as torch does (unbiased variance, momentum),
// num_batches_tracked += 1.
__global__ void bn_stats_kernel(const double* __restrict__ part, int n_chunks, int M, int N, float momentum, float eps,
                                float* __restrict__ running_mean, float* __restrict__ running_var,
                                int64_t* __restrict__ nbt, float* __restrict__ mean, float* __restrict__ invstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0) nbt[0] += 1;
  if (c >= N) return;
  double s0, s1;
  fold_chunks(part, n_chunks, N, c, s0, s1);
  const double mu = s0 / M;
  const double var = fmax(s1 / M - mu * mu, 0.0);
  mean[c] = (float)mu;
  invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mu;
  running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)(var * M / (M - 1));
}

// y = ELU(gamma (x - mean) invstd + beta), or ELU(x) when gamma is NULL; also written to y2 when it is not NULL
__global__ void bn_elu_apply_kernel(const float* __restrict__ x, int M, int N, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, const float* __restrict__ mean,
                                    const float* __restrict__ invstd, float* __restrict__ y, int ldy,
                                    float* __restrict__ y2, int ldy2) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * N) return;
  const int r = (int)(i / N), c = (int)(i % N);
  float u = x[i];
  if (gamma) u = gamma[c] * ((u - mean[c]) * invstd[c]) + beta[c];
  const float v = elu(u);
  y[(size_t)r * ldy + c] = v;
  if (y2) y2[(size_t)r * ldy2 + c] = v;
}

// g = dy ELU'(u); BN off: dx = g.  BN on: g is written to dx first and rewritten by bn_bwd_apply_kernel.
__global__ void elu_bwd_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ y, int ldy, int M, int N,
                               float* __restrict__ dx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * N) return;
  const int r = (int)(i / N), c = (int)(i % N);
  dx[i] = dy[(size_t)r * lddy + c] * elu_grad_from_y(y[(size_t)r * ldy + c]);
}

// xhat = (x - mean) invstd, the operand of the d gamma sum
__global__ void bn_xhat_kernel(const float* __restrict__ x, int M, int N, const float* __restrict__ mean,
                               const float* __restrict__ invstd, float* __restrict__ xhat) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * N) return;
  const int c = (int)(i % N);
  xhat[i] = (x[i] - mean[c]) * invstd[c];
}

__global__ void bn_bwd_fold_kernel(const double* __restrict__ part, int n_chunks, int N, float* __restrict__ dgamma,
                                   float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  double s0, s1;
  fold_chunks(part, n_chunks, N, c, s0, s1);
  dbeta[c] = (float)s0;
  dgamma[c] = (float)s1;
}

// dx = gamma invstd (g - dbeta / M - xhat dgamma / M), g read from dx
__global__ void bn_bwd_apply_kernel(const float* __restrict__ xhat, int M, int N, const float* __restrict__ gamma,
                                    const float* __restrict__ invstd, const float* __restrict__ dgamma,
                                    const float* __restrict__ dbeta, float* __restrict__ dx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * N) return;
  const int c = (int)(i % N);
  const float invM = 1.f / (float)M;
  dx[i] = gamma[c] * invstd[c] * (dx[i] - dbeta[c] * invM - xhat[i] * (dgamma[c] * invM));
}

// ---- RunningMeanStd (OpenAI baselines): float64 state, batch moments merged with the parallel formula -----------------
// One CTA; count is read by every column before thread 0 writes the new count.
__global__ void rms_merge_kernel(const double* __restrict__ part, int n_chunks, int M, int D, double* __restrict__ mean,
                                 double* __restrict__ var, double* __restrict__ count) {
  const double n_a = count[0], n_b = (double)M, tot = n_a + n_b;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    double s0, s1;
    fold_chunks(part, n_chunks, D, c, s0, s1);
    const double bm = s0 / n_b;
    const double bv = fmax(s1 / n_b - bm * bm, 0.0);
    const double delta = bm - mean[c];
    const double m2 = var[c] * n_a + bv * n_b + delta * delta * n_a * n_b / tot;
    mean[c] = mean[c] + delta * n_b / tot;
    var[c] = m2 / tot;
  }
  __syncthreads();
  if (threadIdx.x == 0) count[0] = tot;
}

__global__ void rms_normalize_kernel(const float* __restrict__ x, const int32_t* __restrict__ idx, int M, int D,
                                     const double* __restrict__ mean, const double* __restrict__ var, float clip,
                                     float* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * D) return;
  const int m = (int)(i / D), d = (int)(i % D);
  const int r = idx ? idx[m] : m;
  const float v = x[(size_t)r * D + d];
  if (!mean) { y[i] = v; return; }
  const double z = ((double)v - mean[d]) / sqrt(var[d]);
  y[i] = (float)fmin(fmax(z, -(double)clip), (double)clip);
}

// ---- intrinsic reward: the reward-forward filter, its RunningMeanStd and the reward jb_gae reads --------------------
__global__ void reward_filter_kernel(const float* __restrict__ ri, int N, int T, float gamma, float* __restrict__ rewems,
                                     float* __restrict__ filt) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float e = rewems[n];
  for (int t = 0; t < T; ++t) {
    e = gamma * e + ri[(size_t)n * T + t];
    filt[(size_t)n * T + t] = e;
  }
  rewems[n] = e;
}

__global__ void reward_mix_kernel(const float* __restrict__ reward, const float* __restrict__ ri, long long n,
                                  const double* __restrict__ var, float ext_coef, float int_coef, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float scale = var ? (float)(sqrt(var[0]) + 1e-7) : 1.f;
  out[i] = ext_coef * reward[i] + int_coef * (ri[i] / scale);
}

// ---- the ICM loss ------------------------------------------------------------------------------------------------------
// One warp per row: lane l holds feature columns l + 32 j.  Partials per CTA: sum r_i, sum (f - phi')^2, sum l_i rows.
template <bool CONT>
__global__ void __launch_bounds__(32 * ICM_ROWS)
icm_loss_kernel(const float* __restrict__ f, const float* __restrict__ phi_next, int ld_next, const float* __restrict__ g,
                const int32_t* __restrict__ idx, const void* __restrict__ action, int B, int A, float eta, float beta,
                float* __restrict__ ri, float* __restrict__ df, float* __restrict__ dg, float* __restrict__ stats) {
  __shared__ float sp[3][ICM_ROWS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * ICM_ROWS + warp;
  float p_ri = 0.f, p_sq = 0.f, p_li = 0.f;
  if (b < B) {
    const float* fr = f + (size_t)b * ICM_F;
    const float* pr = phi_next + (size_t)b * ld_next;
    const float cf = 2.f * beta / ((float)B * (float)ICM_F);
    float sa = 0.f, sq = 0.f;
#pragma unroll
    for (int j = 0; j < ICM_F / 32; ++j) {
      const int c = lane + 32 * j;
      const float d = fr[c] - pr[c];
      sa += fabsf(d);
      sq += d * d;
      if (df) df[(size_t)b * ICM_F + c] = cf * d;
    }
    sa = jb_warp_sum(sa);
    sq = jb_warp_sum(sq);
    p_ri = 0.5f * eta * sa;
    p_sq = sq;
    if (ri && lane == 0) ri[b] = p_ri;
    if (dg) {
      const int r = idx ? idx[b] : b;
      const float gv = lane < A ? g[(size_t)b * A + lane] : 0.f;
      if constexpr (CONT) {
        const float d = lane < A ? gv - ((const float*)action)[(size_t)r * A + lane] : 0.f;
        p_li = jb_warp_sum(d * d);
        if (lane < A) dg[(size_t)b * A + lane] = (1.f - beta) * 2.f * d / ((float)B * (float)A);
      } else {
        const int a = ((const int32_t*)action)[r];
        const float mx = jb_warp_max(lane < A ? gv : -INFINITY);
        const float e = lane < A ? expf(gv - mx) : 0.f;
        const float s = jb_warp_sum(e);
        const float ga = __shfl_sync(0xffffffffu, gv, a & 31);
        p_li = -(ga - mx - logf(s));
        if (lane < A) dg[(size_t)b * A + lane] = (1.f - beta) * (e / s - (lane == a ? 1.f : 0.f)) / (float)B;
      }
    }
  }
  if (!stats) return;
  if (lane == 0) { sp[0][warp] = p_ri; sp[1][warp] = p_sq; sp[2][warp] = p_li; }
  __syncthreads();
  if (threadIdx.x < 3) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < ICM_ROWS; ++w) t += sp[threadIdx.x][w];
    stats[4 + 3 * blockIdx.x + threadIdx.x] = t;
  }
}

// stats[0..3] = mean r_i, l_f, l_i, beta l_f + (1 - beta) l_i;  acc[0..2] += stats[0..2], acc[3] += 1
__global__ void icm_finalize_kernel(float* __restrict__ stats, int n_cta, int B, int A, int cont, float beta,
                                    float* __restrict__ acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float s_ri = 0.f, s_sq = 0.f, s_li = 0.f;
  for (int k = 0; k < n_cta; ++k) {
    const float* p = stats + 4 + 3 * k;
    s_ri += p[0]; s_sq += p[1]; s_li += p[2];
  }
  const float l_f = s_sq / ((float)B * (float)ICM_F);
  const float l_i = cont ? s_li / ((float)B * (float)A) : s_li / (float)B;
  stats[0] = s_ri / (float)B;
  stats[1] = l_f;
  stats[2] = l_i;
  stats[3] = beta * l_f + (1.f - beta) * l_i;
  if (acc) { acc[0] += stats[0]; acc[1] += l_f; acc[2] += l_i; acc[3] += 1.f; }
}

__global__ void action_rows_kernel(const void* __restrict__ action, const int32_t* __restrict__ idx, int M, int A, int cont,
                                   float* __restrict__ dst, int ld) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * A) return;
  const int m = (int)(i / A), k = (int)(i % A);
  const int r = idx ? idx[m] : m;
  dst[(size_t)m * ld + k] = cont ? ((const float*)action)[(size_t)r * A + k]
                                 : (((const int32_t*)action)[r] == k ? 1.f : 0.f);
}

__global__ void scale_kernel(float* __restrict__ x, long long n, float s) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] *= s;
}

int launch_colsum2(const float* a, int lda, const float* b, int ldb, int M, int N, double* part, cudaStream_t s) {
  dim3 grid(jb_div_up(N, 32), jb_div_up(M, COL_ROWS));
  colsum2_partial_kernel<<<grid, dim3(32, 8), 0, s>>>(a, lda, b, ldb, M, N, part);
  return jb_div_up(M, COL_ROWS);
}

int elementwise_grid(long long n) { return jb_div_up(n, 256); }

}  // namespace

JB_API int jb_col_partials_doubles(int M, int N) {
  return M <= 0 || N <= 0 ? JB_ERR_INVALID : 2 * jb_div_up(M, COL_ROWS) * N;
}

JB_API int jb_bn_elu_fwd(const float* x, int M, int N, const float* gamma, const float* beta, float* running_mean,
                         float* running_var, int64_t* num_batches_tracked, float momentum, float eps, float* mean,
                         float* invstd, double* partials, float* y, int ldy, float* y2, int ldy2, void* stream) {
  if (!x || !y || M <= 0 || N <= 0 || ldy < N || (y2 && ldy2 < N)) return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  if (gamma) {
    if (M < 2 || !beta || !running_mean || !running_var || !num_batches_tracked || !mean || !invstd || !partials)
      return JB_ERR_INVALID;
    const int n_chunks = launch_colsum2(x, N, nullptr, 0, M, N, partials, s);
    bn_stats_kernel<<<jb_div_up(N, 256), 256, 0, s>>>(partials, n_chunks, M, N, momentum, eps, running_mean, running_var,
                                                     num_batches_tracked, mean, invstd);
  }
  bn_elu_apply_kernel<<<elementwise_grid((long long)M * N), 256, 0, s>>>(x, M, N, gamma, beta, mean, invstd, y, ldy, y2,
                                                                          ldy2);
  return jb_check_launch();
}

JB_API int jb_bn_elu_bwd(const float* dy, int lddy, const float* y, int ldy, const float* x, int M, int N,
                         const float* gamma, const float* mean, const float* invstd, float* xhat, double* partials,
                         float* dx, float* dgamma, float* dbeta, void* stream) {
  if (!dy || !y || !dx || M <= 0 || N <= 0 || lddy < N || ldy < N) return JB_ERR_INVALID;
  if (gamma && (M < 2 || !x || !mean || !invstd || !xhat || !partials || !dgamma || !dbeta)) return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = elementwise_grid((long long)M * N);
  elu_bwd_kernel<<<grid, 256, 0, s>>>(dy, lddy, y, ldy, M, N, dx);
  if (gamma) {
    bn_xhat_kernel<<<grid, 256, 0, s>>>(x, M, N, mean, invstd, xhat);
    const int n_chunks = launch_colsum2(dx, N, xhat, N, M, N, partials, s);
    bn_bwd_fold_kernel<<<jb_div_up(N, 256), 256, 0, s>>>(partials, n_chunks, N, dgamma, dbeta);
    bn_bwd_apply_kernel<<<grid, 256, 0, s>>>(xhat, M, N, gamma, invstd, dgamma, dbeta, dx);
  }
  return jb_check_launch();
}

JB_API int jb_rms_update(const float* x, int M, int D, double* mean, double* var, double* count, double* partials,
                         void* stream) {
  if (!x || !mean || !var || !count || !partials || M <= 0 || D <= 0 || D > 1024) return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const int n_chunks = launch_colsum2(x, D, nullptr, 0, M, D, partials, s);
  rms_merge_kernel<<<1, 256, 0, s>>>(partials, n_chunks, M, D, mean, var, count);
  return jb_check_launch();
}

JB_API int jb_rms_normalize(const float* x, const int32_t* idx, int M, int D, const double* mean, const double* var,
                            float clip, float* y, void* stream) {
  if (!x || !y || M <= 0 || D <= 0 || (!mean) != (!var)) return JB_ERR_INVALID;
  rms_normalize_kernel<<<elementwise_grid((long long)M * D), 256, 0, (cudaStream_t)stream>>>(x, idx, M, D, mean, var,
                                                                                            clip, y);
  return jb_check_launch();
}

JB_API int jb_icm_reward(const float* reward, const float* ri, int N, int T, float gamma, int normalize, float* rewems,
                         double* rms_mean, double* rms_var, double* rms_count, double* partials, float* filt,
                         float ext_coef, float int_coef, float* out, void* stream) {
  if (!reward || !ri || !out || N <= 0 || T <= 0) return JB_ERR_INVALID;
  if (normalize && (!rewems || !rms_mean || !rms_var || !rms_count || !partials || !filt)) return JB_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const long long NT = (long long)N * T;
  if (normalize) {
    reward_filter_kernel<<<jb_div_up(N, 128), 128, 0, s>>>(ri, N, T, gamma, rewems, filt);
    const int n_chunks = launch_colsum2(filt, 1, nullptr, 0, (int)NT, 1, partials, s);
    rms_merge_kernel<<<1, 32, 0, s>>>(partials, n_chunks, (int)NT, 1, rms_mean, rms_var, rms_count);
  }
  reward_mix_kernel<<<elementwise_grid(NT), 256, 0, s>>>(reward, ri, NT, normalize ? rms_var : nullptr, ext_coef,
                                                          int_coef, out);
  return jb_check_launch();
}

JB_API int jb_icm_loss(int continuous, const float* f, const float* phi_next, int ld_next, const float* g,
                       const int32_t* idx, const void* action, int B, int A, int F, float eta, float beta, float* ri,
                       float* df, float* dg, float* stats, float* acc, void* stream) {
  if (!f || !phi_next || B <= 0 || F != ICM_F || ld_next < F) return JB_ERR_INVALID;
  const bool reward_only = !df && !dg;
  if (reward_only) {
    if (!ri) return JB_ERR_INVALID;
  } else if (!df || !dg || !g || !action || !stats || A <= 0 ||
             A > (continuous ? ICM_MAX_A_CONT : ICM_MAX_A_DISC)) {
    return JB_ERR_INVALID;
  }
  if (reward_only) stats = nullptr;
  const int n_cta = jb_div_up(B, ICM_ROWS);
  cudaStream_t s = (cudaStream_t)stream;
  if (continuous)
    icm_loss_kernel<true><<<n_cta, 32 * ICM_ROWS, 0, s>>>(f, phi_next, ld_next, g, idx, action, B, A, eta, beta, ri, df, dg, stats);
  else
    icm_loss_kernel<false><<<n_cta, 32 * ICM_ROWS, 0, s>>>(f, phi_next, ld_next, g, idx, action, B, A, eta, beta, ri, df, dg, stats);
  if (stats) icm_finalize_kernel<<<1, 32, 0, s>>>(stats, n_cta, B, A, continuous, beta, acc);
  return jb_check_launch();
}

JB_API int jb_icm_action_rows(int continuous, const void* action, const int32_t* idx, int M, int A, float* dst, int ld,
                              void* stream) {
  if (!action || !dst || M <= 0 || A <= 0 || ld < A) return JB_ERR_INVALID;
  action_rows_kernel<<<elementwise_grid((long long)M * A), 256, 0, (cudaStream_t)stream>>>(action, idx, M, A, continuous,
                                                                                           dst, ld);
  return jb_check_launch();
}

JB_API int jb_scale_f32(float* x, long long n, float s, void* stream) {
  if (!x || n <= 0) return JB_ERR_INVALID;
  scale_kernel<<<elementwise_grid(n), 256, 0, (cudaStream_t)stream>>>(x, n, s);
  return jb_check_launch();
}
