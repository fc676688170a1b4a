// REINFORCE (Williams, 1992) on whole episodes: discounted returns of the completed episodes of a device episode ring,
// their compact row list, and the policy-gradient loss forward + backward of one chunk of rows.
//
// Reference: jorldy/core/agent/reinforce.py learn():
//   ret = reward copied; for t in reversed(range(len(ret) - 1)): ret[t] += gamma * ret[t + 1]
//   with use_standardization: ret = (ret - ret.mean()) / (ret.std() + 1e-7)          (numpy: ddof = 0)
//   discrete:   loss = -(log(pi.gather(1, a)) * ret).mean()
//   continuous: loss = -(Normal(mu, std).log_prob(atanh(clamp(a, +-(1 - 1e-7)))) * ret).mean()   (mean over M*A)
// The reference's buffer holds exactly one episode; here every env row of the ring holds a run of episodes and each
// completed episode gets the reference's returns and statistics on its own.
//
// Ring layout: reward / done [N, L] f32, action int64 [N, L] (discrete) or f32 [N, L, A] (continuous).  `pos` counts
// the steps written so far (step t lives in column t mod L for every env); head[e] is the absolute step of env e's
// oldest unlearned step.  The caller sizes L so that the window [head[e], pos) never exceeds L steps.
//
// No atomics: every reduction runs in a fixed order, so a learn is bit-reproducible.
#include "common.cuh"
#include "ppo_rowmath.cuh"

namespace {

using jbppo::MAX_A;
using jbppo::MAX_A_DISC;

constexpr int LOSS_THREADS = 256;

// The reference's return recurrence over steps [start, end] of one env row (end holds the episode's done), in float64
// with no FMA contraction: G_end = r_end, G_t = r_t + gamma G_{t+1}.
struct EpisodeWalk {
  const float* r;
  int L;
  double gamma;
  __device__ __forceinline__ double step(long long t, double G, bool last) const {
    const double rt = (double)r[t % L];
    return last ? rt : __dadd_rn(rt, __dmul_rn(gamma, G));
  }
};

__global__ void episode_returns_kernel(const float* __restrict__ reward, const float* __restrict__ done, int N, int L,
                                       const long long* __restrict__ pos, long long* __restrict__ head, double gamma,
                                       int standardize, float* __restrict__ ret_ring, int* __restrict__ count) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N) return;
  const long long P = *pos, h = head[e];
  const float* d = done + (size_t)e * L;
  float* out = ret_ring + (size_t)e * L;
  const EpisodeWalk w{reward + (size_t)e * L, L, gamma};
  long long last = -1;                               // the last done in [h, P): every step up to it is complete
  for (long long t = P - 1; t >= h; --t)
    if (d[t % L] != 0.f) { last = t; break; }
  if (last < 0) { count[e] = 0; return; }
  count[e] = (int)(last - h + 1);
  head[e] = last + 1;
  for (long long end = last; end >= h;) {            // episodes newest first; each is [start, end]
    long long start = end;
    while (start > h && d[(start - 1) % L] == 0.f) --start;
    if (!standardize) {
      double G = 0.0;
      for (long long t = end; t >= start; --t) { G = w.step(t, G, t == end); out[t % L] = (float)G; }
    } else {
      const double n = (double)(end - start + 1);
      double G = 0.0, sum = 0.0;
      for (long long t = end; t >= start; --t) { G = w.step(t, G, t == end); sum = __dadd_rn(sum, G); }
      const double mean = sum / n;
      double sq = 0.0;
      for (long long t = end; t >= start; --t) {
        G = w.step(t, G, t == end);
        const double c = __dadd_rn(G, -mean);
        sq = __dadd_rn(sq, __dmul_rn(c, c));
      }
      const double denom = __dadd_rn(sqrt(sq / n), 1e-7);     // std with ddof = 0, as numpy's
      for (long long t = end; t >= start; --t) {
        G = w.step(t, G, t == end);
        out[t % L] = (float)(__dadd_rn(G, -mean) / denom);
      }
    }
    end = start - 1;
  }
}

// One CTA: offsets[e] = sum of count[0..e) (integer, so exact in any order; written in env order), M = the total; the
// rows [M, ceil(M / C) C) of idx / ret are padding (ring row 0, return 0).
constexpr int SCAN_THREADS = 1024;

__global__ void __launch_bounds__(SCAN_THREADS)
episode_scan_kernel(const int* __restrict__ count, int N, int C, int* __restrict__ offsets, int* __restrict__ M_out,
                    int32_t* __restrict__ idx, float* __restrict__ ret) {
  __shared__ long long s_base[SCAN_THREADS];
  const int per = (N + SCAN_THREADS - 1) / SCAN_THREADS;
  const int e0 = threadIdx.x * per, e1 = min(N, e0 + per);
  long long s = 0;
  for (int e = e0; e < e1; ++e) s += count[e];
  s_base[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long acc = 0;
    for (int k = 0; k < SCAN_THREADS; ++k) { const long long v = s_base[k]; s_base[k] = acc; acc += v; }
    *M_out = (int)acc;
  }
  __syncthreads();
  long long o = s_base[threadIdx.x];
  for (int e = e0; e < e1; ++e) { offsets[e] = (int)o; o += count[e]; }
  __syncthreads();
  const long long M = *M_out;
  const long long pad_end = (M + C - 1) / C * C;
  for (long long i = M + threadIdx.x; i < pad_end; i += SCAN_THREADS) { idx[i] = 0; ret[i] = 0.f; }
}

// One warp per env: its count[e] completed rows, oldest first, at offsets[e] of the compact list.
__global__ void episode_gather_kernel(const int* __restrict__ count, const int* __restrict__ offsets,
                                      const long long* __restrict__ head, const float* __restrict__ ret_ring, int N,
                                      int L, int32_t* __restrict__ idx, float* __restrict__ ret) {
  const int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (e >= N) return;
  const int n = count[e], o = offsets[e];
  const long long first = head[e] - n;               // head[e] was advanced past these rows
  for (int i = lane; i < n; i += 32) {
    const int col = (int)((first + i) % L);
    idx[o + i] = e * L + col;
    ret[o + i] = ret_ring[(size_t)e * L + col];
  }
}

// Rows b < C of the chunk k = *cursor - 1 (jb_take_minibatch has advanced the cursor; NULL: chunk 0): ring row
// rows[k C + b], return ret[k C + b]; the head outputs out[b] were computed from the same ring rows.  Rows at or past M
// are padding: their dout row is 0 and they add nothing to the loss.
template <bool CONT, int NA>
__global__ void __launch_bounds__(LOSS_THREADS)
reinforce_loss_kernel(const float* __restrict__ out, const int32_t* __restrict__ rows, const float* __restrict__ ret,
                      const long long* __restrict__ cursor, const int* __restrict__ M_dev, int C,
                      const void* __restrict__ action, int A, int nout, float* __restrict__ dout,
                      float* __restrict__ partials) {
  __shared__ float sred[32];
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float s = 0.f;                                     // sum of log_prob * ret over this CTA's rows (and dims)
  if (b < C) {
    const long long k = cursor ? *cursor - 1 : 0;
    const long long g = k * C + b;
    const int M = *M_dev;
    const bool valid = g < M;
    const int r = rows[g];
    const float R = valid ? ret[g] : 0.f;
    const float* o = out + (size_t)b * nout;
    float* gd = dout + (size_t)b * nout;
    if constexpr (!CONT) {
      const int a_t = (int)((const int64_t*)action)[r];
      float lg[NA], lsm[NA];
#pragma unroll
      for (int a = 0; a < NA; ++a) lg[a] = a < A ? o[a] : 0.f;
      jbppo::log_softmax_row<NA>(lg, A, lsm);
      const float coef = valid ? -(R / (float)M) : 0.f;     // d loss / d log pi(a_t)
      float la = 0.f;
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        if (a < A) {
          if (a == a_t) la = lsm[a];
          gd[a] = coef * ((a == a_t ? 1.f : 0.f) - expf(lsm[a]));
        }
      }
      if (valid) s = la * R;
    } else {
      const float* act = (const float*)action + (size_t)r * A;
      const float coef = valid ? -(R / ((float)M * (float)A)) : 0.f;
      for (int a = 0; a < A; ++a) {
        const float mu = fminf(fmaxf(o[a], -5.f), 5.f);
        const float ls = tanhf(o[A + a]);
        const float sd = expf(ls);
        const float z = jbppo::atanh_clamped(act[a]);
        if (valid) s += jbppo::normal_logpdf(z, mu, sd) * R;
        const float dz = z - mu, var = sd * sd;
        const float in_mu = (o[a] >= -5.f && o[a] <= 5.f) ? 1.f : 0.f;   // torch.clamp's backward passes at the bounds
        gd[a] = coef * (dz / var) * in_mu;
        gd[A + a] = coef * (dz * dz / (var * sd) - 1.f / sd) * sd * (1.f - ls * ls);
      }
    }
  }
  float v[1] = {s};
  jbppo::block_sum<1>(v, sred);
  if (threadIdx.x == 0) partials[blockIdx.x] = v[0];
}

// One thread folds the per-CTA partials in CTA order: acc[0] += -(sum) / (M [* A]) (this chunk's share of the loss),
// acc[1] += 1 (chunks).  M <= 0 adds nothing.
__global__ void reinforce_fold_kernel(const float* __restrict__ partials, int n_cta, const int* __restrict__ M_dev,
                                      int A, int cont, float* __restrict__ acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int M = *M_dev;
  if (M <= 0) return;
  float s = 0.f;
  for (int k = 0; k < n_cta; ++k) s += partials[k];
  acc[0] += -s / ((float)M * (cont ? (float)A : 1.f));
  acc[1] += 1.f;
}

__global__ void add_f32_kernel(float* __restrict__ y, const float* __restrict__ x, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] += x[i];
}

}  // namespace

JB_API int jb_episode_returns(const float* reward, const float* done, int N, int L, const long long* pos, long long* head,
                              double gamma, int standardize, float* ret_ring, int* count, void* stream) {
  if (!reward || !done || !pos || !head || !ret_ring || !count || N <= 0 || L <= 0) return JB_ERR_INVALID;
  episode_returns_kernel<<<jb_div_up(N, 128), 128, 0, (cudaStream_t)stream>>>(reward, done, N, L, pos, head, gamma,
                                                                              standardize, ret_ring, count);
  return jb_check_launch();
}

JB_API int jb_episode_rows(const int* count, const long long* head, const float* ret_ring, int N, int L, int C,
                           int* offsets, int32_t* idx, float* ret, int* M, void* stream) {
  if (!count || !head || !ret_ring || !offsets || !idx || !ret || !M || N <= 0 || L <= 0 || C <= 0) return JB_ERR_INVALID;
  if ((long long)N * L + C > 0x7fffffffLL) return JB_ERR_INVALID;      // int32 row indices and counts
  cudaStream_t s = (cudaStream_t)stream;
  episode_scan_kernel<<<1, SCAN_THREADS, 0, s>>>(count, N, C, offsets, M, idx, ret);
  episode_gather_kernel<<<jb_div_up(N, 8), 256, 0, s>>>(count, offsets, head, ret_ring, N, L, idx, ret);
  return jb_check_launch();
}

JB_API int jb_reinforce_loss_partials(int C) { return C > 0 ? jb_div_up(C, LOSS_THREADS) : JB_ERR_INVALID; }

JB_API int jb_reinforce_loss(int continuous, const float* out, const int32_t* rows, const float* ret,
                             const long long* cursor, const int* M, int C, const void* action, int A, int nout,
                             float* dout, float* partials, float* acc, void* stream) {
  if (!out || !rows || !ret || !M || !action || !dout || !partials || !acc) return JB_ERR_INVALID;
  if (C <= 0 || A <= 0 || A > (continuous ? MAX_A : MAX_A_DISC) || nout != (continuous ? 2 * A : A)) return JB_ERR_INVALID;
  const int n_cta = jb_div_up(C, LOSS_THREADS);
  cudaStream_t s = (cudaStream_t)stream;
  if (continuous)
    reinforce_loss_kernel<true, MAX_A><<<n_cta, LOSS_THREADS, 0, s>>>(out, rows, ret, cursor, M, C, action, A, nout, dout, partials);
  else if (A <= MAX_A)
    reinforce_loss_kernel<false, MAX_A><<<n_cta, LOSS_THREADS, 0, s>>>(out, rows, ret, cursor, M, C, action, A, nout, dout, partials);
  else
    reinforce_loss_kernel<false, MAX_A_DISC><<<n_cta, LOSS_THREADS, 0, s>>>(out, rows, ret, cursor, M, C, action, A, nout, dout, partials);
  reinforce_fold_kernel<<<1, 32, 0, s>>>(partials, n_cta, M, A, continuous, acc);
  return jb_check_launch();
}

JB_API int jb_add_f32(float* y, const float* x, long long n, void* stream) {
  if (!y || !x || n <= 0) return JB_ERR_INVALID;
  add_f32_kernel<<<jb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(y, x, n);
  return jb_check_launch();
}
