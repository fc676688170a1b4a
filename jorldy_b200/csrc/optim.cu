// Optimiser step over ONE flat fp32 parameter buffer: global-norm clipping fused with Adam or
// centred RMSprop.  Streaming HBM kernels: 28 B/param/step (Adam: read p,g,m,v; write p,m,v),
// 32 B/param/step (centred RMSprop).
//
// Reference call sites: torch.nn.utils.clip_grad_norm_ (ppo.py:166-168, ape_x.py:119),
// torch.optim.Adam via jorldy/core/optimizer/__init__.py:31 (ppo.py:169, dqn.py:141,
// rainbow.py:239), torch.optim.RMSprop(centered) for config/ape_x/*.py.  torch itself is
// third-party (requirements.txt:10); its update rules are restated here:
//   clip : coef = min(1, max_norm / (||g||_2 + 1e-6));  g <- g * coef
//   Adam : m <- m + (g - m)(1-b1);  v <- b2 v + (1-b2) g^2;
//          p <- p - (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
//   RMSprop(centered): s <- a s + (1-a) g^2;  ga <- ga + (g - ga)(1-a);
//          p <- p - lr * g / (sqrt(s - ga^2) + eps)
// The reference launches ~10 ATen kernels per parameter tensor (8 tensors) per step; here it is two
// launches per step regardless of the number of tensors: per-CTA sum-of-squares partials, then
// the update, in which every CTA folds the (<= 1184) partials in a fixed order (deterministic).
// `step` and `lr` live in device memory so a captured CUDA graph can be replayed unchanged.
#include "common.cuh"

namespace {

constexpr int NORM_THREADS = 256;

__global__ void __launch_bounds__(NORM_THREADS)
grad_sumsq_kernel(const float* __restrict__ g, long long P, float* __restrict__ partials, long long* __restrict__ step) {
  __shared__ float sw[NORM_THREADS / 32];
  float acc = 0.f;
  const long long n4 = P >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = g4[i];
    acc = fmaf(v.x, v.x, acc); acc = fmaf(v.y, v.y, acc); acc = fmaf(v.z, v.z, acc); acc = fmaf(v.w, v.w, acc);
  }
  if (blockIdx.x == 0 && threadIdx.x < (P & 3)) { const float v = g[(n4 << 2) + threadIdx.x]; acc = fmaf(v, v, acc); }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < NORM_THREADS / 32; ++w) t += sw[w];
    partials[blockIdx.x] = t;
    if (blockIdx.x == 0 && step) *step += 1;
  }
}

// Every CTA folds the per-CTA partials: thread-strided loads (all in flight at once), f64
// butterfly per warp, then a fixed-order fold of the warp sums — identical in every CTA and run.
// Must be called by all threads of a 256-thread block.
__device__ __forceinline__ float clip_coef_from_partials(const float* __restrict__ partials, int n_partials,
                                                         float max_norm, float* norm_out) {
  __shared__ double s_w[8];
  __shared__ float s_coef;
  double t = 0.0;
  for (int k = threadIdx.x; k < n_partials; k += 256) t += (double)partials[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += s_w[w];
    const float total_norm = (float)sqrt(tot);
    if (norm_out) *norm_out = total_norm;
    float c = 1.f;
    if (max_norm > 0.f) { c = max_norm / (total_norm + 1e-6f); c = c < 1.f ? c : 1.f; }
    s_coef = c;
  }
  __syncthreads();
  return s_coef;
}

// 1 - beta is rounded from the double value (as torch forms it), not computed from the rounded fp32 beta: for
// beta2 = 0.999 the latter is off by 1.3e-5 relative.  The bias corrections use the double betas too.
struct AdamHP { float b1, b2, one_m_b1, one_m_b2, eps, max_norm; double b1d, b2d; };

__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            long long P, const float* __restrict__ lr_ptr, AdamHP hp, const long long* __restrict__ step_ptr,
            const float* __restrict__ partials, int n_partials, float* __restrict__ norm_out) {
  const float coef = clip_coef_from_partials(partials, n_partials, hp.max_norm, blockIdx.x == 0 ? norm_out : nullptr);
  const double t = (double)(*step_ptr);
  const double bc1 = 1.0 - pow(hp.b1d, t);
  const double bc2 = 1.0 - pow(hp.b2d, t);
  const float step_size = (float)((double)(*lr_ptr) / bc1);
  const float bc2_sqrt = (float)sqrt(bc2);
  const float one_m_b1 = hp.one_m_b1, one_m_b2 = hp.one_m_b2;

  auto upd = [&](float& pp, float gg, float& mm, float& vv) {
    gg *= coef;
    mm = fmaf(gg - mm, one_m_b1, mm);
    vv = fmaf(one_m_b2 * gg, gg, hp.b2 * vv);
    const float denom = sqrtf(vv) / bc2_sqrt + hp.eps;
    pp = fmaf(-step_size, mm / denom, pp);
  };
  const long long n4 = P >> 2;
  float4* p4 = reinterpret_cast<float4*>(p);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 pp = p4[i], mm = m4[i], vv = v4[i];
    const float4 gg = g4[i];
    upd(pp.x, gg.x, mm.x, vv.x); upd(pp.y, gg.y, mm.y, vv.y); upd(pp.z, gg.z, mm.z, vv.z); upd(pp.w, gg.w, mm.w, vv.w);
    p4[i] = pp; m4[i] = mm; v4[i] = vv;
  }
  if (blockIdx.x == 0 && threadIdx.x < (P & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    upd(p[i], g[i], m[i], v[i]);
  }
}

struct RmsHP { float alpha, one_m_alpha, eps, max_norm; };

__global__ void __launch_bounds__(256)
rmsprop_centered_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ sq,
                        float* __restrict__ ga, long long P, const float* __restrict__ lr_ptr, RmsHP hp,
                        const float* __restrict__ partials, int n_partials, float* __restrict__ norm_out) {
  const float coef = clip_coef_from_partials(partials, n_partials, hp.max_norm, blockIdx.x == 0 ? norm_out : nullptr);
  const float lr = *lr_ptr;
  const float one_m_a = hp.one_m_alpha;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
    const float gg = g[i] * coef;
    float s = sq[i], a = ga[i];
    s = fmaf(one_m_a * gg, gg, hp.alpha * s);
    a = fmaf(gg - a, one_m_a, a);
    const float avg = sqrtf(fmaf(-a, a, s)) + hp.eps;
    p[i] = fmaf(-lr, gg / avg, p[i]);
    sq[i] = s; ga[i] = a;
  }
}

__global__ void copy_kernel(float* __restrict__ dst, const float* __restrict__ src, long long P) {
  const long long n4 = P >> 2;
  float4* d4 = reinterpret_cast<float4*>(dst);
  const float4* s4 = reinterpret_cast<const float4*>(src);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) d4[i] = s4[i];
  if (blockIdx.x == 0 && threadIdx.x < (P & 3)) dst[(n4 << 2) + threadIdx.x] = src[(n4 << 2) + threadIdx.x];
}

}  // namespace

static int norm_blocks(long long P) {
  long long b = (P / 4 + NORM_THREADS - 1) / NORM_THREADS;
  if (b < 1) b = 1;
  if (b > 4 * JB_SM_COUNT) b = 4 * JB_SM_COUNT;
  return (int)b;
}

// Number of partial slots jb_grad_sumsq writes for a buffer of P floats (size the scratch with it).
JB_API int jb_grad_partials_count(long long P) { return norm_blocks(P); }

// partials[k] = sum of squares of CTA k's slice of g; *step += 1 (step may be NULL).
JB_API int jb_grad_sumsq(const float* g, long long P, float* partials, long long* step, void* stream) {
  if (!g || !partials || P <= 0) return JB_ERR_INVALID;
  grad_sumsq_kernel<<<norm_blocks(P), NORM_THREADS, 0, (cudaStream_t)stream>>>(g, P, partials, step);
  return jb_check_launch();
}

// max_norm <= 0 disables clipping.  norm_out (device float, may be NULL) receives ||g||_2.
JB_API int jb_adam_step(float* p, const float* g, float* m, float* v, long long P, const float* lr, double beta1,
                        double beta2, float eps, const long long* step, const float* partials, int n_partials,
                        float max_norm, float* norm_out, void* stream) {
  if (!p || !g || !m || !v || !lr || !step || P <= 0) return JB_ERR_INVALID;
  if (max_norm > 0.f && (!partials || n_partials <= 0)) return JB_ERR_INVALID;
  AdamHP hp{(float)beta1, (float)beta2, (float)(1.0 - beta1), (float)(1.0 - beta2), eps, partials ? max_norm : 0.f,
            beta1, beta2};
  int blocks = jb_grid_for(P / 4 + 1, 256, 2);
  adam_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(p, g, m, v, P, lr, hp, step, partials, partials ? n_partials : 0, norm_out);
  return jb_check_launch();
}

JB_API int jb_rmsprop_centered_step(float* p, const float* g, float* square_avg, float* grad_avg, long long P,
                                    const float* lr, double alpha, float eps, const float* partials, int n_partials,
                                    float max_norm, float* norm_out, void* stream) {
  if (!p || !g || !square_avg || !grad_avg || !lr || P <= 0) return JB_ERR_INVALID;
  if (max_norm > 0.f && (!partials || n_partials <= 0)) return JB_ERR_INVALID;
  RmsHP hp{(float)alpha, (float)(1.0 - alpha), eps, partials ? max_norm : 0.f};
  int blocks = jb_grid_for(P, 256 * 4, 2);
  rmsprop_centered_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(p, g, square_avg, grad_avg, P, lr, hp, partials,
                                                                  partials ? n_partials : 0, norm_out);
  return jb_check_launch();
}

// Hard target-network update (dqn.py:153-154 load_state_dict) as one streaming copy of the flat buffer.
JB_API int jb_copy_f32(float* dst, const float* src, long long P, void* stream) {
  if (!dst || !src || P <= 0) return JB_ERR_INVALID;
  copy_kernel<<<jb_grid_for(P / 4 + 1, 256, 4), 256, 0, (cudaStream_t)stream>>>(dst, src, P);
  return jb_check_launch();
}
