// Thin "edge" layers of the MLP networks: the D_in -> H input layer (fused with the minibatch
// row gather) and the narrow output heads (H -> a few units), forward and backward.
//
// Reference modules: jorldy/core/network/head.py:6-18 (MLP head: relu(Linear(D_in,H))),
// policy_value.py:11-22,41-57 (pi/mu/log_std/v heads), q_network.py:13-20 (q head),
// dueling.py:13-32 (l2_a / l2_v).  These layers have one tiny dimension (D_in = 1..32,
// outputs = 1..8), so a tiled GEMM would waste >85 % of every tile; instead each is a
// row-/element-parallel kernel that keeps HBM/L2 accesses coalesced along H.
#include "common.cuh"

namespace {

constexpr int MAX_DIN = 32;    // the synthetic control env's widest observation (env_synth.cu MAX_D)
constexpr int MAX_NOUT = 32;

// h1[m, j] = relu(b1[j] + sum_i x[row(m), i] * W1[j, i]);  row(m) = idx ? idx[m] : m.
// Optionally writes the gathered rows xg[m, :] (needed by the weight-gradient product).
__global__ void mlp_in_fwd_kernel(const float* __restrict__ x, const int32_t* __restrict__ idx,
                                  const float* __restrict__ W1, const float* __restrict__ b1,
                                  int M, int D, int H, float* __restrict__ h1, float* __restrict__ xg) {
  const int m = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ float sx[MAX_DIN];
  const int row = idx ? idx[m] : m;
  if (threadIdx.x < D) {
    const float v = x[(size_t)row * D + threadIdx.x];
    sx[threadIdx.x] = v;
    if (xg && blockIdx.x == 0) xg[(size_t)m * D + threadIdx.x] = v;
  }
  __syncthreads();
  if (j >= H) return;
  float acc = 0.f;
  for (int i = 0; i < D; ++i) acc = fmaf(sx[i], W1[(size_t)j * D + i], acc);
  acc += b1[j];
  h1[(size_t)m * H + j] = fmaxf(acc, 0.f);
}

// Flattened per-output row tables (filled on the host from up to 3 heads) so that the kernels
// index their accumulators with compile-time constants (no local-memory spills).
struct HeadRows {
  const float* w[MAX_NOUT];   // row o of the concatenated weight [nout, H]
  const float* b[MAX_NOUT];   // &bias[o]
};
struct HeadGradRows {
  float* dw[MAX_NOUT];
  float* db[MAX_NOUT];
};

// out[m, o] = b[o] + sum_j h[m, j] * W[o, j] for up to 3 heads concatenated along o.
// One warp per row.  The j loop is unrolled 4-deep with every load of an unrolled group issued
// before its first use (these kernels are pure load-latency chains at minibatch sizes: the ncu
// launch list showed one full memory latency per un-pipelined iteration).
__global__ void __launch_bounds__(256)
heads_fwd_kernel(const float* __restrict__ h, int M, int H, HeadRows hr, int nout, float* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= M) return;
  float acc[MAX_NOUT];
#pragma unroll
  for (int o = 0; o < MAX_NOUT; ++o) acc[o] = 0.f;
  const float* hrow = h + (size_t)warp * H;
  int j = lane;
  for (; j + 96 < H; j += 128) {
    float hv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) hv[u] = hrow[j + 32 * u];
#pragma unroll
    for (int o = 0; o < MAX_NOUT; ++o) {
      if (o < nout) {
        float wv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) wv[u] = hr.w[o][j + 32 * u];
#pragma unroll
        for (int u = 0; u < 4; ++u) acc[o] = fmaf(hv[u], wv[u], acc[o]);
      }
    }
  }
  for (; j < H; j += 32) {
    const float hv = hrow[j];
#pragma unroll
    for (int o = 0; o < MAX_NOUT; ++o)
      if (o < nout) acc[o] = fmaf(hv, hr.w[o][j], acc[o]);
  }
#pragma unroll
  for (int o = 0; o < MAX_NOUT; ++o) {
    if (o < nout) {
      const float v = jb_warp_sum(acc[o]);
      if (lane == 0) out[(size_t)warp * nout + o] = v + *hr.b[o];
    }
  }
}

// dh[m, j] = (sum_o dout[m, o] * W[o, j]) * (h[m, j] > 0)
__global__ void heads_bwd_dx_kernel(const float* __restrict__ dout, const float* __restrict__ h, int M, int H,
                                    HeadRows hr, int nout, float* __restrict__ dh) {
  const int m = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ float sd[MAX_NOUT];
  if (threadIdx.x < nout) sd[threadIdx.x] = dout[(size_t)m * nout + threadIdx.x];
  __syncthreads();
  if (j >= H) return;
  float acc = 0.f;
#pragma unroll
  for (int o = 0; o < MAX_NOUT; ++o)
    if (o < nout) acc = fmaf(sd[o], hr.w[o][j], acc);
  dh[(size_t)m * H + j] = (h[(size_t)m * H + j] > 0.f) ? acc : 0.f;
}

// dW[o, j] = sum_m dout[m, o] * h[m, j];  db[o] = sum_m dout[m, o].
// CTA = 32 columns (j) x DW_ROWS row-lanes, each row-lane strides over the batch with a 4-deep
// unrolled, load-first loop; fixed-order smem reduction over the row-lanes.
constexpr int DW_ROWS = 32;
__global__ void __launch_bounds__(32 * DW_ROWS)
heads_bwd_dw_kernel(const float* __restrict__ dout, const float* __restrict__ h, int M, int H, HeadGradRows gr, int nout) {
  __shared__ float s[DW_ROWS][33];
  const int j = blockIdx.x * 32 + threadIdx.x;
  const int ry = threadIdx.y;
  float acc[MAX_NOUT];
#pragma unroll
  for (int o = 0; o < MAX_NOUT; ++o) acc[o] = 0.f;
  float bacc = 0.f;   // lane x < nout of CTA 0 accumulates the bias gradient of output x
  const bool do_b = (blockIdx.x == 0) && (threadIdx.x < nout);
  int m = ry;
  for (; m + 3 * DW_ROWS < M; m += 4 * DW_ROWS) {
    float hv[4], bv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) hv[u] = (j < H) ? h[(size_t)(m + u * DW_ROWS) * H + j] : 0.f;
    if (do_b) {
#pragma unroll
      for (int u = 0; u < 4; ++u) bv[u] = dout[(size_t)(m + u * DW_ROWS) * nout + threadIdx.x];
#pragma unroll
      for (int u = 0; u < 4; ++u) bacc += bv[u];
    }
#pragma unroll
    for (int o = 0; o < MAX_NOUT; ++o) {
      if (o < nout) {
        float dv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) dv[u] = dout[(size_t)(m + u * DW_ROWS) * nout + o];
#pragma unroll
        for (int u = 0; u < 4; ++u) acc[o] = fmaf(dv[u], hv[u], acc[o]);
      }
    }
  }
  for (; m < M; m += DW_ROWS) {
    const float hv = (j < H) ? h[(size_t)m * H + j] : 0.f;
    const float* dr = dout + (size_t)m * nout;
#pragma unroll
    for (int o = 0; o < MAX_NOUT; ++o)
      if (o < nout) acc[o] = fmaf(dr[o], hv, acc[o]);
    if (do_b) bacc += dr[threadIdx.x];
  }
  // one output at a time through a [DW_ROWS][33] staging tile (keeps static smem small)
  for (int o = 0; o <= nout; ++o) {
    float v = bacc;
#pragma unroll
    for (int q = 0; q < MAX_NOUT; ++q) if (q == o && o < nout) v = acc[q];
    __syncthreads();
    s[ry][threadIdx.x] = v;
    __syncthreads();
    if (ry == 0) {
      float t = s[0][threadIdx.x];
      for (int r = 1; r < DW_ROWS; ++r) t += s[r][threadIdx.x];
      if (o < nout) { if (j < H) gr.dw[o][j] = t; }
      else if (do_b) *gr.db[threadIdx.x] = t;
    }
  }
}

static bool fill_rows(HeadRows& hr, const float* const* w, const float* const* b, const int* n, int H) {
  int o = 0;
  for (int g = 0; g < 3; ++g)
    for (int q = 0; q < n[g]; ++q, ++o) {
      if (o >= MAX_NOUT || !w[g]) return false;
      hr.w[o] = w[g] + (size_t)q * H;
      hr.b[o] = b[g] ? b[g] + q : nullptr;
    }
  for (; o < MAX_NOUT; ++o) { hr.w[o] = nullptr; hr.b[o] = nullptr; }
  return true;
}

}  // namespace

JB_API int jb_mlp_in_fwd(const float* x, const int32_t* idx, const float* w1, const float* b1, int M, int D, int H,
                         float* h1, float* xg, void* stream) {
  if (!x || !w1 || !b1 || !h1 || M <= 0 || D <= 0 || D > MAX_DIN || H <= 0) return JB_ERR_INVALID;
  dim3 grid(jb_div_up(H, 128), M);
  mlp_in_fwd_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(x, idx, w1, b1, M, D, H, h1, xg);
  return jb_check_launch();
}

// up to 3 heads; pass NULL/0 for unused ones.  out is [M, n0+n1+n2].
JB_API int jb_heads_fwd(const float* h, int M, int H, const float* w0, const float* b0, int n0, const float* w1,
                        const float* b1, int n1, const float* w2, const float* b2, int n2, float* out, void* stream) {
  const int nout = n0 + n1 + n2;
  if (!h || !out || M <= 0 || H <= 0 || nout <= 0 || nout > MAX_NOUT) return JB_ERR_INVALID;
  const float* w[3] = {w0, w1, w2}; const float* b[3] = {b0, b1, b2}; const int n[3] = {n0, n1, n2};
  for (int g = 0; g < 3; ++g) if (n[g] > 0 && (!w[g] || !b[g])) return JB_ERR_INVALID;
  HeadRows hr;
  if (!fill_rows(hr, w, b, n, H)) return JB_ERR_INVALID;
  const int threads = 256;
  heads_fwd_kernel<<<jb_div_up((long long)M * 32, threads), threads, 0, (cudaStream_t)stream>>>(h, M, H, hr, nout, out);
  return jb_check_launch();
}

JB_API int jb_heads_bwd_dx(const float* dout, const float* h, int M, int H, const float* w0, int n0, const float* w1,
                           int n1, const float* w2, int n2, float* dh, void* stream) {
  const int nout = n0 + n1 + n2;
  if (!dout || !h || !dh || M <= 0 || H <= 0 || nout <= 0 || nout > MAX_NOUT) return JB_ERR_INVALID;
  const float* w[3] = {w0, w1, w2}; const float* b[3] = {nullptr, nullptr, nullptr}; const int n[3] = {n0, n1, n2};
  HeadRows hr;
  if (!fill_rows(hr, w, b, n, H)) return JB_ERR_INVALID;
  dim3 grid(jb_div_up(H, 128), M);
  heads_bwd_dx_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(dout, h, M, H, hr, nout, dh);
  return jb_check_launch();
}

JB_API int jb_heads_bwd_dw(const float* dout, const float* h, int M, int H, float* dw0, float* db0, int n0, float* dw1,
                           float* db1, int n1, float* dw2, float* db2, int n2, void* stream) {
  const int nout = n0 + n1 + n2;
  if (!dout || !h || M <= 0 || H <= 0 || nout <= 0 || nout > MAX_NOUT) return JB_ERR_INVALID;
  float* dw[3] = {dw0, dw1, dw2}; float* db[3] = {db0, db1, db2}; const int n[3] = {n0, n1, n2};
  HeadGradRows gr;
  int o = 0;
  for (int g = 0; g < 3; ++g)
    for (int q = 0; q < n[g]; ++q, ++o) {
      if (!dw[g] || !db[g]) return JB_ERR_INVALID;
      gr.dw[o] = dw[g] + (size_t)q * H;
      gr.db[o] = db[g] + q;
    }
  for (; o < MAX_NOUT; ++o) { gr.dw[o] = nullptr; gr.db[o] = nullptr; }
  heads_bwd_dw_kernel<<<jb_div_up(H, 32), dim3(32, DW_ROWS), 0, (cudaStream_t)stream>>>(dout, h, M, H, gr, nout);
  return jb_check_launch();
}
