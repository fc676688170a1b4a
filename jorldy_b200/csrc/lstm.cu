// One LSTM time step, forward and backward, for the R2D2 recurrent Q-network (core/network/r2d2.py).
//
// torch.nn.LSTM's layout and gate order (i, f, g, o): weight_hh [4H, H], and the input projection of every time step
//   xg = x W_ih^T + b_ih + b_hh        [rows, 4H]
// is ONE jb_linear_fwd over all the stacked rows, done by the caller.  A step then only needs the recurrent product
// h_{t-1} W_hh^T and the cell update, which is what these two kernels fuse:
//   i = sigm(xg_i + h W_hi^T), f = sigm(.), g = tanh(.), o = sigm(.);  c_t = f c_{t-1} + i g;  h_t = o tanh(c_t).
//
// A CTA owns LU hidden units j and LR rows m.  It reads the four weight rows j, H + j, 2H + j, 3H + j of W_hh, so every
// gate of a unit is formed in one CTA and the cell update runs in the epilogue without another launch.  The
// contraction is staged through shared memory LK at a time and accumulated with fp32 FFMA in ascending k by one thread
// per (row, unit): no atomics, no split of the sum, and a row's result does not depend on M or on the row's position,
// so both kernels are bit-reproducible.
//
// reset[m] != 0 marks a row whose episode starts at this step: its h_{t-1} and c_{t-1} are read as zero (on the act
// side and on the learn side alike), and no gradient crosses that step back into the previous one.
#include "common.cuh"

namespace {

constexpr int LU = 8;     // hidden units per CTA
constexpr int LR = 32;    // rows per CTA
constexpr int LK = 64;    // contraction depth staged per shared-memory pass
constexpr int LT = LU * LR;

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ bool is_reset(const float* reset, int m) { return reset != nullptr && reset[m] != 0.f; }

__global__ void __launch_bounds__(LT)
lstm_step_fwd_kernel(const float* __restrict__ xg, const float* __restrict__ h_prev, const float* c_prev,
                     const float* __restrict__ w_hh, const float* __restrict__ reset, int M, int H, float* __restrict__ h,
                     float* c, float* __restrict__ gates, float* __restrict__ hprev_eff) {
  __shared__ float hs[LR][LK + 1];
  __shared__ float ws[4 * LU][LK + 1];
  const int tid = threadIdx.x, r = tid / LU, u = tid % LU;
  const int m0 = blockIdx.y * LR, j0 = blockIdx.x * LU;
  const int m = m0 + r, j = j0 + u;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k0 = 0; k0 < H; k0 += LK) {
    for (int e = tid; e < LR * LK; e += LT) {
      const int rr = e / LK, kk = e % LK, gm = m0 + rr, gk = k0 + kk;
      hs[rr][kk] = (gm < M && gk < H && !is_reset(reset, gm)) ? h_prev[(size_t)gm * H + gk] : 0.f;
    }
    for (int e = tid; e < 4 * LU * LK; e += LT) {
      const int q = e / LK, kk = e % LK, g = q / LU, jj = j0 + q % LU, gk = k0 + kk;
      ws[q][kk] = (jj < H && gk < H) ? w_hh[((size_t)g * H + jj) * H + gk] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < LK; ++kk) {
      const float hv = hs[r][kk];
#pragma unroll
      for (int g = 0; g < 4; ++g) acc[g] = fmaf(hv, ws[g * LU + u][kk], acc[g]);
    }
    __syncthreads();
  }
  if (m >= M || j >= H) return;
  const bool rs = is_reset(reset, m);
  const float* xr = xg + (size_t)m * 4 * H;
  const float gi = sigm(__fadd_rn(xr[j], acc[0]));
  const float gf = sigm(__fadd_rn(xr[H + j], acc[1]));
  const float gg = tanhf(__fadd_rn(xr[2 * H + j], acc[2]));
  const float go = sigm(__fadd_rn(xr[3 * H + j], acc[3]));
  const size_t o = (size_t)m * H + j;
  const float cp = rs ? 0.f : c_prev[o];
  const float cn = __fadd_rn(__fmul_rn(gf, cp), __fmul_rn(gi, gg));
  if (hprev_eff) hprev_eff[o] = rs ? 0.f : h_prev[o];
  c[o] = cn;
  h[o] = __fmul_rn(go, tanhf(cn));
  float* gr = gates + (size_t)m * 4 * H;
  gr[j] = gi; gr[H + j] = gf; gr[2 * H + j] = gg; gr[3 * H + j] = go;
}

__global__ void __launch_bounds__(LT)
lstm_step_bwd_kernel(const float* __restrict__ dh_out, const float* __restrict__ dgates_next, const float* __restrict__ w_hh,
                     const float* __restrict__ gates, const float* __restrict__ c_prev, const float* __restrict__ c,
                     const float* dc_next, const float* __restrict__ reset,
                     const float* __restrict__ reset_next, int M, int H, float* __restrict__ dgates, float* dc) {
  __shared__ float gs[LR][LK + 1];
  __shared__ float ws[LK][LU + 1];
  const int tid = threadIdx.x, r = tid / LU, u = tid % LU;
  const int m0 = blockIdx.y * LR, j0 = blockIdx.x * LU;
  const int m = m0 + r, j = j0 + u;
  const int G = 4 * H;
  float acc = 0.f;                    // (dgates_{t+1} W_hh)[m, j], k ascending over the 4H gate rows
  if (dgates_next) {
    for (int k0 = 0; k0 < G; k0 += LK) {
      for (int e = tid; e < LR * LK; e += LT) {
        const int rr = e / LK, kk = e % LK, gm = m0 + rr, gk = k0 + kk;
        gs[rr][kk] = (gm < M && gk < G) ? dgates_next[(size_t)gm * G + gk] : 0.f;
      }
      for (int e = tid; e < LK * LU; e += LT) {
        const int kk = e / LU, uu = e % LU, gk = k0 + kk, jj = j0 + uu;
        ws[kk][uu] = (gk < G && jj < H) ? w_hh[(size_t)gk * H + jj] : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int kk = 0; kk < LK; ++kk) acc = fmaf(gs[r][kk], ws[kk][u], acc);
      __syncthreads();
    }
  }
  if (m >= M || j >= H) return;
  const bool cross = !is_reset(reset_next, m);      // step t+1 read h_t and c_t (it did not start an episode)
  const size_t o = (size_t)m * H + j;
  const float dh = __fadd_rn(dh_out ? dh_out[o] : 0.f, cross ? acc : 0.f);
  const float* gr = gates + (size_t)m * G;
  const float gi = gr[j], gf = gr[H + j], gg = gr[2 * H + j], go = gr[3 * H + j];
  const float tc = tanhf(c[o]);
  const float dcn = (dc_next && cross) ? dc_next[o] : 0.f;
  const float dcell = __fadd_rn(__fmul_rn(__fmul_rn(dh, go), __fadd_rn(1.f, -__fmul_rn(tc, tc))), dcn);
  const float cp = is_reset(reset, m) ? 0.f : c_prev[o];
  float* dr = dgates + (size_t)m * G;
  dr[j] = __fmul_rn(__fmul_rn(dcell, gg), __fmul_rn(gi, __fadd_rn(1.f, -gi)));
  dr[H + j] = __fmul_rn(__fmul_rn(dcell, cp), __fmul_rn(gf, __fadd_rn(1.f, -gf)));
  dr[2 * H + j] = __fmul_rn(__fmul_rn(dcell, gi), __fadd_rn(1.f, -__fmul_rn(gg, gg)));
  dr[3 * H + j] = __fmul_rn(__fmul_rn(dh, tc), __fmul_rn(go, __fadd_rn(1.f, -go)));
  if (dc) dc[o] = __fmul_rn(dcell, gf);
}

}  // namespace

JB_API int jb_lstm_step_fwd(const float* xg, const float* h_prev, const float* c_prev, const float* w_hh, const float* reset,
                            int M, int H, float* h, float* c, float* gates, float* hprev_eff, void* stream) {
  if (!xg || !h_prev || !c_prev || !w_hh || !h || !c || !gates || M <= 0 || H <= 0) return JB_ERR_INVALID;
  if (h == h_prev || hprev_eff == h_prev) return JB_ERR_INVALID;     // other CTAs still read h_prev rows
  dim3 grid(jb_div_up(H, LU), jb_div_up(M, LR));
  lstm_step_fwd_kernel<<<grid, LT, 0, (cudaStream_t)stream>>>(xg, h_prev, c_prev, w_hh, reset, M, H, h, c, gates,
                                                              hprev_eff);
  return jb_check_launch();
}

JB_API int jb_lstm_step_bwd(const float* dh_out, const float* dgates_next, const float* w_hh, const float* gates,
                            const float* c_prev, const float* c, const float* dc_next, const float* reset,
                            const float* reset_next, int M, int H, float* dgates, float* dc, void* stream) {
  if (!w_hh || !gates || !c_prev || !c || !dgates || M <= 0 || H <= 0) return JB_ERR_INVALID;
  if (dgates == dgates_next) return JB_ERR_INVALID;
  dim3 grid(jb_div_up(H, LU), jb_div_up(M, LR));
  lstm_step_bwd_kernel<<<grid, LT, 0, (cudaStream_t)stream>>>(dh_out, dgates_next, w_hh, gates, c_prev, c, dc_next, reset,
                                                              reset_next, M, H, dgates, dc);
  return jb_check_launch();
}
