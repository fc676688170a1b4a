// Munchausen scalars of one sample (Vieillard, Pietquin, Geist 2020, arXiv:2007.14430), shared by jb_mdqn_loss
// (csrc/dqn.cu) and jb_munchausen_quantile_loss (csrc/quantile.cu).
#pragma once
#include "common.cuh"

constexpr int MUNCHAUSEN_MAX_A = 18;   // ALE's full action set; pi / tlp rows are sized for it

// One thread, actions in ascending order, precise expf / logf.  qs = q'(s, .) and qn = q'(s', .) are the TARGET
// network's values [A]; a_t is the taken action.  With m = max_b q(b) on the same row:
//   tau logpi(a) = (q(a) - m) - tau log sum_b exp((q(b) - m) / tau)
// log(pi) itself is never formed: at tau = 0.03, pi underflows to 0 for ordinary Q spreads.
// Writes pi[a] = softmax(qn / tau)(a) and tlp[a] = tau logpi(a|s'), and returns the bonus
// alpha clip(tau logpi(a_t|s), l0, 0), clipped first and then scaled.  Every sum includes its max term exp(0) = 1, so
// each log argument is >= 1 and every output stays finite when the other terms underflow.
__device__ __forceinline__ float munchausen_row(const float* qs, const float* qn, int A, int a_t, float tau, float alpha,
                                                float l0, float* pi, float* tlp) {
  float m = qs[0];
  for (int a = 1; a < A; ++a) m = fmaxf(m, qs[a]);
  float z = 0.f;
  for (int a = 0; a < A; ++a) z += expf((qs[a] - m) / tau);
  const float tlp_t = (qs[a_t] - m) - tau * logf(z);
  const float bonus = alpha * fminf(fmaxf(tlp_t, l0), 0.f);
  float mn = qn[0];
  for (int a = 1; a < A; ++a) mn = fmaxf(mn, qn[a]);
  float zn = 0.f;
  for (int a = 0; a < A; ++a) {
    const float e = expf((qn[a] - mn) / tau);
    pi[a] = e;
    zn += e;
  }
  const float lzn = tau * logf(zn);
  for (int a = 0; a < A; ++a) {
    tlp[a] = (qn[a] - mn) - lzn;
    pi[a] = pi[a] / zn;
  }
  return bonus;
}
