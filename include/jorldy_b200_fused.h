/* Argument block of the persistent PPO minibatch-loop kernel (jorldy_b200/csrc/ppo_fused.cu).
 * Replaces the body of the epoch loop of jorldy/core/agent/ppo.py:118-175 for the MLP actor-critic
 * networks (policy_value.py).  All pointers are device pointers; the struct itself is read on the host. */
#ifndef JORLDY_B200_FUSED_H
#define JORLDY_B200_FUSED_H
#include <stdint.h>

typedef struct jb_ppo_fused_args {
  /* network: views into the flat parameter / gradient buffers */
  float *W1, *b1, *W2, *b2;
  float *Wh[3], *bh[3];
  float *gW1, *gb1, *gW2, *gb2;
  float *gWh[3], *gbh[3];
  float *flat, *grad, *am, *av;      /* params, grads, Adam exp_avg / exp_avg_sq (flat, 16-B aligned) */
  long long P4;                      /* number of float4 in the flat buffers */
  /* rollout (read-only) */
  const float *state;                /* [NT, D] */
  const void *action;                /* int32 [NT] (discrete) or f32 [NT, A] (continuous) */
  const float *adv, *ret, *vold, *logp_old;
  const int32_t *perm;               /* [>= (cursor + n_steps) * B] shuffled row ids */
  /* workspaces */
  float *h1;                         /* [H/32, B, 32] tiled layer-1 activations */
  float *h2;                         /* [B, H] layer-2 activations, row major */
  float *xg;                         /* [B, D] */
  float *w1p;                        /* [B/32, H, D+1] per-row-tile partial dW1 | db1 */
  float *headp;                      /* [H/32, 2, B, 4] per-column-tile partial head outputs */
  float *dout;                       /* [B, 8] d loss / d head outputs per row (value head: the critic_loss1 candidate) */
  float *dv2;                        /* [B] the critic_loss2 candidate of the value-head gradient */
  float *rowst;                      /* [6, B] per-row v - ret, v_clip - ret, min(surr1, surr2), entropy, ratio, p_min */
  float *h2t;                        /* [H/32, B, 32] tiled copy of h2 */
  float *W2t;                        /* [H/32, H, 32] tiled shadow of W2 (maintained by the Adam phase) */
  float *W2img;                      /* [2 (hi | lo), H/32, H/32, 32 x 32] wgmma-layout (K-major, 128-byte swizzle) images of W2 for the tensor-core
                                      * forward phase (3xTF32 split), maintained by the Adam phase; NULL: FFMA tiles only */
  float *W2Timg;                     /* [2, H/128, H/32, 128 x 32] the same for W2^T (operand of the tensor-core dh1 jobs) */
  float *partials;                   /* [256] per-CTA squared-norm partials */
  float *acc;                        /* [8] learn()-level statistic accumulators */
  int32_t *cur_idx;                  /* [B] */
  unsigned int *barrier;             /* [64] grid-barrier counter, per-row-tile P1 tickets, per-column-tile job counters (zeroed by the launcher) */
  long long *step;                   /* Adam step counter (device) */
  long long *cursor;                 /* minibatch cursor (device) */
  const float *lr;                   /* learning rate (device scalar) */
  /* multi-GPU: gradient exchange through peer-mapped memory (world == 1: unused).  peer[r] = rank r's exchange
   * buffer, laid out in 32-bit words as
   *   [0, 4*P4)                       this rank's gradient (`grad` above is peer[rank])
   *   [xllin_off, + 8*world*q4)       inbox of the slice this rank OWNS (q4 = ceil(P4 / world) float4): for every source
   *                                   rank the raw gradient slice as "LL" words {tag | value} (64 bit each)
   *   [xgred_off, + 8*P4)             the AVERAGED gradient as LL words: slice q is written by its owner, rank q
   *   [xflag_off, + JB_X_WORDS)       JB_X_MSG {critic row sum | tag} x 2 per source rank (the two critic means of
   *                                   ppo.py:151-154 are global), JB_X_PTAB {||chunk||^2 | tag} per (owner rank, owner CTA)
   * An LL word is valid when its tag equals the step number: no flags, no fences.  Tags are monotonic: xbase = number
   * of steps run by earlier launches. */
  float *peer[8];
  int world, rank;
  unsigned int xbase;
  int xflag_off, xgred_off, xllin_off;
  int nh[3];                         /* outputs per head */
  int B, D, H, A, nout, continuous, n_steps;
  float eps_clip, vf_coef, ent_coef, beta1, beta2, adam_eps, max_norm;
} jb_ppo_fused_args;

/* word offsets inside the flag region of the exchange buffer */
#define JB_X_MSG 64
#define JB_X_PTAB 128
#define JB_X_MAX_CTAS 256
#define JB_X_WORDS (JB_X_PTAB + 8 * JB_X_MAX_CTAS * 2)

#endif
