/* jorldy_b200 — C ABI of the H100-native rollout-collect -> buffer -> learn() core.
 *
 * The reference (kakaoenterprise/JORLDY) is pure Python and has no FFI of its own; its plugin
 * boundary is the Python classes Agent / Env / Buffer / Network / Optimizer.  This header is the
 * boundary a maintainer would bind from those classes (ctypes stub in INTEGRATION.md): plain
 * pointers and sizes, no torch types.  Each entry point names the reference code it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name says host; buffers are caller-owned
 *     (the Python host allocates them as torch tensors) and must stay alive until the stream
 *     has drained;
 *   - `stream` is a cudaStream_t passed as void*; calls only enqueue work (async w.r.t. host);
 *   - return value: 0 = ok, negative errno-style code otherwise (-22 bad argument, -5 CUDA
 *     launch/runtime failure).  Nothing throws;
 *   - one learner thread per handle/stream, as in the reference (run_mode.py:327).
 */
#ifndef JORLDY_B200_H
#define JORLDY_B200_H

#include <stdint.h>

#ifdef __cplusplus
#define JB_API extern "C"
#else
#define JB_API
#endif

/* ---------------------------------------------------------------------------------------------
 * Environments — jorldy/core/env/gym_env.py:61-83 (Cartpole.step / _Gym.reset :32-36),
 * :86-95 (Pendulum, MountainCar) + run_mode.py:91 auto-reset line; gym 0.23.0 physics.
 * kind: 0 cartpole (phys[n,4], obs[n,4]), 1 pendulum (phys[n,2], obs[n,3]),
 *       2 mountain_car (phys[n,2], obs[n,2]).
 * action_kind: 0 int64, 1 int32, 2 float32.
 * stats (may be NULL): [2] floats, += {episodes finished, sum of their scores}.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_env_classic_reset(int kind, double* phys, float* obs, int32_t* elapsed, int64_t* episode,
                                float* score, const uint8_t* mask, uint64_t seed, uint64_t stream_base,
                                int n, void* stream);
JB_API int jb_env_classic_step(int kind, double* phys, float* obs, int32_t* elapsed, int64_t* episode,
                               float* score, const void* action, int action_kind, float* next_obs,
                               float* reward, float* done, float* stats, int auto_reset, int max_steps,
                               uint64_t seed, uint64_t stream_base, int n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * GAE — jorldy/core/agent/ppo.py:95-110.  Arrays are [N,T] row-major f32.
 * next_value may be NULL: then V(s'_t) = value[:,t+1] and last_value[N] closes the row.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_gae(const float* reward, const float* done, const float* value, const float* next_value,
                  const float* last_value, int N, int T, float gamma, float lambda, int standardize,
                  float* adv, float* ret, void* stream);

/* Synthetic continuous-control env with MuJoCo-task dimensions (replaces gym + mujoco_py behind
 * jorldy/core/env/mujoco.py:25-58; BASELINE configs[4]: obs 11 / act 3).  s' = tanh(Ws s + Wa a) + 0.01 N(0,I),
 * reward = -|s'|^2 / D, done ~ Bernoulli(p_done) or TimeLimit; obs f32 [n,D], action f32 [n,A]. */
JB_API int
jb_env_synth_reset(float* obs, int32_t* elapsed, int64_t* episode, float* score, uint64_t seed,
                   uint64_t stream_base, int n, int D, void* stream);
JB_API int
jb_env_synth_step(float* obs, int32_t* elapsed, int64_t* episode, int64_t* tcount, float* score,
                  const float* action, const float* Ws, const float* Wa, float* next_obs, float* reward,
                  float* done, float* stats, int auto_reset, int max_steps, float p_done, uint64_t seed,
                  uint64_t stream_base, int n, int D, int A, void* stream);

/* Replay ring rows (jorldy/core/buffer/replay_buffer.py:16-31, base.py:42-56 stack_transition): a field is a
 * [capacity, row_bytes] byte matrix; store scatters n batch rows to ring positions, gather collects a minibatch. */
JB_API int
jb_replay_store(void* ring, const void* batch, const int64_t* pos, int n, long long row_bytes, void* stream);
JB_API int
jb_replay_gather(const void* ring, const int64_t* idx, int n, long long row_bytes, void* batch, void* stream);

/* Single-frame Atari replay (csrc/frame_ring.cu): each lane of n keeps a ring of frames_per_lane 84x84 uint8 frames
 * (frames [n, F, 7056]) with the episode-first position of each (first [n, F] int64) and its push count (head [n]).
 * A frame reference is (lane << 40) | absolute position; the [4,84,84] stack it names is rebuilt on gather.
 * push: obs / next_obs [n,4,84,84], done f32 [n].  next_obs NULL: push obs[:,3] as episode-first frames (after a reset);
 * otherwise push next_obs[:,3], emit state_ref / next_ref (may be NULL), then obs[:,3] where done && auto_reset.
 * gather: stacks of state_refs[idx[i]] / next_refs[idx[i]] (idx NULL: i) into [B,4,84,84]; a reference whose frames
 * were overwritten is zero-filled and sets *status = 1. */
JB_API int jb_frame_push(uint8_t* frames, int64_t* first, int64_t* head, int64_t frames_per_lane, const uint8_t* obs,
                         const uint8_t* next_obs, const float* done, int auto_reset, int64_t* state_ref, int64_t* next_ref,
                         int n, void* stream);
JB_API int jb_frame_gather(const uint8_t* frames, const int64_t* first, const int64_t* head, int64_t frames_per_lane,
                           int n_lanes, const int64_t* state_refs, const int64_t* next_refs, const int64_t* idx, int B,
                           uint8_t* state_out, uint8_t* next_out, int32_t* status, void* stream);
/* conv1's column matrix read straight from the ring (the CNN head's 4x84x84 input, 8x8 kernel, stride 4): col
 * [M*20*20, 256] f32 = im2col of the stacks of refs[idx[i]] (idx int32, NULL: i), each value (float)v / 255.0f, so it is
 * bit-equal to jb_frame_gather followed by jb_im2col_u8.  A non-resident reference writes zero rows and sets *status = 1.
 * frames must be 4-byte and col 16-byte aligned. */
JB_API int jb_im2col_u8_frames(const uint8_t* frames, const int64_t* first, const int64_t* head, int64_t frames_per_lane,
                               int n_lanes, const int64_t* refs, const int32_t* idx, int M, float* col, int32_t* status,
                               void* stream);

/* ---------------------------------------------------------------------------------------------
 * PER sum-tree — jorldy/core/buffer/per_buffer.py:19-101.  tree is f64[2*capacity-1].
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_per_update(double* tree, int64_t capacity, const int64_t* tree_idx, int64_t first_idx,
                         const double* new_p, const double* fill_p, double* max_priority, int B,
                         void* stream);
JB_API int jb_per_sample(const double* tree, int64_t capacity, int64_t counter, int B, double beta,
                         double uniform_sample_prob, const double* u_a, const double* u_b, uint64_t seed,
                         uint64_t rng_ctr, const double* shard_prob, const int64_t* global_counter,
                         int64_t* out_idx, double* out_w, double* out_p, double* out_stats, int normalize,
                         void* stream);
JB_API int jb_per_scale_weights(double* w, const double* wmax, int B, void* stream);
JB_API int jb_per_rebuild(double* tree, int64_t capacity, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Dense layers — jorldy/core/network/head.py:6-18, q_network.py, policy_value.py, dueling.py
 * (torch.nn.Linear: weight [out,in]) and network/utils.py:55-86 (NoisyNet: weight [in,out]).
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_gemm(const float* A, int lda, int a_kc, const float* B, int ldb, int b_kc, float* C, int ldc,
                   int M, int N, int K, const float* bias, int relu, const float* mask, int ldmask,
                   float* rowsum_a, int accumulate, void* stream);
JB_API int jb_linear_fwd(const float* x, const float* w, const float* b, float* y, int M, int in_f, int out_f,
                         int relu, void* stream);
/* wgmma 3xTF32 forward for large M (M % 128 == 0, out_f % 128 == 0, in_f % 32 == 0); -22 otherwise */
JB_API int jb_linear_fwd_tc(const float* x, const float* w, const float* b, float* y, int M, int in_f, int out_f,
                            int relu, void* stream);
JB_API int jb_linear_bwd_dx(const float* dy, const float* w, float* dx, int M, int in_f, int out_f,
                            const float* relu_act, void* stream);
JB_API int jb_linear_bwd_dw(const float* dy, const float* x, float* dw, float* db, int M, int in_f, int out_f,
                            void* stream);
JB_API int
jb_linear_bwd_dw_splitk(const float* dy, const float* x, float* dw, float* db, int M, int in_f, int out_f,
                        float* workspace, int splits, void* stream);
JB_API int jb_linear_io_fwd(const float* x, const float* w, const float* b, float* y, int M, int in_f, int out_f,
                            int relu, void* stream);
JB_API int jb_linear_io_bwd_dx(const float* dy, const float* w, float* dx, int M, int in_f, int out_f,
                               const float* relu_act, void* stream);
JB_API int jb_linear_io_bwd_dw(const float* dy, const float* x, float* dw, int M, int in_f, int out_f, void* stream);
JB_API int jb_colsum(const float* x, int M, int N, float* out, int accumulate, void* stream);
/* h1 = relu(x[idx] W1^T + b1) for 1 <= D <= 32 inputs (the synthetic control env's widest observation). */
JB_API int jb_mlp_in_fwd(const float* x, const int32_t* idx, const float* w1, const float* b1, int M, int D, int H,
                         float* h1, float* xg, void* stream);
JB_API int jb_heads_fwd(const float* h, int M, int H, const float* w0, const float* b0, int n0, const float* w1,
                        const float* b1, int n1, const float* w2, const float* b2, int n2, float* out, void* stream);
JB_API int jb_heads_bwd_dx(const float* dout, const float* h, int M, int H, const float* w0, int n0, const float* w1,
                           int n1, const float* w2, int n2, float* dh, void* stream);
JB_API int jb_heads_bwd_dw(const float* dout, const float* h, int M, int H, float* dw0, float* db0, int n0, float* dw1,
                           float* db1, int n1, float* dw2, float* db2, int n2, void* stream);
/* The same layers over an array of 1 <= n_heads <= 4 heads (host arrays of device pointers and widths, sum(n) <= 32):
 * head g has weight w[g] [n[g], H] and bias b[g] [n[g]], out is [M, sum(n)].  The three-head entry points above are
 * these calls with n_heads = 3. */
JB_API int jb_heads_fwd_n(const float* h, int M, int H, int n_heads, const float* const* w, const float* const* b,
                          const int* n, float* out, void* stream);
JB_API int jb_heads_bwd_dx_n(const float* dout, const float* h, int M, int H, int n_heads, const float* const* w,
                             const int* n, float* dh, void* stream);
JB_API int jb_heads_bwd_dw_n(const float* dout, const float* h, int M, int H, int n_heads, float* const* dw,
                             float* const* db, const int* n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * PPO — jorldy/core/agent/ppo.py:54-69 (act), :83-93 (value / log_prob_old), :127-162 (loss).
 * `out` is the [M,nout] pre-activation head output: discrete [logits(A)|v], continuous
 * [mu(A)|log_std(A)|v].  A wider A than an entry point's bound returns JB_ERR_INVALID.
 * ------------------------------------------------------------------------------------------- */
/* 1 <= A <= 18 (ALE's full action set) */
JB_API int jb_ppo_act_discrete(const float* out, int M, int A, int nout, const float* u, uint64_t seed,
                               uint64_t stream_base, uint64_t ctr, long long* row_ctr, int greedy, int64_t* action,
                               void* stream);
/* 1 <= A <= 8 */
JB_API int jb_ppo_act_continuous(const float* out, int M, int A, int nout, const float* normal, uint64_t seed,
                                 uint64_t stream_base, uint64_t ctr, long long* row_ctr, int greedy, float* action,
                                 void* stream);
/* 1 <= A <= 18 */
JB_API int jb_ppo_prepass_discrete(const float* out, const int32_t* action, int M, int A, int nout, float* value,
                                   float* logp_old, void* stream);
JB_API int jb_ppo_prepass_continuous(const float* out, const float* action, int M, int A, int nout, float* value,
                                     float* logp_old, void* stream);
JB_API int jb_take_minibatch(const int32_t* perm, long long* cursor, int B, int32_t* cur_idx, void* stream);
/* 1 <= A <= 18 discrete, 1 <= A <= 8 continuous */
JB_API int jb_ppo_loss(int continuous, const float* out, const int32_t* idx, const void* action, const float* adv,
                       const float* ret, const float* value_old, const float* logp_old, int B, int A, int nout,
                       float eps_clip, float vf_coef, float ent_coef, float* dout, float* stats, float* acc,
                       void* stream);

/* ---------------------------------------------------------------------------------------------
 * V-MPO (arXiv:1909.12238) minibatch loss on the PPO rollout path (csrc/vmpo.cu).  `out[B,nout]` holds the
 * minibatch rows' head outputs (layout as for PPO), `out_old[NT,nout]` the pre-pass outputs of the whole rollout;
 * out_old / action / adv / ret are gathered through idx (NULL: row b).  `mult` (device) = [eta, alpha_mu,
 * alpha_sigma].  dout[B,nout] receives d loss / d out, dmult[3] d loss / d mult.  stats holds 16 + 4*ceil(B/256)
 * floats: [0] actor_loss [1] critic_loss [2] eta_loss [3] alpha_loss [4] mean KL_mu (discrete: the KL)
 * [5] mean KL_sigma [6] top-half size [7] median advantage; acc (may be NULL) accumulates [0..3] into acc[0..3]
 * and counts minibatches in acc[4].  1 <= A <= 18 discrete, 1 <= A <= 8 continuous.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_vmpo_loss(int continuous, const float* out, const float* out_old, const int32_t* idx, const void* action,
                        const float* adv, const float* ret, int B, int A, int nout, const float* mult, float eps_eta,
                        float eps_alpha_mu, float eps_alpha_sigma, float* dout, float* dmult, float* stats, float* acc,
                        void* stream);
/* mult[k] = max(mult[k], minimum_k) after the multipliers' optimiser step */
JB_API int jb_vmpo_clamp(float* mult, float min_eta, float min_alpha_mu, float min_alpha_sigma, void* stream);

/* ---------------------------------------------------------------------------------------------
 * MPO (arXiv:1806.06920) on the replay path, csrc/mpo.cu: Retrace targets (arXiv:1606.02647) over B stored windows of
 * n <= 32 steps, the sampled E-step and the decoupled-KL M-step (arXiv:1812.02256) with mult = [eta, alpha_mu,
 * alpha_sigma] on the device.  Head rows are PPO's without the value: discrete logits [A] (A <= 18), continuous raw
 * [mu | log_std] [2A] (A <= 8).  State rows of window b are b*(n+1) + t (t = 0..n), step rows b*n + t (t < n).
 *   jb_mpo_logp           logp[M] = log pi(action | out) (discrete: int64 actions, continuous: the Normal log-pdf of
 *                         atanh(clamp(a, +-(1-1e-7))) summed over dims, no Jacobian); out rows nout apart
 *   jb_mpo_sample         for R target-actor rows raw [R, 2A] and normals eps [R, K, A] (K <= 64): z = mu + sd eps
 *                         [R, K, A]; the critic input xs [R*KK, D] (each state row x [R, D] repeated KK times) and
 *                         as [R*KK, A] = tanh(z) for k < K; with `taken` [B*n, A] (R = B*(n+1)), KK = K + 1 and slot K
 *                         holds the taken action a_t (0 at t = n), else KK = K
 *   jb_mpo_critic_target  tq: target critic, discrete [B*(n+1), A], continuous [B*(n+1)*(K+1)] (the K samples, then the
 *                         taken action); tout [B*(n+1), nout] the target actor; q the online critic, discrete [B*n, A],
 *                         continuous [B*n]; action int64 [B*n] / f32 [B*n, A]; log_mu, reward, done [B*n].
 *                         V'_t = E_pi' Q'(s_t, .) (continuous: the mean of the K samples), c_t = min(1, pi'(a_t)/mu_t)
 *                         (retrace = 0: c_t = 0), Qret_{n-1} = r + gamma (1-d) V'_n,
 *                         Qret_t = r_t + gamma (1-d_t) [V'_{t+1} + c_{t+1} (Qret_{t+1} - Q'(s_{t+1}, a_{t+1}))];
 *                         qret [B*n], dq = 2 (Q - Qret) / (B n) (discrete: in the taken action's column, 0 elsewhere);
 *                         stats[0] = mean (Q - Qret)^2, stats[1] = mean Qret.  One CTA, fixed-order sums.
 *   jb_mpo_policy_loss    over the S = B*n states: q(a) ∝ pi'(a) exp(Q'/eta) (discrete, exact) or softmax_k Q'(a_k)/eta
 *                         (continuous, z [B*(n+1), K, A] from jb_mpo_sample); L_eta, L_pi, KL(pi' || pi) (discrete) or
 *                         the decoupled KL_mu / KL_sigma, L_alpha; dout [S, nout] = d loss / d out, dmult[3];
 *                         stats[0..4] = L_pi, L_eta, L_alpha, mean KL_mu, mean KL_sigma; partials holds
 *                         jb_mpo_policy_partials(S) floats, folded in CTA order by a one-thread launch.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_mpo_logp(int continuous, const float* out, int nout, const void* action, int M, int A, float* logp,
                       void* stream);
JB_API int jb_mpo_sample(const float* raw, const float* eps, int R, int K, int A, const float* x, int D, const float* taken,
                         int n, float* z, float* xs, float* as, void* stream);
JB_API int jb_mpo_critic_target(int continuous, const float* tq, const float* tout, const float* q, const void* action,
                                const float* log_mu, const float* reward, const float* done, int B, int n, int A, int K,
                                float gamma, int retrace, float* dq, float* qret, float* stats, void* stream);
JB_API int jb_mpo_policy_partials(int S);
JB_API int jb_mpo_policy_loss(int continuous, const float* out, const float* tout, const float* tq, const float* z, int B,
                              int n, int A, int K, const float* mult, float eps_eta, float eps_alpha_mu,
                              float eps_alpha_sigma, float* dout, float* dmult, float* partials, float* stats,
                              void* stream);

/* ---------------------------------------------------------------------------------------------
 * RND-PPO (Burda et al., arXiv:1810.12894) on the PPO rollout path, csrc/rnd.cu.  The policy network has a second value
 * head: `out[M,nout]` is discrete [logits(A)|v|v_i] (nout = A + 2) or continuous [mu(A)|log_std(A)|v|v_i]
 * (nout = 2A + 2).  1 <= A <= 18 discrete, 1 <= A <= 8 continuous.  No atomics: every entry point is bit-reproducible.
 *   jb_rnd_prepass    value [M], value_i [M] and logp_old (discrete [M], continuous [M, A]) of the pre-pass rows, with
 *                     PPO's pre-pass log-prob.
 *   jb_rnd_ppo_loss   jb_ppo_loss with a second clipped critic: critic_loss = max(mse(v, ret), mse(v_clip, ret))
 *                     + max(mse(v_i, ret_i), mse(v_i_clip, ret_i)), each stream clipped around its own old value;
 *                     loss = actor + vf_coef critic + ent_coef entropy.  ret_i / value_i_old are full-rollout arrays
 *                     gathered through idx like the others.  dout [B, nout].  stats holds 8 + 4*ceil(B/256) floats:
 *                     [0] actor_loss [1] critic_loss [2] entropy_loss [3] max_ratio [4] min_prob [5] extrinsic critic
 *                     [6] intrinsic critic [7] 0; acc (may be NULL) accumulates [0..4] and counts in acc[5] as jb_ppo_loss
 *                     does.  With ret_i = value_i = value_i_old the policy and v columns of dout and stats[0..4] equal
 *                     jb_ppo_loss's bit for bit.
 *   jb_rnd_loss       p [B, F] predictor output, target [rows, F] the cached target features read at idx[b] (NULL: b);
 *                     ri [B] (may be NULL) = mean_F (p - target)^2; dp [B, F] = d rnd_loss / d p with
 *                     rnd_loss = mean_B ri.  stats holds 1 + ceil(B / 8) floats: [0] rnd_loss; acc (may be NULL)
 *                     acc[0] += rnd_loss, acc[1] += 1.  dp = NULL: the reward-only pre-pass (ri required, stats unused).
 *                     F = 256.
 *   jb_adv_mix        adv [N, T] = ext_coef adv_e + int_coef adv_i, then with `standardize` each row standardised as
 *                     jb_gae does it ((adv - mean) / (std + 1e-7), unbiased std, float64 sums in jb_gae's order).
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_rnd_prepass(int continuous, const float* out, const void* action, int M, int A, int nout, float* value,
                          float* value_i, float* logp_old, void* stream);
JB_API int jb_rnd_ppo_loss(int continuous, const float* out, const int32_t* idx, const void* action, const float* adv,
                           const float* ret, const float* value_old, const float* ret_i, const float* value_i_old,
                           const float* logp_old, int B, int A, int nout, float eps_clip, float vf_coef, float ent_coef,
                           float* dout, float* stats, float* acc, void* stream);
JB_API int jb_rnd_loss(const float* p, const float* target, const int32_t* idx, int B, int F, float* ri, float* dp,
                       float* stats, float* acc, void* stream);
JB_API int jb_adv_mix(const float* adv_e, const float* adv_i, int N, int T, float ext_coef, float int_coef,
                      int standardize, float* adv, void* stream);

/* ---------------------------------------------------------------------------------------------
 * REINFORCE (Williams, 1992) on whole episodes, csrc/reinforce.cu.  The episode ring keeps every unlearned step of N envs:
 * reward / done [N, L] f32, action int64 [N, L] (discrete) or f32 [N, L, A] (continuous); step t of every env lives in
 * column t mod L.  pos (device int64) counts the steps written; head[e] (device int64 [N]) is env e's oldest unlearned
 * step.  No atomics: every entry point is bit-reproducible.
 *   jb_episode_returns  for each env, the completed steps [head[e], last done in [head[e], pos)]: per episode the
 *                       discounted returns G_t = r_t + gamma G_{t+1} (G = r at the episode's done) in float64, with
 *                       `standardize` (G - mean) / (std + 1e-7) with the episode's own mean and ddof-0 std; written as
 *                       fp32 into ret_ring [N, L] at the steps' columns.  count[e] = the completed steps; head[e] moves
 *                       past them.
 *   jb_episode_rows     offsets [N] (workspace) = exclusive scan of count in env order; M (device int) = the total;
 *                       idx [.] = e L + column and ret [.] of every completed step, env-major and oldest first, padded
 *                       with idx 0 / ret 0 to a multiple of C.  idx / ret hold at least ceil(N L / C) C entries.
 *                       N L + C must fit an int32.
 *   jb_reinforce_loss   one chunk of C rows: chunk k = *cursor - 1 (after jb_take_minibatch; cursor NULL: chunk 0)
 *                       covers idx / ret entries [k C, k C + C); out [C, nout] holds the head outputs of those ring rows
 *                       (discrete logits, nout = A <= 18; continuous raw [mu | log_std], nout = 2A, A <= 8).
 *                       dout [C, nout] = d loss / d out of loss = -(1/M) sum log pi(a) ret (continuous: -(1/(M A)) sum
 *                       over rows and dims, mu = clamp(raw, +-5), std = exp(tanh(raw)), z = atanh(clamp(a, +-(1-1e-7)))).
 *                       Entries at or past the device M are padding: dout rows 0, no loss.  partials holds
 *                       jb_reinforce_loss_partials(C) floats, folded in CTA order: acc[0] += the chunk's share of the
 *                       loss, acc[1] += 1.  A device M <= 0 adds nothing.
 *   jb_add_f32          y += x over n floats (chunk gradients summed in chunk order).
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_episode_returns(const float* reward, const float* done, int N, int L, const long long* pos, long long* head,
                              double gamma, int standardize, float* ret_ring, int* count, void* stream);
JB_API int jb_episode_rows(const int* count, const long long* head, const float* ret_ring, int N, int L, int C,
                           int* offsets, int32_t* idx, float* ret, int* M, void* stream);
JB_API int jb_reinforce_loss_partials(int C);
JB_API int jb_reinforce_loss(int continuous, const float* out, const int32_t* rows, const float* ret,
                             const long long* cursor, const int* M, int C, const void* action, int A, int nout,
                             float* dout, float* partials, float* acc, void* stream);
JB_API int jb_add_f32(float* y, const float* x, long long n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ICM-PPO (Pathak et al., ICML 2017) on the PPO rollout path, csrc/icm.cu.  Column reductions split the rows into
 * chunks of 256 and fold the chunks' float64 partial sums in chunk order; `partials` holds jb_col_partials_doubles(M, N)
 * doubles.  No atomics anywhere: every entry point is bit-reproducible.
 *   jb_bn_elu_fwd     y [M, ldy] (and y2 [M, ldy2] when not NULL) = ELU(BatchNorm1d(x)) with x [M, N] in training mode:
 *                     biased batch variance, invstd = 1/sqrt(var + eps); mean / invstd [N] receive the batch statistics;
 *                     running_mean / running_var (unbiased variance) updated with `momentum`, num_batches_tracked += 1.
 *                     gamma NULL: y = ELU(x), no BatchNorm.  With BatchNorm, M < 2 is rejected (as torch does).
 *   jb_bn_elu_bwd     dx [M, N] from dy [M, lddy] and the forward's output y [M, ldy]; with BatchNorm also dgamma, dbeta [N]
 *                     (overwritten), from x, mean, invstd; xhat [M, N] is workspace.  gamma NULL: dx = dy ELU'.
 *   jb_rms_update     OpenAI baselines' RunningMeanStd.update over the M rows of x [M, D]: float64 mean / var [D] and count,
 *                     batch mean and population variance merged with the parallel formula.  D <= 1024.
 *   jb_rms_normalize  y [M, D] = clip((x[idx[m]] - mean) / sqrt(var), +-clip) (idx NULL: row m); mean = var = NULL: a gather.
 *   jb_icm_reward     normalize: per env the reward-forward filter rewems[n] = gamma rewems[n] + ri[n, t] over t (filt [N, T]
 *                     receives the filtered values, rewems [N] persists), RunningMeanStd update of (rms_mean, rms_var,
 *                     rms_count) with filt, then out = ext_coef reward + int_coef ri / (sqrt(rms_var) + 1e-7); without
 *                     normalize out = ext_coef reward + int_coef ri.  reward / ri / out [N, T] actor-major.
 *   jb_icm_loss       f [B, F] forward-model output, phi_next [B, ld_next] = phi(s'), g [B, A] inverse-model output,
 *                     action gathered through idx (NULL: row b; int32 discrete, f32 [., A] continuous);
 *                     ri [B] (may be NULL) = eta / 2 sum_F |f - phi_next|;  l_f = mean (f - phi_next)^2 over B F,
 *                     df = beta d l_f / d f;  l_i = cross-entropy of softmax(g) (discrete, mean over B) or mean (g - a)^2
 *                     over B A (continuous), dg = (1 - beta) d l_i / d g.  stats holds 4 + 3 ceil(B / 8) floats:
 *                     [0] mean r_i [1] l_f [2] l_i [3] beta l_f + (1 - beta) l_i; acc (may be NULL) [0..2] += stats[0..2],
 *                     acc[3] += 1.  df = dg = NULL: the reward-only pre-pass (ri required; g, action, stats unused).
 *                     F = 256, 1 <= A <= 18 discrete, 1 <= A <= 8 continuous.
 *   jb_icm_action_rows dst [M, ld] columns 0..A-1 = one-hot of action[idx[m]] (discrete) or the raw action (continuous).
 *   jb_scale_f32      x *= s over n floats.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_col_partials_doubles(int M, int N);
JB_API int jb_bn_elu_fwd(const float* x, int M, int N, const float* gamma, const float* beta, float* running_mean,
                         float* running_var, int64_t* num_batches_tracked, float momentum, float eps, float* mean,
                         float* invstd, double* partials, float* y, int ldy, float* y2, int ldy2, void* stream);
JB_API int jb_bn_elu_bwd(const float* dy, int lddy, const float* y, int ldy, const float* x, int M, int N,
                         const float* gamma, const float* mean, const float* invstd, float* xhat, double* partials,
                         float* dx, float* dgamma, float* dbeta, void* stream);
JB_API int jb_rms_update(const float* x, int M, int D, double* mean, double* var, double* count, double* partials,
                         void* stream);
JB_API int jb_rms_normalize(const float* x, const int32_t* idx, int M, int D, const double* mean, const double* var,
                            float clip, float* y, void* stream);
JB_API int jb_icm_reward(const float* reward, const float* ri, int N, int T, float gamma, int normalize, float* rewems,
                         double* rms_mean, double* rms_var, double* rms_count, double* partials, float* filt,
                         float ext_coef, float int_coef, float* out, void* stream);
JB_API int jb_icm_loss(int continuous, const float* f, const float* phi_next, int ld_next, const float* g,
                       const int32_t* idx, const void* action, int B, int A, int F, float eta, float beta, float* ri,
                       float* df, float* dg, float* stats, float* acc, void* stream);
JB_API int jb_icm_action_rows(int continuous, const void* action, const int32_t* idx, int M, int A, float* dst, int ld,
                              void* stream);
JB_API int jb_scale_f32(float* x, long long n, float s, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Synthetic Atari-shaped env — observation contract of jorldy/core/env/atari.py:56-61,112,145-160.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_env_frames_reset(uint8_t* obs, int64_t* fcount, float* score, uint64_t seed, uint64_t stream_base, int n,
                               void* stream);
JB_API int jb_env_frames_step(uint8_t* obs, int64_t* fcount, float* score, uint8_t* next_obs, float* reward, float* done,
                              float* stats, int auto_reset, uint64_t seed, uint64_t stream_base, int n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CNN head lowering — jorldy/core/network/head.py:21-61 (im2col / col2im around jb_gemm).
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_im2col_u8(const uint8_t* x, int B, int C, int H, int W, int KH, int KW, int S, float* col, void* stream);
JB_API int jb_im2col_nhwc(const float* x, int B, int C, int H, int W, int KH, int KW, int S, float* col, void* stream);
JB_API int jb_col2im_nhwc(const float* dcol, int B, int C, int H, int W, int KH, int KW, int S, const float* relu_act,
                          float* dx, void* stream);
JB_API int jb_nhwc_to_nchw(const float* x, int B, int P, int C, float* y, void* stream);
JB_API int jb_nchw_to_nhwc(const float* x, int B, int P, int C, const float* relu_act, float* y, void* stream);

/* Persistent minibatch-loop kernel (csrc/ppo_fused.cu); `host_args` points to a jb_ppo_fused_args
 * (include/jorldy_b200_fused.h) in HOST memory. */
JB_API int jb_ppo_fused_args_size(void);
JB_API int jb_ppo_fused_max_ctas(void);
JB_API int jb_ppo_fused_run(const void* host_args, void* stream);
/* Debug aid: clock64 stamps of the last step of the previous run made with JB_FUSED_SKIP=256 in the
 * environment; host_out receives 256 x 32 long longs. */
JB_API int jb_ppo_fused_trace(long long* host_out);

/* ---------------------------------------------------------------------------------------------
 * Value-based learners — jorldy/core/agent/dqn.py:99-138, double.py:25-41, multistep.py:41-50,
 * per.py:50-77, ape_x.py:63-116; dueling combine network/dueling.py:21-35, rainbow.py net :66-94.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_q_act(const float* q, int M, int A, float eps, const float* eps_rows, const float* u, uint64_t seed,
                    uint64_t stream_base, long long* row_ctr, int64_t* action, float* q_sel, void* stream);
JB_API int jb_dueling_fwd(const float* adv, const float* val, int B, int A, int K, float* out, void* stream);
JB_API int jb_dueling_bwd(const float* dout, int B, int A, int K, float* dadv, float* dval, void* stream);
JB_API int jb_td_loss(const float* q, const float* q_next, const float* qt_next, const void* action, int action_kind,
                      const float* reward, const float* done, const double* weights, int B, int A, float gamma,
                      float alpha, int n_step, int double_q, int loss_kind, int order, float* dq, double* prio,
                      float* stats, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Distributional learners — jorldy/core/agent/c51.py:62-135, rainbow.py:167-235, :285-292.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_c51_loss(const float* logits, const float* next_online, const float* next_target, const void* action,
                       int action_kind, const float* reward, const float* done, const double* weights, const float* z,
                       int B, int A, int K, float gamma, float v_min, float v_max, float alpha, int n_step, int variant,
                       float* dlogits, float* kl, double* prio, float* stats, float* scratch, void* stream);
JB_API int jb_c51_q(const float* logits, const float* z, int M, int A, int K, float* q, void* stream);

/* ---------------------------------------------------------------------------------------------
 * NoisyNet — jorldy/core/network/utils.py:55-86 (noisy_l), factorised noise.  A drawn (not injected) layer
 * needs in_f + out_f <= 8192, else JB_ERR_INVALID: Philox counter = draw * 4096 + factor / 2.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_noisy_make(const float* mu_w, const float* sig_w, const float* mu_b, const float* sig_b, int in_f,
                         int out_f, const float* eps_i, const float* eps_j, uint64_t seed, uint64_t stream_id,
                         long long* draw_ctr, int is_train, float* f_i, float* f_j, float* w_eff, float* b_eff,
                         void* stream);
JB_API int jb_noisy_grad(const float* dw_eff, const float* db_eff, const float* f_i, const float* f_j, int in_f,
                         int out_f, float* dmu_w, float* dsig_w, float* dmu_b, float* dsig_b, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Optimisers — torch.optim.Adam / RMSprop(centered) via jorldy/core/optimizer/__init__.py:31,
 * torch.nn.utils.clip_grad_norm_ (ppo.py:166-168, ape_x.py:119), target copy dqn.py:153-154.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_grad_partials_count(long long P);
JB_API int jb_grad_sumsq(const float* g, long long P, float* partials, long long* step, void* stream);
/* beta1, beta2 and alpha are doubles so that 1 - beta is formed before rounding to fp32, as torch does */
JB_API int jb_adam_step(float* p, const float* g, float* m, float* v, long long P, const float* lr, double beta1,
                        double beta2, float eps, const long long* step, const float* partials, int n_partials,
                        float max_norm, float* norm_out, void* stream);
JB_API int jb_rmsprop_centered_step(float* p, const float* g, float* square_avg, float* grad_avg, long long P,
                                    const float* lr, double alpha, float eps, const float* partials, int n_partials,
                                    float max_norm, float* norm_out, void* stream);
JB_API int jb_copy_f32(float* dst, const float* src, long long P, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Continuous off-policy family (SURVEY.md 8f-4) — jorldy/core/agent/ddpg.py, td3.py, sac.py; the row / element-wise
 * steps between the dense layers (csrc/actor_critic.cu).
 *   jb_soft_update     t := tau p + (1 - tau) t over a flat buffer            ddpg.py:160-164, td3.py:190-196, sac.py:262-266
 *   jb_tanh_act        out = clip(tanh(pre) + clip(noise*scale, +-noise_clip), +-out_clip); noise NULL: plain tanh head
 *                      (network/policy.py:19-20; td3.py:141-142 act noise; td3.py:153-156 target smoothing)
 *   jb_tanh_bwd        dpre = da (1 - a^2)
 *   jb_ou_act          action = tanh(pre) + clip(X, +-1) with one Ornstein-Uhlenbeck process X[M,A] (f64) per env row and
 *                      ONE normal per row and step (agent/utils.py:8-26, ddpg.py:113-118); greedy: tanh(pre)
 *   jb_philox_fill     standard normals (kind 0) / uniforms in [lo,hi) (kind 1) from the device Philox stream
 *   jb_ac_critic_loss  y = r + ((1-d) gamma)(min(nq1,nq2) + alpha(-next_logp)); dq_i = 2(q_i - y)/B;
 *                      stats = {mse1, mse2, max y}; q2/nq2/alpha/next_logp may be NULL    ddpg.py:131-136, td3.py:150-168, sac.py:172-204
 *   jb_ac_neg_mean     stat = -mean(q), dq = -1/B                              ddpg.py:143-144, td3.py:176-177
 *   jb_sac_sample      a = tanh(mu + std eps), logp with the tanh correction  sac.py:151-160, network/policy.py:50-56
 *   jb_sac_minq        dq_i of L = mean(alpha logp - min(q1,q2)); stats = {L, mean min q, mean entropy, mean entropy - target}
 *   jb_sac_actor_bwd   d L / d (raw mu | raw log_std) [B,2A] from d L / d action and the alpha logp term   sac.py:222-236
 *   jb_sac_alpha       alpha_loss = log_alpha * stats4[3]; alpha := exp(log_alpha); grad := stats4[3]     sac.py:238-246
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_soft_update(float* target, const float* online, int64_t n, double tau, void* stream);
JB_API int jb_tanh_act(const float* pre, const float* noise, int64_t n, float scale, float noise_clip, float out_clip,
                       float* out, void* stream);
JB_API int jb_tanh_bwd(const float* da, const float* a, int64_t n, float* dpre, void* stream);
JB_API int jb_ou_act(const float* pre, int M, int A, double* X, const double* normal, uint64_t seed, uint64_t stream_base,
                     long long* row_ctr, double theta, double mu, double sigma, int greedy, float* action, void* stream);
JB_API int jb_philox_fill(float* out, int64_t n, int kind, float lo, float hi, uint64_t seed, uint64_t stream_base,
                          uint64_t ctr, long long* ctr_dev, void* stream);
JB_API int jb_ac_critic_loss(const float* q1, const float* q2, const float* nq1, const float* nq2, const float* alpha,
                             const float* next_logp, const float* reward, const float* done, int B, float gamma,
                             float* dq1, float* dq2, float* stats, void* stream);
JB_API int jb_ac_neg_mean(const float* q, int B, float* dq, float* stat, void* stream);
JB_API int jb_sac_sample(const float* raw, int nout, const float* eps, int M, int A, float* action, float* logp,
                         void* stream);
JB_API int jb_sac_minq(const float* q1, const float* q2, const float* logp, const float* alpha, float target_entropy,
                       int B, float* dq1, float* dq2, float* stats, void* stream);
JB_API int jb_sac_actor_bwd(const float* raw, int nout, const float* eps, const float* action, const float* da,
                            const float* alpha, int B, int A, float* dout, void* stream);
JB_API int jb_sac_alpha(const float* log_alpha, const float* stats4, float* alpha, float* grad, float* alpha_loss,
                        void* stream);

/* ---------------------------------------------------------------------------------------------
 * Discrete-action SAC (SAC-Discrete, arXiv:1910.07207), A <= 18 actions; logpi = log_softmax(logits), pi = exp(logpi).
 *   jb_sacd_act          a ~ Categorical(pi) by inverse CDF on u[m] (NULL: Philox(seed, stream_base + m, row_ctr[m]++));
 *                        greedy: argmax pi, first index on ties; action int64 [M]
 *   jb_sacd_critic_loss  y = r + ((1-d) gamma) sum_a pi'(a)[min(nq1,nq2)(a) - alpha logpi'(a)] with pi' from next_logits;
 *                        dq_i[b,a_b] = 2(Q_i(s)[a_b] - y)/B, 0 elsewhere; stats = {mse1, mse2, max y}
 *   jb_sacd_actor        f = alpha logpi - min(q1,q2), L_b = sum_a pi f, dlogits = pi (f - L_b)/B;
 *                        stats4 = {mean L, mean sum_a pi min(q1,q2), mean H, mean H - target_entropy}, H = -sum_a pi logpi
 * The two loss kernels run one CTA with fixed-order reductions, so a learn() is bit-reproducible.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_sacd_act(const float* logits, int M, int A, const float* u, uint64_t seed, uint64_t stream_base,
                       long long* row_ctr, int greedy, int64_t* action, void* stream);
JB_API int jb_sacd_critic_loss(const float* q1, const float* q2, const float* nq1, const float* nq2, const float* next_logits,
                               const int64_t* action, const float* reward, const float* done, const float* alpha, int B,
                               int A, float gamma, float* dq1, float* dq2, float* stats, void* stream);
JB_API int jb_sacd_actor(const float* logits, const float* q1, const float* q2, const float* alpha, float target_entropy,
                         int B, int A, float* dlogits, float* stats4, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Quantile regression (QR-DQN arXiv:1710.10044, IQN arXiv:1806.06923), csrc/quantile.cu.
 * A quantile tensor holds A actions x N quantiles per sample at offset b*A*N + a*sa + i*sq:
 * [B, A, K] is (sa, sq) = (K, 1), [B, N, A] is (1, A).
 *   jb_quantile_loss   y_j = r + ((1-d) gamma) next_target[b, a*, j], a* = argmax_a mean_j next_target[b, a, j];
 *                      u_ij = y_j - pred[b, a_b, i], rho = |tau_i - 1{u < 0}| smooth_l1(u), tau_i = tau[b*tau_stride + i]
 *                      (tau_stride 0: one shared set of fractions);
 *                      loss[b] = (1/Np) sum_j sum_i rho_ij, dpred[b, a_b, i] = -(1/(B Np)) sum_j |tau_i - 1{u<0}| clamp(u,-1,1),
 *                      0 on every other action; a_star [B] (may be NULL); stats = {mean_b loss[b], max_{b,a} mean_i pred};
 *                      scratch: 2*B floats.  1 <= A <= 18, 1 <= N, Np <= 256, else JB_ERR_INVALID.  One CTA per sample,
 *                      fixed-order sums: bit-reproducible.
 *   jb_quantile_mean   q [M, A] = mean over the N quantiles of x (same layout convention)
 *   jb_iqn_tau         tau [rows, N] ~ U[lo, hi) from Philox(seed, stream_id, ctr[0] + e/4) word e%4; ctr[0] += ceil(rows*N/4)
 *   jb_iqn_cos         c [rows, E] = cos(pi i tau[r]), i < E
 *   jb_iqn_mul_fwd     z [B, N, D] = psi [B, D] (*) phi [B, N, D]
 *   jb_iqn_mul_bwd     dpsi [B, D] = 1{psi > 0} sum_n dz (*) phi (n ascending; psi is the head's ReLU output, so this is
 *                      the gradient w.r.t. its pre-activation), dpre [B, N, D] = dz (*) psi (*) 1{phi > 0}
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_quantile_loss(const float* pred, int p_sa, int p_sq, const float* next_target, int t_sa, int t_sq,
                            const float* tau, int tau_stride, const void* action, int action_kind, const float* reward,
                            const float* done, int B, int A, int N, int Np, float gamma, float* dpred, float* loss,
                            int32_t* a_star, float* stats, float* scratch, void* stream);
JB_API int jb_quantile_mean(const float* x, int sa, int sq, int M, int A, int N, float* q, void* stream);
JB_API int jb_iqn_tau(float* tau, int rows, int N, float lo, float hi, uint64_t seed, uint64_t stream_id, long long* ctr,
                      void* stream);
JB_API int jb_iqn_cos(const float* tau, int rows, int E, float* c, void* stream);
JB_API int jb_iqn_mul_fwd(const float* psi, const float* phi, int B, int N, int D, float* z, void* stream);
JB_API int jb_iqn_mul_bwd(const float* dz, const float* psi, const float* phi, int B, int N, int D, float* dpsi, float* dpre,
                          void* stream);

/* ---------------------------------------------------------------------------------------------
 * Rainbow-IQN (Toromanoff et al. arXiv:1908.04683: IQN with Rainbow's double-Q, n-step targets and prioritised replay),
 * csrc/quantile.cu.  [B, N, A] layout only: pred [B, N, A] (online on s), next_online [B, Nn, A] (online on s'),
 * next_target [B, Np, A] (target on s'), tau [B, N], reward / done [B, n_step].
 *   a*   = argmax_a mean_j next_online[b, j, a], first index on ties (double-Q);
 *   y_j  = fold_{s = n_step-1 .. 0} (r_s + ((1 - d_s) gamma) y), from y = next_target[b, j, a*]  (c51.cu's float order);
 *   L_b  = (1/Np) sum_j sum_i |tau_i - 1{u_ij < 0}| smooth_l1(u_ij), u_ij = y_j - pred[b, i, a_b]   (kappa = 1);
 *   dpred[b, i, a_b] = -(w_b / (B Np)) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -1, 1), 0 on every other action;
 *   loss [B] = the unweighted L_b, prio [B] (f64, may be NULL) = L_b^alpha, a_star [B] (may be NULL);
 *   stats = {(1/B) sum_b w_b L_b, max_{b,a} mean_i pred, max pred, min pred}; scratch: 4*B floats.
 * weights [B] are the f64 IS weights, each sample its own (NULL = all ones).  1 <= A <= 18, 1 <= N, Nn, Np <= 256,
 * n_step >= 1, else JB_ERR_INVALID.  One CTA per sample, fixed-order sums, a single-thread finalize: bit-reproducible.
 * With n_step = 1, next_online == next_target and weights NULL (or all ones), dpred, loss, a_star and stats[0..1] equal
 * jb_quantile_loss's on the [B, N, A] layout bit for bit.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_rainbow_iqn_loss(const float* pred, const float* next_online, const float* next_target, const float* tau,
                               const void* action, int action_kind, const float* reward, const float* done,
                               const double* weights, int B, int A, int N, int Nn, int Np, int n_step, float gamma,
                               float alpha, float* dpred, float* loss, double* prio, int32_t* a_star, float* stats,
                               float* scratch, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Munchausen RL (M-DQN, M-IQN; Vieillard, Pietquin, Geist 2020, arXiv:2007.14430), csrc/munchausen.cuh with
 * csrc/dqn.cu and csrc/quantile.cu.  q'(s, .) and q'(s', .) are the TARGET network's Q; tau is the entropy temperature
 * (m_tau), alpha the Munchausen scale (m_alpha), l0 the clip floor.  Per sample, one thread, actions ascending:
 *   tau logpi(a|s)  = (q'(s,a) - m) - tau log sum_b exp((q'(s,b) - m)/tau),  m = max_b q'(s,b)   (log(pi) is never formed)
 *   pi'(a)          = softmax(q'(s',.)/tau)(a),  tau logpi'(a|s') in the same stable form
 *   bonus           = alpha clip(tau logpi(a_t|s), l0, 0)        (clipped first, then scaled)
 *   jb_mdqn_loss    y = r + bonus + ((1-d) gamma) sum_a pi'(a) (qt_next[b,a] - tau logpi'(a|s')), q' = qt_s / qt_next [B, A];
 *                   loss = mean_b smooth_l1(q[b, a_b] - y), dq[b, a_b] = smooth_l1'(q - y)/B, 0 on every other action;
 *                   stats = {loss, max_b q[b, a_b]}; reward / done [B]; scratch: 2*B floats.  One warp per sample.
 *   jb_munchausen_quantile_loss
 *                   [B, N, A] layout only (pred, next_target [B, Np, A], cur_target [B, Nc, A]); q'(s, .) and q'(s', .)
 *                   are the means over cur_target's Nc and next_target's Np quantiles;
 *                   y_j = r + bonus + ((1-d) gamma) sum_a pi'(a) (next_target[b, j, a] - tau logpi'(a|s'));
 *                   the loss and dpred are jb_quantile_loss's quantile Huber (kappa = 1) on these y_j with the
 *                   fractions tau[b*tau_stride + i]; stats = {mean_b loss[b], max_{b,a} mean_i pred}; scratch: 2*B floats.
 *                   One CTA per sample.
 * Both: 1 <= A <= 18, 1 <= N, Np, Nc <= 256, m_tau > 0, l0 <= 0, else JB_ERR_INVALID.  Fixed-order sums and a single-thread
 * finalize, no atomics: bit-reproducible.  At m_alpha = 0 with m_tau -> 0 and a unique argmax, pi' is one-hot and both
 * reduce to jb_td_loss (order 0) and jb_quantile_loss.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_mdqn_loss(const float* q, const float* qt_s, const float* qt_next, const void* action, int action_kind,
                        const float* reward, const float* done, int B, int A, float gamma, float m_alpha, float m_tau,
                        float l0, float* dq, float* stats, float* scratch, void* stream);
JB_API int jb_munchausen_quantile_loss(const float* pred, const float* next_target, const float* cur_target, const float* tau,
                                       int tau_stride, const void* action, int action_kind, const float* reward,
                                       const float* done, int B, int A, int N, int Np, int Nc, float gamma, float m_alpha,
                                       float m_tau, float l0, float* dpred, float* stats, float* scratch, void* stream);

/* ---------------------------------------------------------------------------------------------
 * R2D2 (Kapturowski et al., ICLR 2019): a recurrent dueling Q-network on replayed sequences, csrc/lstm.cu and csrc/r2d2.cu.
 * The LSTM uses torch.nn.LSTM's layout and gate order i, f, g, o (weight_hh [4H, H]); the caller forms the input
 * projection of all time steps at once, xg = x W_ih^T + b_ih + b_hh [rows, 4H], with jb_linear_fwd.
 *   jb_lstm_step_fwd   one step over M rows: i, f, o = sigm(xg + h_prev W_hh^T), g = tanh(.), c = f c_prev + i g,
 *                      h = o tanh(c); gates [M, 4H] receives the post-activation (i, f, g, o).  reset [M] (may be NULL):
 *                      rows with reset != 0 read h_prev and c_prev as zero (an episode starts at this step).  hprev_eff
 *                      (may be NULL) receives h_prev with those rows zeroed, the operand of dW_hh.  c may alias c_prev;
 *                      h and hprev_eff must not alias h_prev.
 *   jb_lstm_step_bwd   dh = dh_out + (dgates_next W_hh) and dcell = dh o (1 - tanh^2 c) + dc_next, where the two recurrent
 *                      terms are dropped on rows with reset_next != 0 (the next step did not read this step's state);
 *                      dgates [M, 4H] = d loss / d (i, f, g, o pre-activations), with c_prev read as zero where reset != 0;
 *                      dc [M, H] (may be NULL, may alias dc_next) = dcell f, the gradient into the c_prev this step read.
 *                      dh_out, dgates_next, dc_next, reset, reset_next may be NULL (zero / no reset).
 *                      A CTA owns 8 hidden units and 32 rows; fp32 FFMA in ascending k, no atomics: bit-reproducible.
 *   jb_r2d2_loss       q, q_next (online on s, s'), qt_next (target on s') [B, T, A]; action int64 [B, T];
 *                      reward / done [B, T + n_step] (step t uses columns t .. t + n_step - 1); weights f64 [B] or NULL;
 *                      a* = argmax_a q_next[b, t, a] (first index on ties);
 *                      y = h(fold_{i = n-1 .. 0} (r_{t+i} + (1 - d_{t+i}) gamma y)) from y = h^-1(qt_next[b, t, a*]),
 *                      h(x) = sign(x)(sqrt(|x| + 1) - 1) + 1e-3 x;  td = y - q[b, t, a_t];
 *                      loss = (1/(B T)) sum_b sum_t w_b td^2, dq = its gradient (on the taken action only, 0 elsewhere);
 *                      prio [B] (f64, may be NULL) = (eta max_t |td| + (1 - eta) mean_t |td|)^alpha from the unweighted td;
 *                      stats = {loss, max_{b,t} q[b, t, a_t]}; scratch: 2*B doubles.  Targets and sums in float64.
 *                      1 <= A <= 18, n_step >= 1, B, T >= 1, else JB_ERR_INVALID.  One CTA per sequence, fixed-order
 *                      sums and a single-thread finalize: bit-reproducible.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_lstm_step_fwd(const float* xg, const float* h_prev, const float* c_prev, const float* w_hh, const float* reset,
                            int M, int H, float* h, float* c, float* gates, float* hprev_eff, void* stream);
JB_API int jb_lstm_step_bwd(const float* dh_out, const float* dgates_next, const float* w_hh, const float* gates,
                            const float* c_prev, const float* c, const float* dc_next, const float* reset,
                            const float* reset_next, int M, int H, float* dgates, float* dc, void* stream);
JB_API int jb_r2d2_loss(const float* q, const float* q_next, const float* qt_next, const int64_t* action, const float* reward,
                        const float* done, const double* weights, int B, int T, int A, int n_step, float gamma, float alpha,
                        float eta, float* dq, double* prio, float* stats, double* scratch, void* stream);

/* ---------------------------------------------------------------------------------------------
 * MuZero (Schrittwieser et al., arXiv:1911.08265) on flat observations, csrc/muzero.cu.  h(x) = sign(x)(sqrt(|x| + 1) - 1)
 * + 1e-3 x; a support of V has the 2V + 1 integer atoms -V..V (1 <= V <= 300).  One warp per row / env / (window,
 * position), fixed-order sums, no atomics: every entry point is bit-reproducible.
 *   jb_muzero_scale_fwd   y [M, H] = (x - min) / max(max - min, 1e-5) per row (H <= 256); also into y2 [M, ld2] if not NULL.
 *   jb_muzero_scale_bwd   dx of that map from x and dy: dy / s, plus d min at the argmin and d max at the argmax (lowest
 *                         index on ties); with the range clamped, s is a constant and d max = 0.
 *   jb_muzero_support_to_scalar  out [M] = h^-1(sum_i softmax(logits)_i (i - V)), logits [M, 2V + 1].
 *   jb_muzero_scalar_to_support  out [M, 2V + 1] = two-hot of clamp(h(x), -V, V) on the integer atoms.
 *   Search trees: one per env, S + 1 nodes of A edges (1 <= A <= 18), index e = (env (S + 1) + node) A + action.  An edge
 *   holds edge_n (int32), edge_w, edge_p, edge_r (f32) and edge_child (int32, -1: not expanded); latent [N, S + 1, Hs];
 *   count [N] nodes in use; bounds [N, 2] the min and max backed-up Q; path [N, S + 1] the last walk's edges (node A + a),
 *   path_len [N].
 *   jb_mcts_root          priors = softmax(pi_logits [N, A]); training: (1 - frac) priors + frac Dirichlet(dir_alpha), the
 *                         gamma draws injected (gamma_in f64 [N, A]) or drawn as Gamma(alpha + 1) U^(1/alpha) by
 *                         Marsaglia-Tsang on the Philox subsequence (seed, env << 8 | a) at the row counter
 *                         jb_next_row_ctr(row_ctr, env); resets the tree with latent0 [N, Hs] at node 0;
 *                         root_value [N] (may be NULL) = support_to_scalar(v_logits [N, 2V + 1]).
 *   jb_mcts_select        one walk per env from the root by pUCT (c1 = 1.25, c2 = 19652): Q = R + gamma W / N normalised
 *                         by the bounds (when max > min), 0 on an unvisited edge, ties to the lowest action; writes the path,
 *                         leaf_node / leaf_action [N] (the unexpanded edge) and dyn_in [N, Hs + A] = [latent, onehot(a)].
 *   jb_mcts_expand_backup stores latent_new [N, Hs] and softmax(pi_logits) at node count[env], the scalar reward of
 *                         r_logits [N, 2R + 1] on the leaf edge, and backs G = support_to_scalar(v_logits) up the path
 *                         leaf first: W += G, N += 1, bounds <- R + gamma W / N, G = R + gamma G.
 *   jb_mcts_act           pi [N, A] = N(a) / sum N at the root; root_value [N] (may be NULL) = sum_a (N R + gamma W) /
 *                         sum N; action [N] int64: training samples N(a)^(1 / temperature[0]) with u_in f64 [N] or a
 *                         Philox uniform at the row counter, else argmax N (lowest index on ties).
 *   jb_muzero_loss        B windows of L = K + n_step + 1 steps: reward, done, root_value [B, L], policy [B, L, A];
 *                         logits time-major: pi [K + 1, B, A], v [K + 1, B, 2V + 1], r [K, B, 2R + 1] (r[k - 1] predicts
 *                         position k).  z_k = fold_{i = n-1..0} (r_{k+i} + (1 - d_{k+i}) gamma z) from root_value_{k+n};
 *                         a position after a done in the window is absorbing: z = 0, no policy loss, and a reward target
 *                         r_{k-1} only when position k - 1 is not absorbing.  loss = (1/B) sum_b w_b sum_k c_k
 *                         (value_coef CE_v + CE_r [k >= 1] + CE_pi), c_0 = 1, c_k = 1/K; weights f64 [B] or NULL;
 *                         d_pi, d_v, d_r its gradients (same layouts); prio [B] f64 (may be NULL) = |v_0 - z_0|^alpha;
 *                         stats = {loss, value_loss, reward_loss, policy_loss}; scratch: 3 B (K + 1) doubles.
 * ------------------------------------------------------------------------------------------- */
JB_API int jb_muzero_scale_fwd(const float* x, int M, int H, float* y, float* y2, int ld2, void* stream);
JB_API int jb_muzero_scale_bwd(const float* x, const float* dy, int M, int H, float* dx, void* stream);
JB_API int jb_muzero_support_to_scalar(const float* logits, int M, int V, float* out, void* stream);
JB_API int jb_muzero_scalar_to_support(const float* x, int M, int V, float* out, void* stream);
JB_API int jb_mcts_root(const float* pi_logits, const float* v_logits, const float* latent0, int N, int A, int S, int Hs,
                        int V, int training, float dir_alpha, float frac, const double* gamma_in, uint64_t seed,
                        long long* row_ctr, int* edge_n, float* edge_w, float* edge_p, float* edge_r, int* edge_child,
                        float* latent, int* count, float* bounds, int* path, int* path_len, float* root_value,
                        void* stream);
JB_API int jb_mcts_select(int N, int A, int S, int Hs, float gamma, int* edge_n, float* edge_w, float* edge_p,
                          float* edge_r, int* edge_child, float* latent, int* count, float* bounds, int* path,
                          int* path_len, int* leaf_node, int* leaf_action, float* dyn_in, void* stream);
JB_API int jb_mcts_expand_backup(const float* latent_new, const float* pi_logits, const float* v_logits,
                                 const float* r_logits, int N, int A, int S, int Hs, int V, int R, float gamma,
                                 const int* leaf_node, const int* leaf_action, int* edge_n, float* edge_w, float* edge_p,
                                 float* edge_r, int* edge_child, float* latent, int* count, float* bounds, int* path,
                                 int* path_len, void* stream);
JB_API int jb_mcts_act(int N, int A, int S, float gamma, int training, const float* temperature, const double* u_in,
                       uint64_t seed, long long* row_ctr, const int* edge_n, const float* edge_w, const float* edge_r,
                       int64_t* action, float* pi, float* root_value, void* stream);
JB_API int jb_muzero_loss(const float* pi_logits, const float* v_logits, const float* r_logits, const float* reward,
                          const float* done, const float* root_value, const float* policy, const double* weights, int B,
                          int K, int n_step, int A, int V, int R, float gamma, float value_coef, float alpha, float* d_pi,
                          float* d_v, float* d_r, double* prio, float* stats, double* scratch, void* stream);

#endif /* JORLDY_B200_H */
