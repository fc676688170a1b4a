"""RND-PPO agent (Burda et al., 2018, arXiv:1810.12894, "Exploration by Random Network Distillation") on the PPO rollout
path.

The policy network is PPO's with a second value head v_i (core/network/policy_value.py *PolicyTwoValue).  One learn:
  1. rms_obs (float64 RunningMeanStd) is updated with the rollout's next states (obs_normalize);
  2. the frozen target's features of all N*T next states are computed once into a cached [N*T, F] matrix, which every
     minibatch reads (neither the target nor rms_obs changes during the epochs);
  3. the predictor runs over all N*T rows as one batch (its BatchNorm normalises the whole rollout) and
     r_i = mean_F (p - t)^2;
  4. (ri_normalize) each env's reward-forward filter (gamma_i, state persisting across learns) updates rms_ri and
     r_i is divided by sqrt(rms_ri.var) + 1e-7;
  5. the pre-pass gives logp_old, v_e and v_i of s, and v_e', v_i' of s' from the next-state rows on both the host and the
     resident path;
  6. jb_gae runs per stream: extrinsic (r, done, gamma), intrinsic (r_i, non_episodic ? 0 : done, gamma_i);
  7. adv = extrinsic_coeff adv_e + intrinsic_coeff adv_i, standardised per row (use_standardization); the critics learn
     the unscaled ret_e and ret_i.
One minibatch step = forward -> jb_rnd_ppo_loss (PPO's actor and entropy terms, two clipped critics) -> backward -> clip
+ Adam on the policy network, then the predictor's forward of the B rows -> jb_rnd_loss against the cached target rows
-> predictor backward -> Adam on the predictor.  The two flat Adams equal one torch Adam over network + predictor
parameters with clip_grad_norm_ on the network's parameters only.

The running statistics are not checkpointed, as for ICM-PPO.
"""
import numpy as np
import torch

from ..dev import C, ptr, stream_ptr
from ..network.policy_value import ContinuousPolicyTwoValue, DiscretePolicyTwoValue
from ..network.rnd import FEATURE, RND
from ..optimizer import Optimizer
from .curiosity import CuriosityPPO
from .ppo import MAX_ACTION_SIZE

TWO_VALUE_NETWORKS = {"discrete_policy_value": DiscretePolicyTwoValue, "continuous_policy_value": ContinuousPolicyTwoValue}


class RND_PPO(CuriosityPPO):
    # rnd_next: the next-state rows the predictor reads; rnd_target: the cached target features
    _GRAPH_INPUTS = CuriosityPPO._GRAPH_INPUTS + ("value_i", "ret_i", "rnd_next", "rnd_target")
    FAMILY = "RND-PPO"
    NETWORKS = {"rnd_mlp": "mlp", "rnd_cnn": "cnn"}
    KEY = "rnd"

    def __init__(self, state_size, action_size, optim_config={"name": "adam"}, rnd_network="rnd_mlp", gamma_i=0.99,
                 extrinsic_coeff=2.0, intrinsic_coeff=1.0, obs_normalize=True, ri_normalize=True, batch_norm=True,
                 non_episodic=True, **kwargs):
        network = kwargs.get("network", "discrete_policy_value")
        if network not in TWO_VALUE_NETWORKS:
            raise ValueError(f"RND-PPO: network={network!r} has no two-value variant (available: "
                             f"{', '.join(TWO_VALUE_NETWORKS)})")
        max_a = MAX_ACTION_SIZE[network.split("_")[0]]
        if not 1 <= action_size <= max_a:
            raise ValueError(f"RND-PPO's {network.split('_')[0]} kernels take 1 to {max_a} actions, got "
                             f"action_size={action_size}")
        super().__init__(state_size, action_size, rnd_network, optim_config, extrinsic_coeff, intrinsic_coeff,
                         obs_normalize, ri_normalize, batch_norm, **kwargs)
        self.network = TWO_VALUE_NETWORKS[network](state_size, action_size, D_hidden=kwargs.get("hidden_size", 512),
                                                   head=kwargs.get("head", "mlp"), device=self.device)
        self.optimizer = Optimizer(**dict(optim_config), params=self.network.parameters())
        self.gamma_i, self.non_episodic = float(gamma_i), bool(non_episodic)
        cnn = rnd_network == "rnd_cnn"
        self.rnd = RND(state_size if cnn else int(np.prod(state_size)), batch_norm=self.batch_norm, device=self.device,
                       seed=self.seed, cnn=cnn)
        self.rnd_optimizer = Optimizer(**dict(optim_config), params=self.rnd.parameters())
        self._rnd_acc = torch.zeros(2, dtype=torch.float32, device=self.device)
        self._ri_mean = None

    # ----------------------------------------------------------------------------------- learn --
    def _intrinsic_reward(self, s_next, N, T):
        """Steps 1-4: r_i of every row, normalised when ri_normalize; fills the target cache."""
        NT = N * T
        pred = self.rnd.predictor
        self._update_rms_obs(pred, s_next, NT)
        ri = pred._buf("pre.ri", (NT,))
        self.rnd.prepass(s_next, NT, self._rms(), ri)
        if not self.ri_normalize:
            return ri
        return self._filtered_reward(pred, "pre.ri_hat", ri, ri, N, T, self.gamma_i, 0.0, 1.0)

    def _advantages(self, st, state, action, reward, done, next_state, last_next_state, next_rows, N, T):
        net = self.network
        NT = N * T
        s = stream_ptr()
        s_next = st["rnd_next"] = self._next_rows(next_state if next_state is not None else next_rows, NT)
        ri = self._intrinsic_reward(s_next, N, T)
        st["rnd_target"] = self.rnd.target_cache(NT)
        self._ri_mean = ri.mean()
        buf = lambda k: net._buf("rnd." + k, (NT,))
        st["value_i"], st["ret_i"] = buf("value_i"), buf("ret_i")
        # ---- pre-pass: logp_old, v_e, v_i of s; v_e', v_i' of s' ----
        net.forward_rows(state, st["out"])
        C.jb_rnd_prepass(int(self.continuous), ptr(st["out"]), ptr(action), NT, self.action_size, net.nout,
                         ptr(st["value"]), ptr(st["value_i"]), ptr(st["logp_old"]), s)
        nout = net._buf("next.out", (NT, net.nout))
        net.forward_rows(s_next, nout)
        st["next_value"].copy_(nout[:, -2])
        nv_i = buf("next_value_i")
        nv_i.copy_(nout[:, -1])
        # ---- one jb_gae per stream, then the weighted sum and the per-row standardisation ----
        adv_e, adv_i = buf("adv_e"), buf("adv_i")
        C.jb_gae(ptr(reward), ptr(done), ptr(st["value"]), ptr(st["next_value"]), 0, N, T, self.gamma, self._lambda, 0,
                 ptr(adv_e), ptr(st["ret"]), s)
        if self.non_episodic:
            done_i = buf("no_done")
            done_i.zero_()
        else:
            done_i = done
        C.jb_gae(ptr(ri), ptr(done_i), ptr(st["value_i"]), ptr(nv_i), 0, N, T, self.gamma_i, self._lambda, 0,
                 ptr(adv_i), ptr(st["ret_i"]), s)
        C.jb_adv_mix(ptr(adv_e), ptr(adv_i), N, T, self.extrinsic_coeff, self.intrinsic_coeff,
                     int(self.use_standardization), ptr(st["adv"]), s)
        return st["ret"].mean()

    def _loss(self, st, idx, B, out, dout, tag):
        stats = self.network._buf(tag + "stats", (8 + 4 * ((B + 255) // 256),))
        C.jb_rnd_ppo_loss(int(self.continuous), ptr(out), ptr(idx), ptr(st["action"]), ptr(st["adv"]), ptr(st["ret"]),
                          ptr(st["value"]), ptr(st["ret_i"]), ptr(st["value_i"]), ptr(st["logp_old"]), B,
                          self.action_size, self.network.nout, self.epsilon_clip, self.vf_coef, self.ent_coef,
                          ptr(dout), ptr(stats), ptr(self._acc), stream_ptr())

    def _after_step(self, st, idx, B, tag):
        rtag = tag + "rnd."
        pred = self.rnd.predictor
        p = self.rnd.predict(st["rnd_next"], idx, B, self._rms(), rtag)
        dp = pred._buf(rtag + "dp", (B, FEATURE))
        rstats = pred._buf(rtag + "stats", (1 + (B + 7) // 8,))
        C.jb_rnd_loss(ptr(p), ptr(st["rnd_target"]), ptr(idx), B, FEATURE, 0, ptr(dp), ptr(rstats), ptr(self._rnd_acc),
                      stream_ptr())
        self.rnd.backward(dp, B, rtag)
        self.rnd_optimizer.step()

    @property
    def LAUNCHES_PER_MINIBATCH(self):
        # PPO's 13 (jb_rnd_ppo_loss + finalize in place of jb_ppo_loss's two), then the predictor.  Forward: normalise +
        # fc1 + BN-ELU (3, or 1 ELU) + fc2 + ELU + fc3 + loss + finalize.  Backward: 2 per fc3 / fc2 + ELU + BN-ELU (5, or
        # 1 ELU) + fc1's dW.  Then sumsq + adam.  rnd_cnn: the trunk (3 im2col + 3 GEMM + layout) replaces the normalise
        # launch, and its backward adds fc1's dx, the layout, 3 dW and 2 (dx + col2im).
        bn_f, bn_b = (3, 5) if self.batch_norm else (1, 1)
        trunk = (6, 9) if self.rnd.cnn else (0, 0)
        return 13 + 7 + bn_f + 6 + bn_b + 2 + sum(trunk)

    def _learn_result(self, mean_ret):
        v = torch.cat([self._acc[:6], mean_ret.view(1), self._rnd_acc, self._ri_mean.view(1)]).cpu().numpy()  # ONE read
        cnt, rcnt = max(v[5], 1.0), max(v[8], 1.0)
        return {
            "actor_loss": float(v[0] / cnt),
            "critic_loss": float(v[1] / cnt),
            "entropy_loss": float(v[2] / cnt),
            "max_ratio": float(v[3]),
            "min_prob": float(v[4]),
            "mean_ret": float(v[6]),
            "r_i": float(v[9]),
            "rnd_loss": float(v[7] / rcnt),
        }
