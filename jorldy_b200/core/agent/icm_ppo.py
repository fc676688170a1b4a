"""ICM-PPO agent (Pathak et al., ICML 2017, "Curiosity-driven Exploration by Self-supervised Prediction") on the PPO
rollout path.

Everything up to the reward jb_gae reads is PPO's (act, the batched rollout, the pre-pass, the CUDA-graph minibatch loop
driven by the device cursor).  Before jb_gae the ICM pre-pass replaces the extrinsic reward r with
extrinsic_coeff * r + intrinsic_coeff * r_i:
  1. rms_obs (float64 RunningMeanStd) is updated with the rollout's next states (obs_normalize);
  2. r_i = eta / 2 * sum_F |f - phi(s')| for all N*T rows, no gradient, with both BatchNorms in training mode over the
     whole rollout as one batch (the reference's module is never put in eval mode);
  3-5. (ri_normalize) each env's reward-forward filter rewems = gamma * rewems + r_i runs over t (its state persists
     across learns), rms_ri is updated with the filtered values, and r_i is divided by sqrt(rms_ri.var) + 1e-7.
One minibatch step = PPO's forward -> jb_ppo_loss (head gradient scaled by lamb) -> backward -> clip + Adam on the
policy network, then the ICM forward -> jb_icm_loss (beta * l_f + (1 - beta) * l_i) -> ICM backward -> Adam on the ICM.
Adam is per element and the two parameter sets are disjoint, so the two flat Adams with the same lr, betas and eps equal
one torch Adam over network + ICM parameters with clip_grad_norm_ on the network's parameters only.

The running statistics are not checkpointed (the reference does not save them).
"""
import os

import numpy as np
import torch

from ..dev import C, ptr, stream_ptr
from ..network.icm import FEATURE, ICM_MLP
from ..optimizer import Optimizer
from .base import cpu_state_dict
from .curiosity import _RunningMeanStd, check_batch_norm_rows, load_two_adam_state, two_adam_state
from .ppo import PPO

ICM_NETWORKS = {"icm_mlp": "mlp", "icm_cnn": "cnn"}       # ICM network -> the policy head (observation kind) it pairs with


class ICM_PPO(PPO):
    _GRAPH_INPUTS = PPO._GRAPH_INPUTS + ("icm_next",)     # icm_next: the next-state rows the ICM reads
    replicas_only = True          # parallel.attach: BatchNorm batch statistics and the running statistics are per replica
    FAMILY = "ICM-PPO"
    needs_next_state = True       # RolloutCollector: keep every step's next state in the rollout

    def __init__(self, state_size, action_size, optim_config={"name": "adam"}, icm_network="icm_mlp", beta=0.2, lamb=1.0,
                 eta=0.01, extrinsic_coeff=1.0, intrinsic_coeff=1.0, obs_normalize=True, ri_normalize=True,
                 batch_norm=True, **kwargs):
        if icm_network not in ICM_NETWORKS:
            raise ValueError(f"ICM-PPO: unknown icm_network={icm_network!r} (available: {', '.join(ICM_NETWORKS)})")
        head = kwargs.get("head", "mlp")
        if ICM_NETWORKS[icm_network] != head:
            raise ValueError(f"ICM-PPO: icm_network={icm_network!r} takes the observations of head="
                             f"{ICM_NETWORKS[icm_network]!r}, got head={head!r}")
        if icm_network == "icm_cnn" and obs_normalize:
            raise ValueError("ICM-PPO: icm_cnn needs obs_normalize=False; per-pixel observation normalisation of frames "
                             "is not implemented")
        kwargs["use_fused"] = False       # the persistent kernel computes PPO's loss only
        super().__init__(state_size, action_size, optim_config=optim_config, **kwargs)
        self.beta, self.lamb, self.eta = float(beta), float(lamb), float(eta)
        self.extrinsic_coeff, self.intrinsic_coeff = float(extrinsic_coeff), float(intrinsic_coeff)
        self.obs_normalize, self.ri_normalize, self.batch_norm = bool(obs_normalize), bool(ri_normalize), bool(batch_norm)
        D = int(np.prod(state_size))
        cnn = icm_network == "icm_cnn"
        self.icm = ICM_MLP(state_size if cnn else D, action_size, self.action_type, batch_norm=self.batch_norm,
                           device=self.device, seed=self.seed, cnn=cnn)
        self.icm_optimizer = Optimizer(**dict(optim_config), params=self.icm.parameters())
        self.rms_obs = _RunningMeanStd((D,), self.device) if self.obs_normalize else None
        self.rms_ri = _RunningMeanStd((1,), self.device)
        self.rewems = None                # [N] reward-forward filter state, created at the first learn
        self._icm_acc = torch.zeros(4, dtype=torch.float32, device=self.device)

    # ----------------------------------------------------------------------------------- learn --
    def _check_batch(self, NT):
        check_batch_norm_rows(self.FAMILY, self.batch_norm, self.batch_size, NT)

    def _gae_reward(self, st, reward, next_state, N, T):
        NT = N * T
        self._check_batch(NT)
        if next_state is None:
            raise ValueError("ICM-PPO needs every step's next state (a rollout with next_state, or host transitions)")
        st["icm_next"] = next_state
        s_ = stream_ptr()
        icm, D = self.icm, self.icm.D_in
        if self.obs_normalize:
            part = icm._buf("rms.partials", (C.jb_col_partials_doubles(NT, D),), torch.float64)
            C.jb_rms_update(ptr(next_state), NT, D, *(ptr(t) for t in self.rms_obs.tensors()), ptr(part), s_)
        rms = (self.rms_obs.mean, self.rms_obs.var) if self.obs_normalize else None
        chunk = icm.head.max_rows if icm.head is not None else None     # conv1's im2col is 400 KB a row
        f, phi_next, _ = icm.forward(st["state"], next_state, st["action"], None, NT, rms=rms, inverse=False, tag="pre.",
                                     chunk_rows=chunk)
        ri = icm._buf("pre.ri", (NT,))
        C.jb_icm_loss(int(self.continuous), ptr(f), ptr(phi_next), 2 * FEATURE, 0, 0, 0, NT, self.action_size, FEATURE,
                      self.eta, self.beta, ptr(ri), 0, 0, 0, 0, s_)
        if self.rewems is None or self.rewems.shape[0] != N:
            self.rewems = torch.zeros(N, dtype=torch.float32, device=self.device)
        out = icm._buf("pre.reward", (NT,))
        if self.ri_normalize:
            part = icm._buf("ri.partials", (C.jb_col_partials_doubles(NT, 1),), torch.float64)
            C.jb_icm_reward(ptr(reward), ptr(ri), N, T, self.gamma, 1, ptr(self.rewems),
                            *(ptr(t) for t in self.rms_ri.tensors()), ptr(part), ptr(icm._buf("pre.filt", (NT,))),
                            self.extrinsic_coeff, self.intrinsic_coeff, ptr(out), s_)
        else:
            C.jb_icm_reward(ptr(reward), ptr(ri), N, T, self.gamma, 0, 0, 0, 0, 0, 0, 0, self.extrinsic_coeff,
                            self.intrinsic_coeff, ptr(out), s_)
        return out

    def _minibatch_step(self, st, idx, B):
        net, icm = self.network, self.icm
        tag = f"mb{B}."
        s_ = stream_ptr()
        out = net.forward_raw(st["state"], idx, B, tag=tag)
        dout = net._buf(tag + "dout", (B, net.nout))
        stats = net._buf(tag + "stats", (8 + 4 * ((B + 255) // 256),))
        C.jb_ppo_loss(int(self.continuous), ptr(out), ptr(idx), ptr(st["action"]), ptr(st["adv"]), ptr(st["ret"]),
                      ptr(st["value"]), ptr(st["logp_old"]), B, self.action_size, net.nout, self.epsilon_clip,
                      self.vf_coef, self.ent_coef, ptr(dout), ptr(stats), ptr(self._acc), s_)
        if self.lamb != 1.0:
            C.jb_scale_f32(ptr(dout), B * net.nout, self.lamb, s_)
        net.backward_raw(dout, B, tag=tag)
        self.optimizer.step(max_norm=self.clip_grad_norm)
        itag = tag + "icm."
        rms = (self.rms_obs.mean, self.rms_obs.var) if self.obs_normalize else None
        f, phi_next, g = icm.forward(st["state"], st["icm_next"], st["action"], idx, B, rms=rms, tag=itag)
        df, dg = icm._buf(itag + "df", (B, FEATURE)), icm._buf(itag + "dg", (B, self.action_size))
        istats = icm._buf(itag + "stats", (4 + 3 * ((B + 7) // 8),))
        C.jb_icm_loss(int(self.continuous), ptr(f), ptr(phi_next), 2 * FEATURE, ptr(g), ptr(idx), ptr(st["action"]), B,
                      self.action_size, FEATURE, self.eta, self.beta, 0, ptr(df), ptr(dg), ptr(istats),
                      ptr(self._icm_acc), s_)
        icm.backward(df, dg, B, tag=itag)
        self.icm_optimizer.step()

    @property
    def LAUNCHES_PER_MINIBATCH(self):
        # PPO's 13 (+1 for the lamb scale), then the ICM.  Forward: 2 normalise + fc1 + BN-ELU (2 x 3, or 1 ELU) + fc2
        # + 2 ELU + 2 action rows + fc_f1 + fc_f2 + inv + pi + loss + finalize.  Backward: 2 per pi / inv / fc_f2 / fc_f1
        # + 2 ELU + 2 fc2 + BN-ELU (2 x 5, or 1 ELU) + fc1.  Then sumsq + adam.  icm_cnn: the trunk (3 im2col + 3 GEMM +
        # layout) replaces the 2 normalise launches, and its backward adds fc1's dx, the layout, 3 dW and 2 (dx + col2im).
        bn_f, bn_b = (6, 10) if self.batch_norm else (1, 1)
        trunk = (5, 9) if self.icm.head is not None else (0, 0)
        return 13 + (self.lamb != 1.0) + 14 + bn_f + 13 + bn_b + 2 + sum(trunk)

    def _step_state(self):
        return super()._step_state() + [self.icm.flat, *self.icm.buffer_tensors(), *self.icm_optimizer.state_tensors(),
                                        self._icm_acc]

    def _begin_epochs(self):
        super()._begin_epochs()
        self.icm_optimizer._sync_lr()
        self._icm_acc.zero_()

    def _learn_result(self, mean_ret):
        v = torch.cat([self._acc[:6], mean_ret.view(1), self._icm_acc]).cpu().numpy()     # ONE device->host read
        cnt, icnt = max(v[5], 1.0), max(v[10], 1.0)
        return {
            "actor_loss": float(v[0] / cnt),
            "critic_loss": float(v[1] / cnt),
            "entropy_loss": float(v[2] / cnt),
            "max_ratio": float(v[3]),
            "min_prob": float(v[4]),
            "mean_ret": float(v[6]),
            "r_i": float(v[7] / icnt),
            "l_f": float(v[8] / icnt),
            "l_i": float(v[9] / icnt),
        }

    def learning_rate_decay(self, step, optimizers=None, mode="cosine"):
        super().learning_rate_decay(step, [self.optimizer, self.icm_optimizer] if optimizers is None else optimizers, mode)

    # ------------------------------------------------------------------------------ checkpoint --
    # network / icm / optimizer, the optimizer one torch-Adam layout over network.parameters() + icm.parameters().
    def save(self, path):
        print(f"...Save model to {path}...")
        ck = {"network": cpu_state_dict(self.network), "icm": cpu_state_dict(self.icm),
              "optimizer": two_adam_state(self.optimizer, self.icm_optimizer)}
        torch.save(ck, os.path.join(path, "ckpt"))

    def load(self, path):
        print(f"...Load model from {path}...")
        ck = torch.load(os.path.join(path, "ckpt"), map_location="cpu", weights_only=False)
        self.network.load_state_dict(ck["network"])
        self.icm.load_state_dict(ck["icm"])
        load_two_adam_state(ck["optimizer"], self.optimizer, self.icm_optimizer)
