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
import numpy as np
import torch

from ..dev import C, ptr, stream_ptr
from ..network.icm import FEATURE, ICM_MLP
from ..optimizer import Optimizer
from .curiosity import CuriosityPPO, _RunningMeanStd  # noqa: F401  (_RunningMeanStd: ICM-PPO's statistics, importable here)


class ICM_PPO(CuriosityPPO):
    _GRAPH_INPUTS = CuriosityPPO._GRAPH_INPUTS + ("icm_next",)     # icm_next: the next-state rows the ICM reads
    FAMILY = "ICM-PPO"
    NETWORKS = {"icm_mlp": "mlp", "icm_cnn": "cnn"}
    KEY = "icm"

    def __init__(self, state_size, action_size, optim_config={"name": "adam"}, icm_network="icm_mlp", beta=0.2, lamb=1.0,
                 eta=0.01, extrinsic_coeff=1.0, intrinsic_coeff=1.0, obs_normalize=True, ri_normalize=True,
                 batch_norm=True, **kwargs):
        super().__init__(state_size, action_size, icm_network, optim_config, extrinsic_coeff, intrinsic_coeff,
                         obs_normalize, ri_normalize, batch_norm, **kwargs)
        self.beta, self.lamb, self.eta = float(beta), float(lamb), float(eta)
        cnn = icm_network == "icm_cnn"
        self.icm = ICM_MLP(state_size if cnn else int(np.prod(state_size)), action_size, self.action_type,
                           batch_norm=self.batch_norm, device=self.device, seed=self.seed, cnn=cnn)
        self.icm_optimizer = Optimizer(**dict(optim_config), params=self.icm.parameters())
        self._icm_acc = torch.zeros(4, dtype=torch.float32, device=self.device)

    # ----------------------------------------------------------------------------------- learn --
    def _gae_reward(self, st, reward, next_state, N, T):
        NT = N * T
        next_state = st["icm_next"] = self._next_rows(next_state, NT)
        s_ = stream_ptr()
        icm = self.icm
        self._update_rms_obs(icm, next_state, NT)
        chunk = icm.head.max_rows if icm.head is not None else None     # conv1's im2col is 400 KB a row
        f, phi_next, _ = icm.forward(st["state"], next_state, st["action"], None, NT, rms=self._rms(), inverse=False,
                                     tag="pre.", chunk_rows=chunk)
        ri = icm._buf("pre.ri", (NT,))
        C.jb_icm_loss(int(self.continuous), ptr(f), ptr(phi_next), 2 * FEATURE, 0, 0, 0, NT, self.action_size, FEATURE,
                      self.eta, self.beta, ptr(ri), 0, 0, 0, 0, s_)
        return self._filtered_reward(icm, "pre.reward", reward, ri, N, T, self.gamma, self.extrinsic_coeff,
                                     self.intrinsic_coeff)

    def _loss(self, st, idx, B, out, dout, tag):
        super()._loss(st, idx, B, out, dout, tag)
        if self.lamb != 1.0:
            C.jb_scale_f32(ptr(dout), B * self.network.nout, self.lamb, stream_ptr())

    def _after_step(self, st, idx, B, tag):
        icm, s_ = self.icm, stream_ptr()
        itag = tag + "icm."
        f, phi_next, g = icm.forward(st["state"], st["icm_next"], st["action"], idx, B, rms=self._rms(), tag=itag)
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
