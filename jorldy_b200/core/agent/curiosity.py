"""What the curiosity agents on the PPO rollout path (ICM-PPO, RND-PPO) share: the settings checks, the running
statistics, the BatchNorm minibatch-size rule, the reward-forward filter, the curiosity network's Adam and accumulator,
and the checkpoint layout of their two Adams."""
import os

import numpy as np
import torch

from ..dev import C, ptr, stream_ptr
from .base import cpu_state_dict, load_two_adam_state, two_adam_state
from .ppo import PPO


class _RunningMeanStd:
    """OpenAI baselines' RunningMeanStd on the device: float64 mean / var, count starting at 1e-4."""

    def __init__(self, shape, device):
        self.mean = torch.zeros(shape, dtype=torch.float64, device=device)
        self.var = torch.ones(shape, dtype=torch.float64, device=device)
        self.count = torch.full((1,), 1e-4, dtype=torch.float64, device=device)

    def tensors(self):
        return [self.mean, self.var, self.count]


class CuriosityPPO(PPO):
    """PPO whose reward gains an intrinsic term from a curiosity network trained next to the policy.  A subclass sets
    NETWORKS and KEY, and after this constructor its curiosity network `<KEY>`, that network's optimiser
    `<KEY>_optimizer` and the accumulator `_<KEY>_acc` its minibatch loss adds to."""
    replicas_only = True          # parallel.attach: BatchNorm batch statistics and the running statistics are per replica
    needs_next_state = True       # RolloutCollector: keep every step's next state in the rollout
    NETWORKS = {}                 # curiosity network -> the policy head (observation kind) it pairs with
    KEY = ""                      # "icm" / "rnd": the network's argument prefix, attribute name and checkpoint key

    def __init__(self, state_size, action_size, curiosity_network, optim_config, extrinsic_coeff, intrinsic_coeff,
                 obs_normalize, ri_normalize, batch_norm, **kwargs):
        arg = f"{self.KEY}_network"
        if curiosity_network not in self.NETWORKS:
            raise ValueError(f"{self.FAMILY}: unknown {arg}={curiosity_network!r} (available: {', '.join(self.NETWORKS)})")
        head = kwargs.get("head", "mlp")
        if self.NETWORKS[curiosity_network] != head:
            raise ValueError(f"{self.FAMILY}: {arg}={curiosity_network!r} takes the observations of head="
                             f"{self.NETWORKS[curiosity_network]!r}, got head={head!r}")
        if self.NETWORKS[curiosity_network] == "cnn" and obs_normalize:
            raise ValueError(f"{self.FAMILY}: {curiosity_network} needs obs_normalize=False; per-pixel observation "
                             "normalisation of frames is not implemented")
        kwargs["use_fused"] = False       # the persistent kernel computes PPO's loss only
        super().__init__(state_size, action_size, optim_config=optim_config, **kwargs)
        self.extrinsic_coeff, self.intrinsic_coeff = float(extrinsic_coeff), float(intrinsic_coeff)
        self.obs_normalize, self.ri_normalize, self.batch_norm = bool(obs_normalize), bool(ri_normalize), bool(batch_norm)
        D = int(np.prod(state_size))
        self.rms_obs = _RunningMeanStd((D,), self.device) if self.obs_normalize else None
        self.rms_ri = _RunningMeanStd((1,), self.device)
        self.rewems = None                # [N] reward-forward filter state, created at the first learn

    def _curiosity(self):
        """The curiosity network, its optimiser and its accumulator."""
        return getattr(self, self.KEY), getattr(self, f"{self.KEY}_optimizer"), getattr(self, f"_{self.KEY}_acc")

    def _optimizers(self):
        return [self.optimizer, self._curiosity()[1]]

    # ----------------------------------------------------------------------------------- learn --
    def _check_batch(self, NT):
        """A training-mode BatchNorm cannot normalise a one-row minibatch: neither a batch of 1 nor a one-row epoch
        tail."""
        B = self.batch_size
        if self.batch_norm and (B < 2 or NT % B == 1):
            raise ValueError(f"{self.FAMILY} with batch_norm: a minibatch of one row cannot be batch-normalised "
                             f"(batch_size={B}, rollout of {NT} rows); choose batch_size >= 2 with rollout % batch_size != 1")

    def _next_rows(self, next_state, NT):
        """The N*T next-state rows the curiosity network reads, after the checks a learn makes before any launch."""
        self._check_batch(NT)
        if next_state is None:
            raise ValueError(f"{self.FAMILY} needs every step's next state (a rollout with next_state, or host transitions)")
        return next_state

    def _rms(self):
        return (self.rms_obs.mean, self.rms_obs.var) if self.obs_normalize else None

    def _update_rms_obs(self, net, s_next, NT):
        """rms_obs absorbs the rollout's next states (obs_normalize); net (width D_in) holds the workspace."""
        if self.obs_normalize:
            D = net.D_in
            part = net._buf("rms.partials", (C.jb_col_partials_doubles(NT, D),), torch.float64)
            C.jb_rms_update(ptr(s_next), NT, D, *(ptr(t) for t in self.rms_obs.tensors()), ptr(part), stream_ptr())

    def _filtered_reward(self, net, out_tag, reward, ri, N, T, gamma, ext_coef, int_coef):
        """ext_coef * reward + int_coef * r_i into net's buffer out_tag; with ri_normalize, each env's reward-forward
        filter rewems = gamma * rewems + r_i runs over t, rms_ri absorbs the filtered values and r_i is divided by
        sqrt(rms_ri.var) + 1e-7 first."""
        NT = N * T
        if self.rewems is None or self.rewems.shape[0] != N:
            self.rewems = torch.zeros(N, dtype=torch.float32, device=self.device)
        out = net._buf(out_tag, (NT,))
        if self.ri_normalize:
            part = net._buf("ri.partials", (C.jb_col_partials_doubles(NT, 1),), torch.float64)
            C.jb_icm_reward(ptr(reward), ptr(ri), N, T, gamma, 1, ptr(self.rewems),
                            *(ptr(t) for t in self.rms_ri.tensors()), ptr(part), ptr(net._buf("pre.filt", (NT,))),
                            ext_coef, int_coef, ptr(out), stream_ptr())
        else:
            C.jb_icm_reward(ptr(reward), ptr(ri), N, T, gamma, 0, 0, 0, 0, 0, 0, 0, ext_coef, int_coef, ptr(out),
                            stream_ptr())
        return out

    def _step_state(self):
        net, _, acc = self._curiosity()
        return super()._step_state() + [*net.buffer_tensors(), acc]

    def _zero_acc(self):
        super()._zero_acc()
        self._curiosity()[2].zero_()

    # ------------------------------------------------------------------------------ checkpoint --
    # network / <KEY> / optimizer, the optimizer one torch-Adam layout over network.parameters() + the curiosity
    # network's trained parameters.  The running statistics are not checkpointed (the references do not save them).
    def save(self, path):
        print(f"...Save model to {path}...")
        net, opt, _ = self._curiosity()
        ck = {"network": cpu_state_dict(self.network), self.KEY: cpu_state_dict(net),
              "optimizer": two_adam_state(self.optimizer, opt)}
        torch.save(ck, os.path.join(path, "ckpt"))

    def load(self, path):
        print(f"...Load model from {path}...")
        ck = torch.load(os.path.join(path, "ckpt"), map_location="cpu", weights_only=False)
        net, opt, _ = self._curiosity()
        self.network.load_state_dict(ck["network"])
        net.load_state_dict(ck[self.KEY])
        load_two_adam_state(ck["optimizer"], self.optimizer, opt)
