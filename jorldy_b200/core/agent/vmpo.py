"""V-MPO agent (Song et al., ICLR 2020, arXiv:1909.12238) on the PPO rollout path.

Everything up to the minibatch loss is PPO's (act, the batched and Atari-frame rollouts, the pre-pass, jb_gae, the
CUDA-graph minibatch loop driven by the device cursor).  One minibatch step here = forward -> jb_vmpo_loss (top-half
advantages, learned temperature eta, KL trust regions with learned multipliers alpha_mu / alpha_sigma, critic MSE;
csrc/vmpo.cu) -> backward -> network clip + Adam -> multiplier Adam -> clamp of the multipliers to their minima.

The three multipliers live in one device vector [eta, alpha_mu, alpha_sigma] with its own flat Adam (same lr, betas
and eps as the network's).  Adam is per element and both step every minibatch, so this equals one torch Adam over
network.parameters() + [eta, alpha_mu, alpha_sigma] with clip_grad_norm_ on the network's parameters only.  The loss
kernel reads the multipliers from device memory, so captured graphs never bake a host value.

Deviation: a minibatch whose advantages all equal their median has an empty top half; its policy and temperature
terms are 0 here instead of the NaN a mean over an empty tensor gives.
"""
import os

import torch

from ..dev import C, ptr, stream_ptr
from ..optimizer import Optimizer
from .base import (_Scalar, cpu_state_dict, joint_optimizer_state, load_joint_optimizer_state, load_multipliers,
                   multiplier_values)
from .ppo import PPO


class VMPO(PPO):
    LAUNCHES_PER_MINIBATCH = 16   # PPO's 13 with the V-MPO loss + finalize, plus the multipliers' sumsq + adam + clamp
    _GRAPH_INPUTS = PPO._GRAPH_INPUTS + ("out",)       # out: the pre-pass head outputs, the old policy of the KL terms
    replicas_only = True          # parallel.attach: the median and psi are per minibatch, an averaged shard gradient is not V-MPO
    FAMILY = "V-MPO"

    def __init__(self, state_size, action_size, optim_config={"name": "adam"}, min_eta=1e-8, min_alpha_mu=1e-8,
                 min_alpha_sigma=1e-8, eps_eta=0.01, eps_alpha_mu=0.01, eps_alpha_sigma=5e-5, eta=1.0, alpha_mu=1.0,
                 alpha_sigma=1.0, **kwargs):
        kwargs["use_fused"] = False       # the persistent kernel computes PPO's loss only
        super().__init__(state_size, action_size, optim_config=optim_config, **kwargs)
        self.min_eta, self.min_alpha_mu, self.min_alpha_sigma = float(min_eta), float(min_alpha_mu), float(min_alpha_sigma)
        self.eps_eta, self.eps_alpha_mu, self.eps_alpha_sigma = float(eps_eta), float(eps_alpha_mu), float(eps_alpha_sigma)
        self.mult = _Scalar("multipliers", [eta, alpha_mu, alpha_sigma], self.device)
        self.mult_optimizer = Optimizer(**dict(optim_config), params=self.mult.parameters())

    # ----------------------------------------------------------------------------------- learn --
    def _optimizers(self):
        return [self.optimizer, self.mult_optimizer]

    def _loss(self, st, idx, B, out, dout, tag):
        stats = self.network._buf(tag + "vstats", (16 + 4 * ((B + 255) // 256),))
        C.jb_vmpo_loss(int(self.continuous), ptr(out), ptr(st["out"]), ptr(idx), ptr(st["action"]), ptr(st["adv"]),
                       ptr(st["ret"]), B, self.action_size, self.network.nout, ptr(self.mult.flat), self.eps_eta,
                       self.eps_alpha_mu, self.eps_alpha_sigma, ptr(dout), ptr(self.mult.grad), ptr(stats),
                       ptr(self._acc), stream_ptr())

    def _after_step(self, st, idx, B, tag):
        self.mult_optimizer.step()
        C.jb_vmpo_clamp(ptr(self.mult.flat), self.min_eta, self.min_alpha_mu, self.min_alpha_sigma, stream_ptr())

    def _zero_acc(self):
        self._acc.zero_()         # all sums from 0: slot 4 counts the minibatches

    def _learn_result(self, mean_ret):
        v = torch.cat([self._acc[:5], mean_ret.view(1), self.mult.flat[:3]]).cpu().numpy()    # ONE device->host read
        cnt = max(v[4], 1.0)
        return {
            "actor_loss": float(v[0] / cnt),
            "critic_loss": float(v[1] / cnt),
            "eta_loss": float(v[2] / cnt),
            "alpha_loss": float(v[3] / cnt),
            "eta": float(v[6]),
            "alpha_mu": float(v[7]),
            "alpha_sigma": float(v[8]),
            "mean_ret": float(v[5]),
        }

    # ------------------------------------------------------------------------------ checkpoint --
    def save(self, path):
        print(f"...Save model to {path}...")
        ck = {"network": cpu_state_dict(self.network), "optimizer": joint_optimizer_state(self.optimizer, self.mult_optimizer)}
        ck.update(multiplier_values(self.mult))
        torch.save(ck, os.path.join(path, "ckpt"))

    def load(self, path):
        print(f"...Load model from {path}...")
        ck = torch.load(os.path.join(path, "ckpt"), map_location="cpu", weights_only=False)
        self.network.load_state_dict(ck["network"])
        load_joint_optimizer_state(ck["optimizer"], self.optimizer, self.mult_optimizer)
        load_multipliers(ck, self.mult)

