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
from .base import cpu_optimizer_state, cpu_state_dict
from .ddpg import _Scalar
from .ppo import PPO

MULTIPLIERS = ("eta", "alpha_mu", "alpha_sigma")


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
    def _minibatch_step(self, st, idx, B):
        net = self.network
        tag = f"mb{B}."
        out = net.forward_raw(st["state"], idx, B, tag=tag)
        dout = net._buf(tag + "dout", (B, net.nout))
        stats = net._buf(tag + "vstats", (16 + 4 * ((B + 255) // 256),))
        C.jb_vmpo_loss(int(self.continuous), ptr(out), ptr(st["out"]), ptr(idx), ptr(st["action"]), ptr(st["adv"]),
                       ptr(st["ret"]), B, self.action_size, net.nout, ptr(self.mult.flat), self.eps_eta,
                       self.eps_alpha_mu, self.eps_alpha_sigma, ptr(dout), ptr(self.mult.grad), ptr(stats),
                       ptr(self._acc), stream_ptr())
        net.backward_raw(dout, B, tag=tag)
        self.optimizer.step(max_norm=self.clip_grad_norm)
        self.mult_optimizer.step()
        C.jb_vmpo_clamp(ptr(self.mult.flat), self.min_eta, self.min_alpha_mu, self.min_alpha_sigma, stream_ptr())

    def _step_state(self):
        return super()._step_state() + [self.mult.flat, *self.mult_optimizer.state_tensors()]

    def _begin_epochs(self):
        self.optimizer._sync_lr()
        self.mult_optimizer._sync_lr()
        self._acc.zero_()

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

    def learning_rate_decay(self, step, optimizers=None, mode="cosine"):
        super().learning_rate_decay(step, [self.optimizer, self.mult_optimizer] if optimizers is None else optimizers, mode)

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


# One torch-Adam layout over network.parameters() + [eta, alpha_mu, alpha_sigma]: the multipliers are the three parameter
# indices after the network's, each a 0-d tensor; their values are stored under their own names too.  V-MPO's and MPO's
# checkpoints share it.
def joint_optimizer_state(optimizer, mult_optimizer):
    sd = cpu_optimizer_state(optimizer)
    P = len(optimizer.network.p)
    step = float(mult_optimizer._step_dev.item())
    if step > 0:
        m, v = mult_optimizer.exp_avg[:3].cpu(), mult_optimizer.exp_avg_sq[:3].cpu()
        for k in range(3):
            sd["state"][P + k] = {"step": torch.tensor(step), "exp_avg": m[k].clone(), "exp_avg_sq": v[k].clone()}
    sd["param_groups"][0]["params"] = list(range(P + 3))
    return sd


def multiplier_values(mult):
    vals = mult.flat[:3].cpu()
    return {name: vals[k].clone() for k, name in enumerate(MULTIPLIERS)}


def load_joint_optimizer_state(sd, optimizer, mult_optimizer):
    P = len(optimizer.network.p)
    st = sd.get("state", {})
    get = lambda i: st[i] if i in st else st.get(str(i))
    group = dict(sd["param_groups"][0], params=list(range(P)))
    optimizer.load_state_dict({"state": {i: get(i) for i in range(P)} if st else {}, "param_groups": [group]})
    mult_optimizer.param_groups[0]["lr"] = float(group["lr"])
    if get(P) is not None:
        for k in range(3):
            e = get(P + k)
            mult_optimizer.exp_avg[k].copy_(torch.as_tensor(e["exp_avg"]).reshape(()))
            mult_optimizer.exp_avg_sq[k].copy_(torch.as_tensor(e["exp_avg_sq"]).reshape(()))
        mult_optimizer._step_dev.fill_(int(float(get(P)["step"])))


def load_multipliers(ck, mult):
    for k, name in enumerate(MULTIPLIERS):
        if name in ck:
            mult.flat[k].copy_(torch.as_tensor(ck[name], dtype=torch.float32).reshape(()))
