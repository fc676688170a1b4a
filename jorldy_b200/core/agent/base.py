"""Agent contract (jorldy/core/agent/base.py:6-111): act / learn / process / save / load /
sync_in / sync_out / set_distributed / interact_callback / learning_rate_decay."""
import os
from abc import ABC, abstractmethod

import numpy as np
import torch

from ..dev import f32
from ..network.base import FlatNetwork

MULTIPLIERS = ("eta", "alpha_mu", "alpha_sigma")       # V-MPO's and MPO's learned multipliers, in their vector's order


def cpu_state_dict(net):
    """A network's state_dict with every tensor copied to the CPU, as checkpoints store it."""
    return {k: v.cpu() for k, v in net.state_dict().items()}


def cpu_optimizer_state(optimizer):
    """An optimizer's state_dict with every state tensor copied to the CPU, as checkpoints store it."""
    sd = optimizer.state_dict()
    for st in sd["state"].values():
        for k, v in st.items():
            if torch.is_tensor(v):
                st[k] = v.cpu()
    return sd


class _Scalar(FlatNetwork):
    """Learnable scalars held like a network so that the flat Adam applies: SAC's log_alpha (sac.py:95-100), or V-MPO's
    [eta, alpha_mu, alpha_sigma] as one contiguous vector when `value` is a sequence."""

    def __init__(self, name, value, device):
        super().__init__(device)
        values = [float(v) for v in np.atleast_1d(value)]
        self._specs = [(name, (len(values),))]
        self._allocate()
        self.flat[:len(values)] = torch.tensor(values, dtype=torch.float32)


# Adam is per element and the two parameter sets are disjoint, so the policy network's Adam and the curiosity network's
# Adam are one torch Adam over network.parameters() + the curiosity network's parameters: the checkpoint stores that one
# layout, the second optimiser's entries at the parameter indices after the network's.  ICM-PPO's and RND-PPO's
# checkpoints share it.
def two_adam_state(optimizer, aux_optimizer):
    sd = cpu_optimizer_state(optimizer)
    asd = cpu_optimizer_state(aux_optimizer)
    P = len(optimizer.network.p)
    for i, e in asd["state"].items():
        sd["state"][P + i] = e
    sd["param_groups"][0]["params"] = list(range(P + len(aux_optimizer.network.p)))
    return sd


def load_two_adam_state(sd, optimizer, aux_optimizer):
    P, Q = len(optimizer.network.p), len(aux_optimizer.network.p)
    st = sd.get("state", {})
    get = lambda i: st[i] if i in st else st.get(str(i))
    group = dict(sd["param_groups"][0])
    optimizer.load_state_dict({"state": {i: get(i) for i in range(P)} if st else {},
                               "param_groups": [dict(group, params=list(range(P)))]})
    aux_optimizer.load_state_dict({"state": {i: get(P + i) for i in range(Q)} if get(P) is not None else {},
                                   "param_groups": [dict(group, params=list(range(Q)))]})


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


class BaseAgent(ABC):
    @abstractmethod
    def act(self, state):
        ...

    @abstractmethod
    def learn(self):
        ...

    @abstractmethod
    def process(self, transitions, step):
        ...

    def _state_to_device(self, state):
        """act()'s input as a tensor: a tensor is used as it is, anything else is copied to the agent's device."""
        return state if isinstance(state, torch.Tensor) else torch.as_tensor(np.asarray(state), device=self.device)

    def _row_counter(self, M):
        """Device int64 [M] per-row Philox draw counters of the act kernels for batches of M rows, created on first use.
        The kernels read and advance them on the device, so CUDA-graph replays draw fresh numbers."""
        ctr = self._row_ctr.get(M)
        if ctr is None:
            ctr = self._row_ctr[M] = torch.zeros(M, dtype=torch.int64, device=self.device)
        return ctr

    def _replay_indices(self, device=None):
        """int64 replay indices of the next learn(): the injected ones if a test set them, else a uniform sample."""
        src = self._inject_idx if self._inject_idx is not None else self.memory.sample_indices(self.batch_size)
        return torch.as_tensor(np.asarray(src), dtype=torch.int64, device=device)

    def as_tensor(self, x):
        if isinstance(x, list):
            return [f32(v, self.device) for v in x]
        return f32(x, self.device)

    def sync_in(self, weights):
        self.network.load_state_dict(weights)

    def sync_out(self, device="cpu"):
        weights = self.network.state_dict()
        for k, v in weights.items():
            weights[k] = v.to(device)
        return {"weights": weights}

    def set_distributed(self, *args, **kwargs):
        return self

    def interact_callback(self, transition):
        return transition

    def _optimizers(self):
        """Every optimiser a learn steps: learning_rate_decay's default list."""
        return [self.optimizer]

    def learning_rate_decay(self, step, optimizers=None, mode="cosine"):
        """lr = lr0 * w(step/run_step) after every learn (base.py:93-111)."""
        frac = step / self.run_step
        if mode == "linear":
            weight = 1 - frac
        elif mode == "cosine":
            weight = np.cos((np.pi / 2) * frac)
        elif mode == "sqrt":
            weight = (1 - frac) ** (1 / 2)
        else:
            raise Exception(f"check learning rate decay mode again! => {mode}")
        if optimizers is None:
            optimizers = self._optimizers()
        if not isinstance(optimizers, list):
            optimizers = [optimizers]
        for optimizer in optimizers:
            for g in optimizer.param_groups:
                g["lr"] = float(optimizer.defaults["lr"] * weight)

    # checkpoint format = the reference's: {"network": state_dict, "optimizer": state_dict} -> path/ckpt
    def save(self, path):
        print(f"...Save model to {path}...")
        torch.save({"network": cpu_state_dict(self.network), "optimizer": cpu_optimizer_state(self.optimizer)},
                   os.path.join(path, "ckpt"))

    def load(self, path):
        print(f"...Load model from {path}...")
        checkpoint = torch.load(os.path.join(path, "ckpt"), map_location="cpu", weights_only=False)
        self.network.load_state_dict(checkpoint["network"])
        if hasattr(self, "target_network"):
            self.target_network.load_state_dict(checkpoint["network"])
        self.optimizer.load_state_dict(checkpoint["optimizer"])
