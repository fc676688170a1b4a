"""Agent contract (jorldy/core/agent/base.py:6-111): act / learn / process / save / load /
sync_in / sync_out / set_distributed / interact_callback / learning_rate_decay."""
import os
from abc import ABC, abstractmethod

import numpy as np
import torch

from ..dev import f32


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
            optimizers = [self.optimizer]
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
