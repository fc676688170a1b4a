"""What the curiosity agents on the PPO rollout path (ICM-PPO, RND-PPO) share: the running statistics, the BatchNorm
minibatch-size rule and the checkpoint layout of their two Adams."""
import torch

from .base import cpu_optimizer_state


class _RunningMeanStd:
    """OpenAI baselines' RunningMeanStd on the device: float64 mean / var, count starting at 1e-4."""

    def __init__(self, shape, device):
        self.mean = torch.zeros(shape, dtype=torch.float64, device=device)
        self.var = torch.ones(shape, dtype=torch.float64, device=device)
        self.count = torch.full((1,), 1e-4, dtype=torch.float64, device=device)

    def tensors(self):
        return [self.mean, self.var, self.count]


def check_batch_norm_rows(family, batch_norm, B, NT):
    """A training-mode BatchNorm cannot normalise a one-row minibatch: neither a batch of 1 nor a one-row epoch tail."""
    if batch_norm and (B < 2 or NT % B == 1):
        raise ValueError(f"{family} with batch_norm: a minibatch of one row cannot be batch-normalised "
                         f"(batch_size={B}, rollout of {NT} rows); choose batch_size >= 2 with rollout % batch_size != 1")


# Adam is per element and the two parameter sets are disjoint, so the policy network's Adam and the curiosity network's
# Adam are one torch Adam over network.parameters() + the curiosity network's parameters: the checkpoint stores that one
# layout, the second optimiser's entries at the parameter indices after the network's.
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
