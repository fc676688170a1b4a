"""Float64 oracle of MuZero on Atari frames — TEST INFRASTRUCTURE, never imported by the product.

The representation input and network of `Agent("muzero", head="cnn")` restated from a parameter dict keyed like the
product's state_dict; dynamics, prediction, the targets and the loss are oracle/muzero.py's.

action_planes()         the 4 action planes' values: a_k / A where stack frame k follows an action in its episode, else 0
frame_action_input()    4 frames / 255 and the 4 constant planes -> the [B, 8, 84, 84] representation input
represent()             conv 8x8s4 -> 4x4s2 -> 3x3s1 (ReLU each) -> flatten -> linear to the latent, min-max scaled
unroll_loss(), learn()  oracle/muzero.py's, with represent() above over batch["state"] = frame_action_input()
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import muzero as om


def action_planes(prev_actions, pos, first, A):
    """prev_actions [B, 4] (the actions that produced stack frames 0..3), pos [B] (the stack's newest frame position),
    first [B] (its episode's first frame position) -> planes [B, 4]: a_k / A where frame k, at pos - 3 + k, comes after
    the episode's first frame, else 0 (the first frame, and its repeats in a short episode's stack, follow no action)."""
    a = torch.as_tensor(np.asarray(prev_actions), dtype=torch.float64)
    k = torch.arange(4, dtype=torch.int64)
    live = (torch.as_tensor(np.asarray(pos)).view(-1, 1) - 3 + k) > torch.as_tensor(np.asarray(first)).view(-1, 1)
    return torch.where(live, a / A, torch.zeros_like(a))


def frame_action_input(stacks, planes):
    """stacks uint8 [B, 4, 84, 84], planes [B, 4] -> the representation input [B, 8, 84, 84] in float64."""
    x = torch.as_tensor(np.asarray(stacks)).to(torch.float64) / 255.0
    pl = torch.as_tensor(planes, dtype=torch.float64).view(-1, 4, 1, 1).expand(-1, -1, *x.shape[2:])
    return torch.cat([x, pl], 1)


def represent(p, x):
    for name, stride in (("conv1", 4), ("conv2", 2), ("conv3", 1)):
        x = F.relu(F.conv2d(x, p[f"head.{name}.weight"], p[f"head.{name}.bias"], stride=stride))
    return om.scale(F.linear(x.flatten(1), p["h.l.weight"], p["h.l.bias"]))


def unroll_loss(p, batch, weights, hp):
    """oracle/muzero.py unroll_loss with the CNN representation; batch["state"] = frame_action_input() [B, 8, 84, 84]."""
    A, K = hp["A"], hp["K"]
    x = torch.as_tensor(np.asarray(batch["state"]), dtype=torch.float64)
    action = torch.as_tensor(np.asarray(batch["action"])).long()
    s = represent(p, x)
    pis, vs, rs = [], [], []
    for k in range(K + 1):
        pi_k, v_k = om.predict(p, s)
        pis.append(pi_k)
        vs.append(v_k)
        if k < K:
            s_in = 0.5 * s + 0.5 * s.detach()          # the pseudocode's scale_gradient(hidden_state, 0.5)
            s, r_k = om.dynamics(p, s_in, action[:, k], A)
            rs.append(r_k)
    return om.loss(torch.stack(pis), torch.stack(vs), torch.stack(rs), batch, weights, hp)


def learn(params, batch, weights, hp, lr, clip):
    """One learn on frames from float64 copies of `params`; returns (new params, stats, priorities, grads)."""
    p = {k: torch.as_tensor(v, dtype=torch.float64).clone().requires_grad_(True) for k, v in params.items()}
    total, stats, prio = unroll_loss(p, batch, weights, hp)
    total.backward()
    grads = {k: v.grad.clone() for k, v in p.items()}
    torch.nn.utils.clip_grad_norm_(list(p.values()), clip)
    opt = torch.optim.Adam(list(p.values()), lr=lr)
    opt.step()
    return {k: v.detach() for k, v in p.items()}, stats, prio, grads
