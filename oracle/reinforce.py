"""Float64 oracle of REINFORCE — TEST INFRASTRUCTURE, never imported by the product.

Written literally after the reference's jorldy/core/agent/reinforce.py learn():
  ret = reward copied; for t in reversed(range(len(ret) - 1)): ret[t] += gamma * ret[t + 1]
  use_standardization: ret = (ret - ret.mean()) / (ret.std() + 1e-7)               (numpy, ddof = 0)
  discrete:   loss = -(log(pi.gather(1, a)) * ret).mean()
  continuous: loss = -(Normal(mu, std).log_prob(atanh(clamp(a, +-(1 - 1e-7)))) * ret).mean()   (over M*A elements)
  one optimiser step, no gradient clipping

reference_returns()   the reference's loop and numpy standardisation on one episode
ring_rows()           the batched mapping: every completed episode of every env row of an episode ring -> the compact
                      env-major, oldest-first (idx, ret) list, the counts and the new heads
loss()                the reference expression through torch autograd
closed_form()         the gradient w.r.t. the head outputs as the kernel computes it
learn()               one whole learn (network, loss, float64 Adam) on the rows
"""
import numpy as np
import torch
import torch.nn.functional as F
from torch.distributions import Normal

from . import nets


def reference_returns(reward, gamma, standardize):
    ret = np.array(reward, dtype=np.float64).copy()
    for t in reversed(range(len(ret) - 1)):
        ret[t] += gamma * ret[t + 1]
    if standardize:
        ret = (ret - ret.mean()) / (ret.std() + 1e-7)
    return ret


def ring_rows(reward, done, pos, head, gamma, standardize):
    """reward, done [N, L]; pos: steps written; head [N] absolute -> (idx int64 [M], ret f64 [M], count [N], new head)."""
    reward, done = np.asarray(reward, np.float64), np.asarray(done)
    N, L = reward.shape
    idx, ret, count, new_head = [], [], np.zeros(N, np.int64), np.array(head, np.int64).copy()
    for e in range(N):
        steps = list(range(int(head[e]), int(pos)))
        dones = [t for t in steps if done[e, t % L] != 0]
        if not dones:
            continue
        start = int(head[e])
        for end in dones:                                  # episodes oldest first
            ts = list(range(start, end + 1))
            idx += [e * L + t % L for t in ts]
            ret += list(reference_returns([reward[e, t % L] for t in ts], gamma, standardize))
            start = end + 1
        count[e] = dones[-1] + 1 - int(head[e])
        new_head[e] = dones[-1] + 1
    return np.array(idx, np.int64), np.array(ret, np.float64), count, new_head


def _z(action):
    """atanh(clamp(a, +-(1 - 1e-7))) with the clamp on float32 actions, as the reference applies it to its float32
    action tensor (the bound rounds to 1 - 2^-23)."""
    return torch.atanh(torch.clamp(action.to(torch.float32), min=-1 + 1e-7, max=1 - 1e-7).to(torch.float64))


def _head_terms(out, action, A, continuous):
    out = out.to(torch.float64)
    if continuous:
        mu = torch.clamp(out[:, :A], min=-5.0, max=5.0)
        std = torch.tanh(out[:, A:2 * A]).exp()
        z = _z(action)
        return Normal(mu, std).log_prob(z)                 # [M, A]
    pi = F.softmax(out[:, :A], dim=-1)
    return torch.log(pi.gather(1, action.view(-1, 1).long()))      # [M, 1]


def loss(out, action, ret, A, continuous):
    """The reference loss of head outputs out [M, nout] (a leaf or not) with actions and returns [M]."""
    lp = _head_terms(out, action, A, continuous)
    return -(lp * ret.to(torch.float64).view(-1, 1)).mean()


def closed_form(out, action, ret, A, continuous):
    """d loss / d out [M, nout], as jb_reinforce_loss forms it."""
    out, ret = out.to(torch.float64), ret.to(torch.float64)
    M = out.shape[0]
    if continuous:
        raw_mu, raw_ls = out[:, :A], out[:, A:2 * A]
        mu = raw_mu.clamp(-5.0, 5.0)
        ls = torch.tanh(raw_ls)
        sd = ls.exp()
        z = _z(action)
        coef = -(ret / (M * A)).view(-1, 1)
        d = z - mu
        in_mu = ((raw_mu >= -5.0) & (raw_mu <= 5.0)).to(torch.float64)
        dmu = coef * d / sd ** 2 * in_mu
        dls = coef * (d * d / sd ** 3 - 1 / sd) * sd * (1 - ls * ls)
        return torch.cat([dmu, dls], dim=1)
    p = F.softmax(out[:, :A], dim=-1)
    onehot = F.one_hot(action.view(-1).long(), A).to(torch.float64)
    return -(ret / M).view(-1, 1) * (onehot - p)


def policy_out(p, x, continuous):
    """discrete_policy / continuous_policy head outputs before their activations: logits or [mu_raw | log_std_raw]."""
    h = F.relu(F.linear(nets.head(p, x), p["l.weight"], p["l.bias"]))
    if continuous:
        return torch.cat([F.linear(h, p["mu.weight"], p["mu.bias"]), F.linear(h, p["log_std.weight"], p["log_std.bias"])], 1)
    return F.linear(h, p["pi.weight"], p["pi.bias"])


def learn(params, state, action, ret, A, continuous, lr, betas=(0.9, 0.999), eps=1e-8, state_m=None, state_v=None, step=0):
    """One learn on the rows (state [M, D], action, ret [M]) in float64: the loss through autograd and one Adam step.
    Returns {"loss", "params", "exp_avg", "exp_avg_sq", "grads"}."""
    p = {k: v.detach().to(torch.float64).clone().requires_grad_(True) for k, v in params.items()}
    L = loss(policy_out(p, state.to(torch.float64), continuous), action, ret, A, continuous)
    L.backward()
    t = step + 1
    b1, b2 = betas
    new, m_out, v_out, grads = {}, {}, {}, {}
    for k, v in p.items():
        g = v.grad if v.grad is not None else torch.zeros_like(v)
        m = (state_m[k].to(torch.float64) if state_m else torch.zeros_like(g)) * b1 + (1 - b1) * g
        s = (state_v[k].to(torch.float64) if state_v else torch.zeros_like(g)) * b2 + (1 - b2) * g * g
        mhat, vhat = m / (1 - b1 ** t), s / (1 - b2 ** t)
        new[k] = v.detach() - lr * mhat / (vhat.sqrt() + eps)
        m_out[k], v_out[k], grads[k] = m, s, g.detach()
    return {"loss": float(L.item()), "params": new, "exp_avg": m_out, "exp_avg_sq": v_out, "grads": grads}
