"""Float64 oracle of the Munchausen agents — TEST INFRASTRUCTURE, never imported by the product.

M-DQN and M-IQN (Vieillard, Pietquin, Geist 2020, arXiv:2007.14430) restated in torch, given weights, a minibatch and, for
M-IQN, the three fraction sets.  Parity with the upstream JORLDY classes is unpinned.  q' is the TARGET network's Q;
tau is the entropy temperature, not IQN's fractions.

tau_logpi()      tau logpi(.|s) = (q - m) - tau log sum_b exp((q_b - m)/tau), m = max_b q_b  (log(pi) is never formed)
bonus()          alpha clip(tau logpi(a_t|s), l_0, 0): clipped first, then scaled
soft_value()     sum_a pi'(a) (x(a) - tau logpi'(a|s')), pi' = softmax(q'(s', .)/tau), for x = q'(s', .) or theta'_j(s', .)
mdqn_target()    y = r + bonus + ((1 - d) gamma) soft_value(q'(s', .))
miqn_targets()   y_j = r + bonus + ((1 - d) gamma) soft_value(theta'_j(s', .)), q' = the per-action quantile means
mdqn_learn() / miqn_learn()   one learn(): forward, loss (DQN's smooth_l1 mean / IQN's quantile Huber), autograd, one
                 torch.optim.Adam step
"""
import torch
import torch.nn.functional as F

from . import nets
from . import quantile as oq


def tau_logpi(q, tau):
    """q [..., A] -> tau logpi [..., A], in the stable form."""
    z = q - q.max(-1, keepdim=True).values
    return z - tau * torch.logsumexp(z / tau, -1, keepdim=True)


def bonus(q_s, action, alpha, tau, l_0):
    """q_s [B, A] = q'(s, .), action [B] -> [B]."""
    t = tau_logpi(q_s, tau).gather(1, action.view(-1, 1).long()).view(-1)
    return alpha * t.clamp(min=l_0, max=0.0)


def soft_value(q_next, x, tau):
    """q_next [B, A] = q'(s', .); x [B, A] or [B, A, N'] -> [B] or [B, N']."""
    pi = torch.softmax(q_next / tau, -1)
    tl = tau_logpi(q_next, tau)
    if x.dim() == 3:
        pi, tl = pi.unsqueeze(-1), tl.unsqueeze(-1)
    return (pi * (x - tl)).sum(1)


def mdqn_target(qt_s, qt_next, action, reward, done, gamma, alpha, tau, l_0):
    """[B, A] target-network Q on s and s' -> y [B]."""
    return reward + bonus(qt_s, action, alpha, tau, l_0) + (1 - done) * gamma * soft_value(qt_next, qt_next, tau)


def miqn_targets(theta_cur, theta_next, action, reward, done, gamma, alpha, tau, l_0):
    """theta_cur [B, A, Nc] and theta_next [B, A, N'] target-network quantiles on s and s' -> y [B, N']."""
    b = bonus(theta_cur.mean(2), action, alpha, tau, l_0)
    v = soft_value(theta_next.mean(2), theta_next, tau)
    return (reward + b).view(-1, 1) + ((1 - done) * gamma).view(-1, 1) * v


def _x(x):
    return x.to(torch.float64)


def _batch(batch):
    a = batch["action"].view(-1).to(torch.int64)
    return a, batch["reward"].to(torch.float64).view(-1), batch["done"].to(torch.float64).view(-1)


def _step(params, lr, opt_state, loss_fn):
    p = {k: v.detach().to(torch.float64).clone().requires_grad_(True) for k, v in params.items()}
    opt = torch.optim.Adam(list(p.values()), lr=lr)
    if opt_state is not None:
        opt.load_state_dict(opt_state)
    L, extra = loss_fn(p)
    opt.zero_grad(set_to_none=True)
    L.backward()
    grads = {k: (v.grad.clone() if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    opt.step()
    return dict(extra, params={k: v.detach().clone() for k, v in p.items()}, grads=grads, opt_state=opt.state_dict())


def mdqn_learn(params, target_params, batch, hp, opt_state=None):
    """hp: gamma, lr, alpha, tau, l_0.  batch: state, next_state, action [B], reward [B], done [B]."""
    tp = {k: v.to(torch.float64) for k, v in target_params.items()}
    a, r, d = _batch(batch)
    s, ns = _x(batch["state"]), _x(batch["next_state"])
    with torch.no_grad():
        y = mdqn_target(nets.discrete_q_network(tp, s), nets.discrete_q_network(tp, ns), a, r, d, hp["gamma"],
                        hp["alpha"], hp["tau"], hp["l_0"])

    def loss_fn(p):
        q = nets.discrete_q_network(p, s).gather(1, a.view(-1, 1)).view(-1)
        L = F.smooth_l1_loss(q, y)
        return L, {"y": y, "result": {"loss": L.item(), "max_Q": q.max().item()}}

    return _step(params, hp["lr"], opt_state, loss_fn)


def miqn_learn(params, target_params, batch, tau, tau_next, tau_cur, hp, opt_state=None):
    """tau, tau_next, tau_cur: fractions [B, N], [B, N'], [B, Nc] of the online pass on s, the target pass on s' and the
    target pass on s.  hp: D_em, gamma, lr, alpha, tau, l_0 (tau here is the entropy temperature)."""
    tp = {k: v.to(torch.float64) for k, v in target_params.items()}
    a, r, d = _batch(batch)
    s, ns = _x(batch["state"]), _x(batch["next_state"])
    tau, tau_next, tau_cur = (t.to(torch.float64) for t in (tau, tau_next, tau_cur))
    with torch.no_grad():
        theta_next = oq.iqn_network(tp, ns, tau_next, hp["D_em"]).transpose(1, 2)
        theta_cur = oq.iqn_network(tp, s, tau_cur, hp["D_em"]).transpose(1, 2)
        y = miqn_targets(theta_cur, theta_next, a, r, d, hp["gamma"], hp["alpha"], hp["tau"], hp["l_0"])

    def loss_fn(p):
        all_theta = oq.iqn_network(p, s, tau, hp["D_em"]).transpose(1, 2)          # [B, A, N]
        theta = all_theta[torch.arange(a.shape[0]), a]
        L = oq.loss(theta, y, tau)
        return L, {"y": y, "per_sample": oq.per_sample_loss(theta.detach(), y, tau),
                   "result": {"loss": L.item(), "max_Q": all_theta.detach().mean(2).max().item()}}

    return _step(params, hp["lr"], opt_state, loss_fn)
