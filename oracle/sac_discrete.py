"""Float64 oracle of the discrete-action SAC — TEST INFRASTRUCTURE, never imported by the product.

A torch restatement of SAC-Discrete (Christodoulou 2019, arXiv:1910.07207) with the bookkeeping of the project's
continuous SAC (oracle/actor_critic.py sac_learn): one learn() steps critic1, critic2, the actor (through the UPDATED
critics) and, with a dynamic temperature, log_alpha; the alpha used inside a learn() is the one carried in, and the
alpha handed out is exp(log_alpha) from before this learn's step.  Notation: logpi = log_softmax(z), pi = exp(logpi).

discrete_policy()   head -> l -> pi logits
target()            y = r + (1 - d) gamma sum_a pi'(a) [min(Q1', Q2')(s', a) - alpha logpi'(a)]
critic_closed()     L_i = mean (Q_i(s)[a] - y)^2 and dQ_i = 2 (q_i - y) / B at the taken action
actor_closed()      dz = pi (f - L_b) / B with f = alpha logpi - min(Q1, Q2), L_b = sum_a pi f, and the four stats
act()               inverse CDF of pi on uniforms (first index whose running sum exceeds u * sum pi), greedy argmax
learn()             the whole update with autograd and torch.optim.Adam
"""
import math

import torch
import torch.nn.functional as F

from . import nets


def target_entropy(A):
    return 0.98 * math.log(A)


def discrete_policy(p, x):
    h = F.relu(F.linear(nets.head(p, x), p["l.weight"], p["l.bias"]))
    return F.linear(h, p["pi.weight"], p["pi.bias"])


def _x(x):
    return x.to(torch.float64)


def target(nz, nq1, nq2, reward, done, gamma, alpha):
    """nz, nq_i [B, A]; reward, done [B] -> y [B]."""
    lp = F.log_softmax(nz, dim=-1)
    v = (lp.exp() * (torch.minimum(nq1, nq2) - alpha * lp)).sum(-1)
    return reward + (1 - done) * gamma * v


def critic_closed(q1, q2, action, y):
    """q_i [B, A], action int64 [B] -> (loss1, loss2, dq1, dq2)."""
    B = q1.shape[0]
    out = []
    for q in (q1, q2):
        e = q.gather(1, action.view(B, 1)).view(B) - y
        dq = torch.zeros_like(q)
        dq.scatter_(1, action.view(B, 1), (2 * e / B).view(B, 1))
        out.append(((e * e).mean(), dq))
    return out[0][0], out[1][0], out[0][1], out[1][1]


def actor_closed(z, q1, q2, alpha, A_target_entropy):
    """z, q_i [B, A] -> (dz, stats): stats = {actor_loss, mean_Q, entropy, entropy - target_entropy}."""
    B = z.shape[0]
    lp = F.log_softmax(z, dim=-1)
    pi = lp.exp()
    m = torch.minimum(q1, q2)
    f = alpha * lp - m
    L = (pi * f).sum(-1)
    H = -(pi * lp).sum(-1)
    dz = pi * (f - L.view(B, 1)) / B
    return dz, {"actor_loss": L.mean().item(), "mean_Q": (pi * m).sum(-1).mean().item(), "entropy": H.mean().item(),
                "entropy_gap": H.mean().item() - A_target_entropy}


def actor_loss(z, q1, q2, alpha):
    """The actor objective as autograd sees it (for checking actor_closed's dz)."""
    lp = F.log_softmax(z, dim=-1)
    return (lp.exp() * (alpha * lp - torch.minimum(q1, q2))).sum(-1).mean()


def act(z, u=None):
    """Inverse CDF of pi = softmax(z) on u [M] (first k with u * sum(pi) < cumsum(pi)_k; the last action if none), or
    argmax pi (first index on ties) when u is None."""
    pi = F.log_softmax(z.to(torch.float64), dim=-1).exp()
    if u is None:
        return pi.argmax(-1)
    c = pi.cumsum(-1)
    t = u.to(torch.float64).view(-1, 1) * pi.sum(-1, keepdim=True)
    hit = t < c
    return torch.where(hit.any(-1), hit.to(torch.int64).argmax(-1), torch.full_like(hit[:, 0], z.shape[1] - 1, dtype=torch.int64))


def _leaf(params):
    return {k: v.detach().to(torch.float64).clone().requires_grad_(True) for k, v in params.items()}


def _adam(p, lr, state):
    opt = torch.optim.Adam(list(p.values()), lr=lr)
    if state is not None:
        opt.load_state_dict(state)
    return opt


def _step(opt, loss, p):
    opt.zero_grad(set_to_none=True)
    loss.backward()
    grads = {k: (v.grad.clone() if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    opt.step()
    return grads


def _detach(p):
    return {k: v.detach().clone() for k, v in p.items()}


def learn(actor, critic1, critic2, t_critic1, t_critic2, log_alpha, alpha, batch, hp, opt_state=None):
    """One learn() in float64.  hp: gamma, actor_lr, critic_lr, alpha_lr, use_dynamic_alpha, A.  batch: state / next_state
    (float or uint8 stacks), action int64 [B], reward [B], done [B].  `alpha` is the value carried into this learn;
    returns post-step params, gradients, the new (log_alpha, alpha), optimiser states and the result dict."""
    opt_state = opt_state or {}
    a_p, c1_p, c2_p = _leaf(actor), _leaf(critic1), _leaf(critic2)
    tc1, tc2 = ({k: v.to(torch.float64) for k, v in t.items()} for t in (t_critic1, t_critic2))
    la = log_alpha.detach().to(torch.float64).clone().requires_grad_(hp["use_dynamic_alpha"])
    alpha = float(alpha)
    a_opt = _adam(a_p, hp["actor_lr"], opt_state.get("actor"))
    c1_opt, c2_opt = _adam(c1_p, hp["critic_lr"], opt_state.get("critic1")), _adam(c2_p, hp["critic_lr"], opt_state.get("critic2"))
    s, ns = _x(batch["state"]), _x(batch["next_state"])
    a, r, d = batch["action"].view(-1).to(torch.int64), _x(batch["reward"]).view(-1), _x(batch["done"]).view(-1)
    B = a.shape[0]
    with torch.no_grad():
        y = target(discrete_policy(a_p, ns), nets.discrete_q_network(tc1, ns), nets.discrete_q_network(tc2, ns), r, d,
                   hp["gamma"], alpha)
    loss1 = F.mse_loss(nets.discrete_q_network(c1_p, s).gather(1, a.view(B, 1)).view(B), y)
    g1 = _step(c1_opt, loss1, c1_p)
    loss2 = F.mse_loss(nets.discrete_q_network(c2_p, s).gather(1, a.view(B, 1)).view(B), y)
    g2 = _step(c2_opt, loss2, c2_p)
    with torch.no_grad():
        q1n, q2n = nets.discrete_q_network(c1_p, s), nets.discrete_q_network(c2_p, s)
    z = discrete_policy(a_p, s)
    a_loss = actor_loss(z, q1n, q2n, alpha)
    ga = _step(a_opt, a_loss, a_p)
    _, stats = actor_closed(z.detach(), q1n, q2n, alpha, target_entropy(hp["A"]))
    alpha_loss = la * stats["entropy_gap"]
    new_alpha = la.detach().exp()
    st = {"actor": a_opt.state_dict(), "critic1": c1_opt.state_dict(), "critic2": c2_opt.state_dict()}
    if hp["use_dynamic_alpha"]:
        al_opt = _adam({"log_alpha": la}, hp["alpha_lr"], opt_state.get("alpha"))
        al_opt.zero_grad(set_to_none=True)
        alpha_loss.backward()
        al_opt.step()
        st["alpha"] = al_opt.state_dict()
    return {"actor": _detach(a_p), "critic1": _detach(c1_p), "critic2": _detach(c2_p), "actor_grads": ga,
            "critic1_grads": g1, "critic2_grads": g2, "log_alpha": la.detach().clone(), "alpha": new_alpha.item(),
            "opt_state": st,
            "result": {"critic_loss1": loss1.item(), "critic_loss2": loss2.item(), "actor_loss": stats["actor_loss"],
                       "alpha_loss": alpha_loss.item(), "max_Q": y.max().item(), "mean_Q": stats["mean_Q"],
                       "alpha": new_alpha.item(), "entropy": stats["entropy"]}}


def soft_update(target_p, online, tau):
    return {k: tau * online[k].to(torch.float64) + (1 - tau) * target_p[k].to(torch.float64) for k in target_p}
