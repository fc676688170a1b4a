"""Float64 oracle of the quantile-regression agents — TEST INFRASTRUCTURE, never imported by the product.

QR-DQN (Dabney et al. 2017, arXiv:1710.10044) and IQN (Dabney et al. 2018, arXiv:1806.06923) restated in torch,
given weights, a minibatch and the fractions tau.  Parity with the upstream JORLDY classes is unpinned.

loss()            (1/B) sum_b (1/N') sum_j sum_i |tau_i - 1{u_ij < 0}| smooth_l1(u_ij), u_ij = y_j - theta_i (kappa = 1)
grad_closed()     d loss / d theta_i = -(1/(B N')) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -1, 1)
targets()         a* = argmax_a mean_j theta'_j(s', a) (first index on ties), y_j = r + (1 - d) gamma theta'_j(s', a*)
qr_network()      discrete_q_network viewed as [B, A, K];  qr_tau(K) = (2i + 1) / (2K)
iqn_network()     q(relu(l(head(x) * relu(sample_embed(cos(pi i tau)))))) -> [B, N, A]
qrdqn_learn() / iqn_learn()   one learn(): forward, loss, autograd, one torch.optim.Adam step
"""
import math

import torch
import torch.nn.functional as F

from . import nets


def qr_tau(K):
    return (2 * torch.arange(K, dtype=torch.float64) + 1) / (2 * K)


def qr_network(p, x, A, K):
    return nets.discrete_q_network(p, x).view(x.shape[0], A, K)


def iqn_embed(tau, W, b, D_em):
    """tau [B, N] -> phi [B, N, Dh] = relu(cos(pi i tau) W^T + b)."""
    i = torch.arange(D_em, dtype=torch.float64)
    c = torch.cos(math.pi * i * tau.to(torch.float64).unsqueeze(-1))
    return F.relu(F.linear(c, W, b))


def iqn_network(p, x, tau, D_em):
    """x [B, ...], tau [B, N] -> [B, N, A]."""
    psi = nets.head(p, x)
    z = psi.unsqueeze(1) * iqn_embed(tau, p["sample_embed.weight"], p["sample_embed.bias"], D_em)
    h = F.relu(F.linear(z, p["l.weight"], p["l.bias"]))
    return F.linear(h, p["q.weight"], p["q.bias"])


def loss(theta, y, tau):
    """theta [B, N], y [B, N'], tau [B, N] or [N] -> scalar."""
    tau = tau.expand_as(theta)
    u = y.unsqueeze(1) - theta.unsqueeze(2)                                  # [B, N, N']
    huber = F.smooth_l1_loss(y.unsqueeze(1).expand_as(u), theta.unsqueeze(2).expand_as(u), reduction="none")
    t = tau.unsqueeze(2)
    rho = torch.where(u < 0, (1 - t) * huber, t * huber)
    return rho.sum(1).mean(1).mean(0)


def per_sample_loss(theta, y, tau):
    tau = tau.expand_as(theta)
    u = y.unsqueeze(1) - theta.unsqueeze(2)
    huber = torch.where(u.abs() < 1, 0.5 * u * u, u.abs() - 0.5)
    t = tau.unsqueeze(2)
    return torch.where(u < 0, 1 - t, t).mul(huber).sum(1).mean(1)


def grad_closed(theta, y, tau):
    B, Np = y.shape
    tau = tau.expand_as(theta)
    u = y.unsqueeze(1) - theta.unsqueeze(2)
    t = tau.unsqueeze(2)
    return -(torch.where(u < 0, 1 - t, t) * u.clamp(-1, 1)).sum(2) / (B * Np)


def targets(theta_next, reward, done, gamma):
    """theta_next [B, A, N'] -> (a* [B], y [B, N'])."""
    B = theta_next.shape[0]
    a_star = theta_next.mean(2).argmax(1)
    sel = theta_next[torch.arange(B), a_star]
    return a_star, reward.view(B, 1) + (1 - done.view(B, 1)) * gamma * sel


def _x(x):
    return x.to(torch.float64)


def _learn(params, theta_fn, theta_next, batch, tau, lr, opt_state, gamma):
    p = {k: v.detach().to(torch.float64).clone().requires_grad_(True) for k, v in params.items()}
    opt = torch.optim.Adam(list(p.values()), lr=lr)
    if opt_state is not None:
        opt.load_state_dict(opt_state)
    a = batch["action"].view(-1).to(torch.int64)
    B = a.shape[0]
    r, d = batch["reward"].to(torch.float64).view(-1), batch["done"].to(torch.float64).view(-1)
    with torch.no_grad():
        a_star, y = targets(theta_next, r, d, gamma)
    all_theta = theta_fn(p)                                                 # [B, A, N]
    theta = all_theta[torch.arange(B), a]
    L = loss(theta, y, tau)
    opt.zero_grad(set_to_none=True)
    L.backward()
    grads = {k: (v.grad.clone() if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    opt.step()
    return {"params": {k: v.detach().clone() for k, v in p.items()}, "grads": grads, "a_star": a_star,
            "per_sample": per_sample_loss(theta.detach(), y, tau), "opt_state": opt.state_dict(),
            "result": {"loss": L.item(), "max_Q": all_theta.detach().mean(2).max().item()}}


def qrdqn_learn(params, target_params, batch, hp, opt_state=None):
    """hp: A, K, gamma, lr.  batch: state, next_state, action [B], reward [B], done [B]."""
    A, K = hp["A"], hp["K"]
    tp = {k: v.to(torch.float64) for k, v in target_params.items()}
    with torch.no_grad():
        theta_next = qr_network(tp, _x(batch["next_state"]), A, K)
    return _learn(params, lambda p: qr_network(p, _x(batch["state"]), A, K), theta_next, batch, qr_tau(K), hp["lr"],
                  opt_state, hp["gamma"])


def iqn_learn(params, target_params, batch, tau, tau_next, hp, opt_state=None):
    """tau, tau_next [B, N] for the online pass on s and the target pass on s'.  hp: D_em, gamma, lr."""
    tp = {k: v.to(torch.float64) for k, v in target_params.items()}
    tau, tau_next = tau.to(torch.float64), tau_next.to(torch.float64)
    with torch.no_grad():
        theta_next = iqn_network(tp, _x(batch["next_state"]), tau_next, hp["D_em"]).transpose(1, 2)
    return _learn(params, lambda p: iqn_network(p, _x(batch["state"]), tau, hp["D_em"]).transpose(1, 2), theta_next,
                  batch, tau, hp["lr"], opt_state, hp["gamma"])


def qrdqn_q(params, x, A, K):
    p = {k: v.to(torch.float64) for k, v in params.items()}
    return qr_network(p, _x(x), A, K).mean(2)


def iqn_q(params, x, tau, D_em):
    p = {k: v.to(torch.float64) for k, v in params.items()}
    return iqn_network(p, _x(x), tau.to(torch.float64), D_em).mean(1)
