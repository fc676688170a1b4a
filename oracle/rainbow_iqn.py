"""Float64 oracle of the Rainbow-IQN agent — TEST INFRASTRUCTURE, never imported by the product.

Rainbow-IQN (Toromanoff et al. 2019, arXiv:1908.04683) restated in torch, given weights, a PER minibatch with its IS
weights, the three fraction sets and the three forwards' noise.  Parity with the upstream JORLDY class is unpinned.

network()          IQN's embedding into Rainbow's noisy dueling streams -> [B, N, A]; noise = [(eps_i, eps_j)] x 4
                   (a1, v1, a2, v2) or None (the mu weights)
targets()          a* = argmax_a mean_j online(s')[b, j, a] (first index on ties),
                   y_j = fold_{s = n-1 .. 0} (r_s + (1 - d_s) gamma y) from y = target(s')[b, j, a*]
loss()             (1/B) sum_b w_b L_b with IQN's per-sample quantile Huber L_b (kappa = 1)
grad_closed()      d loss / d theta_i = -(w_b / (B N')) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -1, 1)
priorities()       L_b^alpha
learn()            one learn(): forward, loss, autograd, one torch.optim.Adam step
"""
import torch
import torch.nn.functional as F

from . import nets
from . import quantile as oq
from .munchausen import _step


def _noisy(p, x, lt, noise):
    return nets.noisy_l(x, p[f"mu_w{lt}"], p[f"sig_w{lt}"], p[f"mu_b{lt}"], p[f"sig_b{lt}"], noise)


def network(p, x, tau, D_em, noise):
    """x [B, ...], tau [B, N] -> [B, N, A]."""
    na1, nv1, na2, nv2 = (None,) * 4 if noise is None else noise
    psi = nets.head(p, x)
    phi = oq.iqn_embed(tau, p["sample_embed.weight"], p["sample_embed.bias"], D_em)
    f = F.relu(F.linear(psi.unsqueeze(1) * phi, p["l.weight"], p["l.bias"]))
    xa = F.relu(_noisy(p, f, "_a1", na1))
    xv = F.relu(_noisy(p, f, "_v1", nv1))
    a = _noisy(p, xa, "_a2", na2)
    v = _noisy(p, xv, "_v2", nv2)
    return v + (a - a.mean(-1, keepdim=True))


def targets(next_online, next_target, reward, done, gamma):
    """next_online [B, N'', A], next_target [B, N', A], reward / done [B, n] -> (a* [B], y [B, N'])."""
    B = next_target.shape[0]
    a_star = next_online.mean(1).argmax(1)
    y = next_target[torch.arange(B), :, a_star]
    for s in reversed(range(reward.shape[1])):
        y = reward[:, s:s + 1] + (1 - done[:, s:s + 1]) * gamma * y
    return a_star, y


def loss(theta, y, tau, w):
    """theta [B, N], y [B, N'], tau [B, N], w [B] -> scalar."""
    return (w * oq.per_sample_loss(theta, y, tau)).mean()


def grad_closed(theta, y, tau, w):
    return w.view(-1, 1) * oq.grad_closed(theta, y, tau)


def priorities(theta, y, tau, alpha):
    return oq.per_sample_loss(theta, y, tau) ** alpha


def _x(x):
    return x.to(torch.float64)


def learn(params, target_params, batch, weights, taus, noise, hp, opt_state=None):
    """batch: state, next_state, action [B], reward / done [B, n].  weights [B] (IS).  taus = [tau(s), tau''(s') for the
    online net, tau'(s') for the target net]; noise = three forwards' [(eps_i, eps_j)] x 4 in that order.
    hp: D_em, gamma, alpha (PER exponent), lr."""
    tp = {k: v.to(torch.float64) for k, v in target_params.items()}
    op = {k: v.to(torch.float64) for k, v in params.items()}
    a = batch["action"].view(-1).to(torch.int64)
    B = a.shape[0]
    r, d = batch["reward"].to(torch.float64).view(B, -1), batch["done"].to(torch.float64).view(B, -1)
    s, ns = _x(batch["state"]), _x(batch["next_state"])
    w = weights.to(torch.float64).view(-1)
    tau, tau_online, tau_target = (t.to(torch.float64) for t in taus)
    n0, n1, n2 = noise if noise is not None else (None, None, None)
    with torch.no_grad():
        next_online = network(op, ns, tau_online, hp["D_em"], n1)
        next_target = network(tp, ns, tau_target, hp["D_em"], n2)
        a_star, y = targets(next_online, next_target, r, d, hp["gamma"])

    def loss_fn(p):
        out = network(p, s, tau, hp["D_em"], n0)                                 # [B, N, A]
        theta = out[torch.arange(B), :, a]
        L = loss(theta, y, tau, w)
        td = theta.detach()
        return L, {"y": y, "a_star": a_star, "per_sample": oq.per_sample_loss(td, y, tau),
                   "prio": priorities(td, y, tau, hp["alpha"]),
                   "result": {"loss": L.item(), "max_Q": out.detach().mean(1).max().item(),
                              "max_logit": out.detach().max().item(), "min_logit": out.detach().min().item()}}

    return _step(params, hp["lr"], opt_state, loss_fn)
