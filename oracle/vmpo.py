"""Float64 CPU oracle of V-MPO (Song et al., ICLR 2020, arXiv:1909.12238) on PPO's rollout path, functional style.

head_out()        the pre-activation head outputs [logits | v] / [mu_raw | log_std_raw | v] of a policy-value network
minibatch_loss()  the V-MPO loss of one minibatch as a function of the head outputs and the multipliers (autograd)
closed_form()     its gradients in closed form (what csrc/vmpo.cu computes)
learn()           one learn: PPO's pre-pass and GAE (oracle.ppo.gae), then n_epoch passes of injected permutations, one
                  torch Adam over the network's parameters + [eta, alpha_mu, alpha_sigma], clip_grad_norm_ on the
                  network's parameters only, and the clamps of the multipliers to their minima after every step.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import nets
from .ppo import gae

LOG_SQRT_2PI = 0.5 * math.log(2 * math.pi)


def head_out(p, x, continuous):
    h = F.relu(F.linear(nets.head(p, x), p["l.weight"], p["l.bias"]))
    if continuous:
        parts = [F.linear(h, p["mu.weight"], p["mu.bias"]), F.linear(h, p["log_std.weight"], p["log_std.bias"])]
    else:
        parts = [F.linear(h, p["pi.weight"], p["pi.bias"])]
    return torch.cat(parts + [F.linear(h, p["v.weight"], p["v.bias"])], dim=1)


def _rows(out, out_old, action, A, continuous):
    """Per-row log pi(a|s), KL_mu (discrete: the KL), KL_sigma (discrete: 0) and v."""
    v = out[:, -1]
    if continuous:
        mu, sd = out[:, :A].clamp(-5, 5), torch.tanh(out[:, A:2 * A]).exp()
        mu_o, sd_o = out_old[:, :A].clamp(-5, 5), torch.tanh(out_old[:, A:2 * A]).exp()
        z = torch.atanh(torch.clamp(action, -1 + 1e-7, 1 - 1e-7))
        logpi = (-(z - mu) ** 2 / (2 * sd ** 2) - sd.log() - LOG_SQRT_2PI).sum(1)
        kl_mu = 0.5 * ((mu - mu_o) ** 2 / sd_o ** 2).sum(1)
        kl_sigma = 0.5 * (sd_o ** 2 / sd ** 2 - 1 + torch.log(sd ** 2 / sd_o ** 2)).sum(1)
        return logpi, kl_mu, kl_sigma, v
    lsm, lsm_o = F.log_softmax(out[:, :A], dim=1), F.log_softmax(out_old[:, :A], dim=1)
    logpi = lsm.gather(1, action.long().view(-1, 1)).squeeze(1)
    kl = (lsm_o.exp() * (lsm_o - lsm)).sum(1)
    return logpi, kl, torch.zeros_like(kl), v


def top_half(adv):
    """Lower median (torch.median) and the strict top set adv > median."""
    m = adv.median()
    return m, adv > m


def minibatch_loss(out, out_old, action, adv, ret, eta, alpha_mu, alpha_sigma, eps, A, continuous):
    """eta / alpha_mu / alpha_sigma: 0-d tensors (leaves if their gradients are wanted); eps = (eps_eta, eps_alpha_mu,
    eps_alpha_sigma).  Returns (loss, aux)."""
    eps_eta, eps_mu, eps_sigma = eps
    logpi, kl_mu, kl_sigma, v = _rows(out, out_old, action, A, continuous)
    m, top = top_half(adv)
    n = int(top.sum())
    if n > 0:
        z = adv[top] / eta
        M = z.max()
        e = torch.exp(z - M)
        S = e.sum()
        psi = (e / S).detach()
        actor_loss = -(psi * logpi[top]).sum()
        eta_loss = eta * eps_eta + eta * (M + torch.log(S) - math.log(n))
    else:                               # empty top half: both terms 0 (a documented deviation from the reference's NaN)
        actor_loss = (logpi * 0).sum()
        eta_loss = eta * 0
    alpha_loss = torch.mean(alpha_mu * (eps_mu - kl_mu.detach()) + alpha_mu.detach() * kl_mu)
    if continuous:
        alpha_loss = alpha_loss + torch.mean(alpha_sigma * (eps_sigma - kl_sigma.detach()) + alpha_sigma.detach() * kl_sigma)
    critic_loss = F.mse_loss(v, ret)
    loss = actor_loss + eta_loss + alpha_loss + critic_loss
    aux = {"actor_loss": actor_loss, "critic_loss": critic_loss, "eta_loss": eta_loss, "alpha_loss": alpha_loss,
           "kl_mu": kl_mu.mean(), "kl_sigma": kl_sigma.mean(), "n": n, "median": m}
    return loss, aux


def closed_form(out, out_old, action, adv, ret, eta, alpha_mu, alpha_sigma, eps, A, continuous):
    """(d loss / d out [B, nout], d loss / d [eta, alpha_mu, alpha_sigma]) in closed form; all float64 tensors."""
    eps_eta, eps_mu, eps_sigma = eps
    B = out.shape[0]
    m, top = top_half(adv)
    n = int(top.sum())
    w = torch.zeros_like(adv)
    d_eta = torch.zeros((), dtype=out.dtype)
    if n > 0:
        z = adv[top] / eta
        M = z.max()
        e = torch.exp(z - M)
        S = e.sum()
        w[top] = e / S
        d_eta = eps_eta + (M + torch.log(S) - math.log(n)) - (w[top] * adv[top]).sum() / eta
    g = torch.zeros_like(out)
    g[:, -1] = 2 * (out[:, -1] - ret) / B
    if continuous:
        omu, ols = out[:, :A], out[:, A:2 * A]
        mu, ls = omu.clamp(-5, 5), torch.tanh(ols)
        sd = ls.exp()
        mu_o, sd_o = out_old[:, :A].clamp(-5, 5), torch.tanh(out_old[:, A:2 * A]).exp()
        zc = torch.atanh(torch.clamp(action, -1 + 1e-7, 1 - 1e-7))
        d = zc - mu
        wb = w.view(-1, 1)
        gmu = -wb * d / sd ** 2 + alpha_mu / B * (mu - mu_o) / sd_o ** 2
        gsd = -wb * (d ** 2 / sd ** 3 - 1 / sd) + alpha_sigma / B * (1 / sd - sd_o ** 2 / sd ** 3)
        g[:, :A] = gmu * ((omu >= -5) & (omu <= 5)).to(out.dtype)
        g[:, A:2 * A] = gsd * sd * (1 - ls ** 2)
        kl_mu = 0.5 * ((mu - mu_o) ** 2 / sd_o ** 2).sum(1)
        kl_sigma = 0.5 * (sd_o ** 2 / sd ** 2 - 1 + torch.log(sd ** 2 / sd_o ** 2)).sum(1)
        d_sigma = eps_sigma - kl_sigma.mean()
    else:
        lsm, lsm_o = F.log_softmax(out[:, :A], dim=1), F.log_softmax(out_old[:, :A], dim=1)
        p, p_o = lsm.exp(), lsm_o.exp()
        onehot = F.one_hot(action.long().view(-1), A).to(out.dtype)
        g[:, :A] = -w.view(-1, 1) * (onehot - p) + alpha_mu / B * (p * p_o.sum(1, keepdim=True) - p_o)
        kl_mu = (p_o * (lsm_o - lsm)).sum(1)
        d_sigma = torch.zeros((), dtype=out.dtype)
    dmult = torch.stack([d_eta, eps_mu - kl_mu.mean(), d_sigma])
    return g, dmult


def learn(params, batch, hp, perms, lr, mult, mins, eps):
    """params: dict name -> tensor; batch: dict of [N*T, ...] tensors (state, next_state, action, reward, done);
    hp: PPO's learn keys (continuous, n_step, gamma, lambda, standardize, batch_size, n_epoch, clip_grad_norm) and the
    action size A; mult: (eta, alpha_mu, alpha_sigma) initial values; mins: their minima; eps: (eps_eta, eps_alpha_mu,
    eps_alpha_sigma).  Everything runs in float64.  Returns post-learn params, multipliers, the optimiser state and the
    result dict."""
    continuous, A = hp["continuous"], hp["A"]
    dd = lambda t: t.detach().to(torch.float64)
    p = {k: dd(v).clone().requires_grad_(True) for k, v in params.items()}
    m = [torch.tensor(float(v), dtype=torch.float64, requires_grad=True) for v in mult]
    opt = torch.optim.Adam(list(p.values()) + m, lr=lr)
    state, next_state, action = dd(batch["state"]), dd(batch["next_state"]), dd(batch["action"])
    reward, done = dd(batch["reward"]).view(-1, 1), dd(batch["done"]).view(-1, 1)
    with torch.no_grad():
        out_old = head_out(p, state, continuous)
        value = out_old[:, -1:].clone()
        next_value = head_out(p, next_state, continuous)[:, -1:]
    adv, ret = gae(reward, done, value, next_value, hp["n_step"], hp["gamma"], hp["lambda"], hp["standardize"])
    adv, ret = adv.view(-1), ret.view(-1)
    if not continuous:
        action = action.view(-1)
    stats = {k: [] for k in ("actor_loss", "critic_loss", "eta_loss", "alpha_loss")}
    B = hp["batch_size"]
    for epoch in range(hp["n_epoch"]):
        idxs = np.asarray(perms[epoch])
        for offset in range(0, len(adv), B):
            idx = torch.as_tensor(idxs[offset:offset + B], dtype=torch.long)
            out = head_out(p, state[idx], continuous)
            loss, aux = minibatch_loss(out, out_old[idx], action[idx], adv[idx], ret[idx], m[0], m[1], m[2], eps, A,
                                       continuous)
            opt.zero_grad(set_to_none=False)
            for t in m:                     # a multiplier the loss does not use (discrete alpha_sigma) gets a zero gradient
                t.grad = torch.zeros_like(t)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(list(p.values()), hp["clip_grad_norm"])
            opt.step()
            with torch.no_grad():
                for t, lo in zip(m, mins):
                    t.clamp_(min=lo)
            for k in stats:
                stats[k].append(float(aux[k]))
    result = {k: float(np.mean(v)) for k, v in stats.items()}
    result.update(eta=float(m[0]), alpha_mu=float(m[1]), alpha_sigma=float(m[2]), mean_ret=float(ret.mean()))
    return {"params": {k: v.detach().clone() for k, v in p.items()}, "mult": [float(t) for t in m],
            "opt_state": opt.state_dict(), "result": result, "adv": adv, "ret": ret, "out_old": out_old}
