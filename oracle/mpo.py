"""Float64 CPU oracle of MPO (Abdolmaleki et al., arXiv:1806.06920) on replayed n-step windows, functional style.

A batch holds B windows: state [B, n+1, D], action [B, n] (discrete, int) or [B, n, A] (continuous), reward / done /
log_mu [B, n].  Continuous E-step normals eps are [B, n+1, K, A].

actor_out() / critic_q()   the pre-activation actor head ([logits] / [mu_raw | log_std_raw]) and the critic's values
logp()                     log pi(a | s), continuous: Normal log-pdf of atanh(clamp(a, +-(1-1e-7))), no Jacobian
retrace()                  the Retrace recursion from V'_{t+1}, c_{t+1}, Q'(s_{t+1}, a_{t+1}), r, d
critic_target()            Qret from the target networks' outputs (c = 0 for "1step_TD")
policy_loss()              L_pi + L_eta + L_alpha as a function of the actor rows and the multipliers (autograd)
policy_closed()            its gradients in closed form (what csrc/mpo.cu computes)
Learner                    whole learn()s: critic Adam, actor Adam with clip_grad_norm_ on the actor over actor +
                           multipliers, the clamps to the minima, the hard target copy every target_update_period learns
"""
import math

import torch
import torch.nn.functional as F

from . import nets
from .actor_critic import continuous_q_network

LOG_SQRT_2PI = 0.5 * math.log(2 * math.pi)


def actor_out(p, x, continuous):
    h = F.relu(F.linear(nets.mlp_head(p, x), p["l.weight"], p["l.bias"]))
    if continuous:
        return torch.cat([F.linear(h, p["mu.weight"], p["mu.bias"]), F.linear(h, p["log_std.weight"], p["log_std.bias"])], -1)
    return F.linear(h, p["pi.weight"], p["pi.bias"])


def critic_q(p, x, a=None):
    """Discrete: all A values [.., A]; continuous: Q(x, a) [..]."""
    if a is None:
        return nets.discrete_q_network(p, x)
    return continuous_q_network(p, x, a).squeeze(-1)


def gauss(out, A):
    return out[..., :A].clamp(-5, 5), torch.tanh(out[..., A:2 * A])


def normal_logpdf(z, mu, ls):
    return (-(z - mu) ** 2 / (2 * torch.exp(2 * ls)) - ls - LOG_SQRT_2PI).sum(-1)


def logp(out, action, A, continuous):
    if continuous:
        mu, ls = gauss(out, A)
        return normal_logpdf(torch.atanh(torch.clamp(action, -1 + 1e-7, 1 - 1e-7)), mu, ls)
    return F.log_softmax(out[..., :A], -1).gather(-1, action.long().unsqueeze(-1)).squeeze(-1)


def sample(tout, eps, A):
    """tout [..., 2A], eps [..., K, A] -> (z, tanh(z)) [..., K, A]."""
    mu, ls = gauss(tout, A)
    z = mu.unsqueeze(-2) + ls.exp().unsqueeze(-2) * eps
    return z, torch.tanh(z)


def retrace(v_next, c_next, qt_next, reward, done, gamma):
    """All [B, n]: v_next[:, t] = V'_{t+1}, c_next[:, t] = c_{t+1}, qt_next[:, t] = Q'(s_{t+1}, a_{t+1}) (the last
    column of c_next / qt_next is unused).  Returns Qret [B, n]."""
    n = reward.shape[1]
    out = torch.zeros_like(reward)
    nxt = torch.zeros_like(reward[:, 0])
    for t in reversed(range(n)):
        c = c_next[:, t] if t < n - 1 else torch.zeros_like(nxt)
        q = qt_next[:, t] if t < n - 1 else torch.zeros_like(nxt)
        nxt = reward[:, t] + gamma * (1 - done[:, t]) * (v_next[:, t] + c * (nxt - q))
        out[:, t] = nxt
    return out


def critic_target(tout, tq, action, log_mu, reward, done, gamma, A, continuous, use_retrace=True):
    """tout [B, n+1, nout]; tq discrete [B, n+1, A], continuous [B, n+1, K+1] (K samples, then the taken action)."""
    n = reward.shape[1]
    if continuous:
        v = tq[:, 1:, :-1].mean(-1)
        qt = tq[:, 1:n, -1]
    else:
        v = (F.softmax(tout[..., :A], -1) * tq)[:, 1:].sum(-1)
        qt = tq[:, 1:n].gather(-1, action[:, 1:].long().unsqueeze(-1)).squeeze(-1)
    lp = logp(tout[:, 1:n], action[:, 1:], A, continuous)
    c = torch.clamp(torch.exp(lp - log_mu[:, 1:]), max=1.0) if use_retrace else torch.zeros_like(lp)
    pad = torch.zeros_like(reward[:, :1])
    return retrace(v, torch.cat([c, pad], 1), torch.cat([qt, pad], 1), reward, done, gamma)


def policy_loss(out, tout, tq, z, eta, alpha_mu, alpha_sigma, eps, A, continuous):
    """Rows s: out / tout [S, nout] (online / target actor), tq discrete [S, A] = Q'(s, .), continuous [S, K] = Q'(s, a_k),
    z [S, K, A] the pre-tanh samples.  eta / alpha_*: 0-d tensors.  Returns (loss, aux)."""
    eps_eta, eps_mu, eps_sigma = eps
    if continuous:
        mu, ls = gauss(out, A)
        mu_o, ls_o = gauss(tout, A)
        x = tq / eta
        lme = torch.logsumexp(x, -1) - math.log(x.shape[-1])
        q = torch.softmax(x, -1).detach()
        lp = normal_logpdf(z, mu.unsqueeze(1), ls_o.unsqueeze(1)) + normal_logpdf(z, mu_o.unsqueeze(1), ls.unsqueeze(1))
        actor_loss = -(q * lp).sum(-1).mean()
        sd, sd_o = ls.exp(), ls_o.exp()
        kl_mu = 0.5 * ((mu - mu_o) ** 2 / sd_o ** 2).sum(-1)
        kl_sigma = 0.5 * (sd_o ** 2 / sd ** 2 - 1 + torch.log(sd ** 2 / sd_o ** 2)).sum(-1)
    else:
        lsm, lsm_o = F.log_softmax(out[:, :A], -1), F.log_softmax(tout[:, :A], -1)
        x = lsm_o + tq / eta
        lme = torch.logsumexp(x, -1)
        q = torch.softmax(x, -1).detach()
        actor_loss = -(q * lsm).sum(-1).mean()
        kl_mu = (lsm_o.exp() * (lsm_o - lsm)).sum(-1)
        kl_sigma = torch.zeros_like(kl_mu)
    eta_loss = eta * eps_eta + eta * lme.mean()
    alpha_loss = torch.mean(alpha_mu * (eps_mu - kl_mu.detach()) + alpha_mu.detach() * kl_mu)
    if continuous:
        alpha_loss = alpha_loss + torch.mean(alpha_sigma * (eps_sigma - kl_sigma.detach()) + alpha_sigma.detach() * kl_sigma)
    loss = actor_loss + eta_loss + alpha_loss
    return loss, {"actor_loss": actor_loss, "eta_loss": eta_loss, "alpha_loss": alpha_loss, "kl_mu": kl_mu.mean(),
                  "kl_sigma": kl_sigma.mean()}


def policy_closed(out, tout, tq, z, eta, alpha_mu, alpha_sigma, eps, A, continuous):
    """(d loss / d out [S, nout], d loss / d [eta, alpha_mu, alpha_sigma]) in closed form."""
    eps_eta, eps_mu, eps_sigma = eps
    S = out.shape[0]
    g = torch.zeros_like(out)
    if continuous:
        omu = out[:, :A]
        mu, ls = gauss(out, A)
        mu_o, ls_o = gauss(tout, A)
        sd, sd_o = ls.exp(), ls_o.exp()
        x = tq / eta
        q = torch.softmax(x, -1)
        d_eta = eps_eta + (torch.logsumexp(x, -1) - math.log(x.shape[-1]) - (q * x).sum(-1)).mean()
        qz = (q.unsqueeze(-1) * z).sum(1)
        q3 = (q.unsqueeze(-1) * (z - mu_o.unsqueeze(1)) ** 2).sum(1)
        gmu = -(qz - mu) / sd_o ** 2 / S + alpha_mu / S * (mu - mu_o) / sd_o ** 2
        gsd = -(q3 / sd ** 3 - 1 / sd) / S + alpha_sigma / S * (1 / sd - sd_o ** 2 / sd ** 3)
        g[:, :A] = gmu * ((omu >= -5) & (omu <= 5)).to(out.dtype)
        g[:, A:] = gsd * sd * (1 - ls ** 2)
        kl_mu = 0.5 * ((mu - mu_o) ** 2 / sd_o ** 2).sum(-1)
        kl_sigma = 0.5 * (sd_o ** 2 / sd ** 2 - 1 + torch.log(sd ** 2 / sd_o ** 2)).sum(-1)
        d_sigma = eps_sigma - kl_sigma.mean()
    else:
        lsm, lsm_o = F.log_softmax(out[:, :A], -1), F.log_softmax(tout[:, :A], -1)
        p, p_o = lsm.exp(), lsm_o.exp()
        x = lsm_o + tq / eta
        q = torch.softmax(x, -1)
        d_eta = eps_eta + (torch.logsumexp(x, -1) - (q * tq).sum(-1) / eta).mean()
        g[:, :A] = -(q - p) / S + alpha_mu / S * (p * p_o.sum(-1, keepdim=True) - p_o)
        kl_mu = (p_o * (lsm_o - lsm)).sum(-1)
        d_sigma = torch.zeros((), dtype=out.dtype)
    return g, torch.stack([torch.as_tensor(d_eta, dtype=out.dtype), eps_mu - kl_mu.mean(), torch.as_tensor(d_sigma, dtype=out.dtype)])


class Learner:
    """Float64 restatement of MPO.learn(): hp = dict(continuous, A, K, gamma, lr, clip_grad_norm, target_update_period,
    critic_loss_type, eps=(eps_eta, eps_alpha_mu, eps_alpha_sigma), mins=(min_eta, min_alpha_mu, min_alpha_sigma))."""

    def __init__(self, actor, critic, mult, hp):
        dd = lambda p: {k: v.detach().to(torch.float64).clone().requires_grad_(True) for k, v in p.items()}
        self.hp = hp
        self.actor, self.critic = dd(actor), dd(critic)
        self.t_actor = {k: v.detach().clone() for k, v in self.actor.items()}
        self.t_critic = {k: v.detach().clone() for k, v in self.critic.items()}
        self.mult = [torch.tensor(float(v), dtype=torch.float64, requires_grad=True) for v in mult]
        self.actor_opt = torch.optim.Adam(list(self.actor.values()) + self.mult, lr=hp["lr"])
        self.critic_opt = torch.optim.Adam(list(self.critic.values()), lr=hp["lr"])
        self.num_learn = 0

    def learn(self, batch, eps=None):
        hp, cont, A = self.hp, self.hp["continuous"], self.hp["A"]
        dd = lambda t: t.detach().to(torch.float64) if t.is_floating_point() else t.detach()
        st, a, r, d, lmu = (dd(batch[k]) for k in ("state", "action", "reward", "done", "log_mu"))
        B, n = r.shape
        S = B * n
        with torch.no_grad():
            tout = actor_out(self.t_actor, st, cont)                       # [B, n+1, nout]
            if cont:
                z, a_s = sample(tout, dd(eps), A)                           # [B, n+1, K, A]
                K = z.shape[2]
                xs = st.unsqueeze(2).expand(B, n + 1, K, st.shape[-1])
                q_s = critic_q(self.t_critic, xs, a_s)                       # [B, n+1, K]
                q_a = torch.cat([critic_q(self.t_critic, st[:, :n], a), torch.zeros(B, 1, dtype=st.dtype)], 1)
                tq = torch.cat([q_s, q_a.unsqueeze(-1)], -1)
            else:
                z, tq = None, critic_q(self.t_critic, st)
            qret = critic_target(tout, tq, a, lmu, r, d, hp["gamma"], A, cont, hp["critic_loss_type"] == "retrace")
        # critic
        if cont:
            q = critic_q(self.critic, st[:, :n], a)
        else:
            q = critic_q(self.critic, st[:, :n]).gather(-1, a.long().unsqueeze(-1)).squeeze(-1)
        critic_loss = ((q - qret) ** 2).mean()
        self.critic_opt.zero_grad(set_to_none=False)
        critic_loss.backward()
        self.critic_opt.step()
        # actor + multipliers
        out = actor_out(self.actor, st[:, :n].reshape(S, -1), cont)
        tq_rows = (tq[:, :n, :-1] if cont else tq[:, :n]).reshape(S, -1)
        z_rows = z[:, :n].reshape(S, z.shape[2], A) if cont else None
        loss, aux = policy_loss(out, tout[:, :n].reshape(S, -1), tq_rows, z_rows, *self.mult, hp["eps"], A, cont)
        self.actor_opt.zero_grad(set_to_none=False)
        for t in self.mult:
            t.grad = torch.zeros_like(t)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(list(self.actor.values()), hp["clip_grad_norm"])
        self.actor_opt.step()
        with torch.no_grad():
            for t, lo in zip(self.mult, hp["mins"]):
                t.clamp_(min=lo)
            if (self.num_learn + 1) % hp["target_update_period"] == 0:
                for src, dst in ((self.actor, self.t_actor), (self.critic, self.t_critic)):
                    for k in src:
                        dst[k].copy_(src[k])
        self.num_learn += 1
        result = {k: float(aux[k].detach()) for k in ("actor_loss", "eta_loss", "alpha_loss")}
        result.update(critic_loss=float(critic_loss), mean_Q=float(qret.mean()), eta=float(self.mult[0]),
                      alpha_mu=float(self.mult[1]), alpha_sigma=float(self.mult[2]))
        return result, qret
