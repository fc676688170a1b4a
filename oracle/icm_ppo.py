"""Float64 CPU oracle of ICM-PPO (Pathak et al., ICML 2017) on PPO's rollout path, functional style.

RunningMeanStd    OpenAI baselines' running statistics (numpy float64, count starting at 1e-4, parallel merge)
reward_filter()   the per-env reward-forward filter rewems = gamma * rewems + r_i over t
icm_forward()     phi(x) = elu(fc2(elu(BN(fc1(norm(x))))))  (icm_cnn: the CNN trunk in place of norm(x)) with bn1 on s and bn1_next on s' in training mode (running
                  buffers updated in place), f = fc_f2([relu(fc_f1([phi(s), a])), a]), g = pi(relu(inv([phi(s), phi(s')])))
icm_loss()        r_i = eta / 2 sum_F |f - phi(s')|, l_f = MSE(f, phi(s').detach()), l_i = cross-entropy / MSE
learn()           one learn: rms_obs update, the no-grad r_i pre-pass over the whole rollout, the filter / rms_ri / scaling
                  of r_i, PPO's pre-pass and GAE on extrinsic_coeff * r + intrinsic_coeff * r_i, then n_epoch passes of
                  injected permutations with loss = lamb * L_ppo + beta * l_f + (1 - beta) * l_i, clip_grad_norm_ on the
                  policy network's parameters only and one torch Adam over the policy + ICM parameters.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import nets
from . import ppo as oppo

BN_EPS, BN_MOMENTUM, OBS_CLIP = 1e-5, 0.1, 5.0


class RunningMeanStd:
    def __init__(self, shape):
        self.mean = np.zeros(shape, np.float64)
        self.var = np.ones(shape, np.float64)
        self.count = 1e-4

    def update(self, x):
        x = np.asarray(x, np.float64)
        bm, bv, bc = x.mean(axis=0), x.var(axis=0), x.shape[0]
        delta = bm - self.mean
        tot = self.count + bc
        m2 = self.var * self.count + bv * bc + delta ** 2 * self.count * bc / tot
        self.mean = self.mean + delta * bc / tot
        self.var = m2 / tot
        self.count = tot


def reward_filter(rewems, ri, gamma):
    """rewems [N] (float64), ri [N, T] -> (filtered [N, T], new rewems)."""
    out = np.empty_like(ri, dtype=np.float64)
    e = np.asarray(rewems, np.float64).copy()
    for t in range(ri.shape[1]):
        e = gamma * e + ri[:, t]
        out[:, t] = e
    return out, e


def normalize(x, rms):
    if rms is None:
        return x
    m, v = torch.as_tensor(rms.mean, dtype=x.dtype), torch.as_tensor(rms.var, dtype=x.dtype)
    return ((x - m) / torch.sqrt(v)).clamp(-OBS_CLIP, OBS_CLIP)


def action_rows(action, A, continuous):
    if continuous:
        return action.reshape(-1, A)
    return F.one_hot(action.long().reshape(-1), A).to(torch.float64)


def encoder(p, buffers, x, bn):
    if "head.conv1.weight" in p:                          # icm_cnn: the CNN trunk on the [B, 4, 84, 84] stacks
        x = nets.cnn_head(p, x.reshape(x.shape[0], 4, 84, 84))
    h = F.linear(x, p["fc1.weight"], p["fc1.bias"])
    if bn is not None:
        h = F.batch_norm(h, buffers[f"{bn}.running_mean"], buffers[f"{bn}.running_var"], p[f"{bn}.weight"],
                         p[f"{bn}.bias"], training=True, momentum=BN_MOMENTUM, eps=BN_EPS)
        buffers[f"{bn}.num_batches_tracked"] += 1
    return F.elu(F.linear(F.elu(h), p["fc2.weight"], p["fc2.bias"]))


def icm_forward(p, buffers, s, s_next, a, batch_norm=True, inverse=True):
    """s / s_next already normalised; a: the action rows ([B, A] one-hot or raw).  Returns (f, phi(s'), g or None)."""
    phi = encoder(p, buffers, s, "bn1" if batch_norm else None)
    phi_n = encoder(p, buffers, s_next, "bn1_next" if batch_norm else None)
    h = F.relu(F.linear(torch.cat([phi, a], 1), p["fc_f1.weight"], p["fc_f1.bias"]))
    f = F.linear(torch.cat([h, a], 1), p["fc_f2.weight"], p["fc_f2.bias"])
    g = None
    if inverse:
        g = F.linear(F.relu(F.linear(torch.cat([phi, phi_n], 1), p["inv.weight"], p["inv.bias"])), p["pi.weight"], p["pi.bias"])
    return f, phi_n, g


def icm_loss(f, phi_n, g, action, A, continuous, eta, beta):
    """Returns (r_i [B], l_f, l_i, beta * l_f + (1 - beta) * l_i)."""
    r_i = eta * 0.5 * (f - phi_n).abs().sum(1)
    l_f = F.mse_loss(f, phi_n.detach())
    if continuous:
        l_i = F.mse_loss(g, action.reshape(-1, A))
    else:
        l_i = F.cross_entropy(g, action.long().reshape(-1))
    return r_i, l_f, l_i, beta * l_f + (1 - beta) * l_i


def closed_form(f, phi_n, g, action, A, continuous, beta):
    """(d loss / d f, d loss / d g) of beta * l_f + (1 - beta) * l_i in closed form (what csrc/icm.cu computes)."""
    B, Fw = f.shape
    df = beta * 2 * (f - phi_n) / (B * Fw)
    if continuous:
        dg = (1 - beta) * 2 * (g - action.reshape(-1, A)) / (B * A)
    else:
        dg = (1 - beta) * (torch.softmax(g, 1) - F.one_hot(action.long().reshape(-1), A).to(g.dtype)) / B
    return df, dg


def new_state(D, N):
    """The learner's persistent statistics: rms_obs, rms_ri and the filter state."""
    return {"rms_obs": RunningMeanStd((D,)), "rms_ri": RunningMeanStd(()), "rewems": np.zeros(N)}


def learn(params, icm_params, icm_buffers, batch, hp, ihp, perms, lr, stats_state, opt_state=None):
    """params / icm_params / icm_buffers: dicts name -> tensor; batch: dict of [N*T, ...] tensors (state, next_state,
    action, reward, done); hp: PPO's learn keys (continuous, A, n_step, gamma, lambda, standardize, batch_size, n_epoch,
    clip_grad_norm, eps_clip, vf_coef, ent_coef); ihp: the ICM keys (beta, lamb, eta, extrinsic_coeff, intrinsic_coeff,
    obs_normalize, ri_normalize, batch_norm); stats_state: new_state(), updated in place; opt_state: a previous learn's.  Everything runs in float64.
    Returns post-learn params, ICM params and buffers, the optimiser state, the reward gae read and the result dict."""
    continuous, A = hp["continuous"], hp["A"]
    dd = lambda t: t.detach().to(torch.float64)
    p = {k: dd(v).clone().requires_grad_(True) for k, v in params.items()}
    q = {k: dd(v).clone().requires_grad_(True) for k, v in icm_params.items()}
    buf = {k: (v.detach().clone() if v.dtype == torch.int64 else dd(v).clone()) for k, v in icm_buffers.items()}
    opt = torch.optim.Adam(list(p.values()) + list(q.values()), lr=lr)
    if opt_state is not None:
        opt.load_state_dict(opt_state)
    state, next_state, action = dd(batch["state"]), dd(batch["next_state"]), dd(batch["action"])
    reward, done = dd(batch["reward"]).view(-1, 1), dd(batch["done"]).view(-1, 1)
    NT, T = state.shape[0], hp["n_step"]
    N = NT // T
    a_rows = action_rows(action, A, continuous)
    rms = stats_state["rms_obs"] if ihp["obs_normalize"] else None
    if rms is not None:
        rms.update(next_state.numpy())
    with torch.no_grad():
        f, phi_n, _ = icm_forward(q, buf, normalize(state, rms), normalize(next_state, rms), a_rows, ihp["batch_norm"],
                                  inverse=False)
        r_i = (ihp["eta"] * 0.5 * (f - phi_n).abs().sum(1)).numpy()
    if ihp["ri_normalize"]:
        filt, stats_state["rewems"] = reward_filter(stats_state["rewems"], r_i.reshape(N, T), hp["gamma"])
        stats_state["rms_ri"].update(filt.reshape(-1))
        r_i = r_i / (np.sqrt(stats_state["rms_ri"].var) + 1e-7)
    mixed = ihp["extrinsic_coeff"] * reward + ihp["intrinsic_coeff"] * torch.as_tensor(r_i).view(-1, 1)
    value, next_value, log_prob_old = oppo.prepass(p, state, action, next_state, continuous)
    adv, ret = oppo.gae(mixed, done, value, next_value, T, hp["gamma"], hp["lambda"], hp["standardize"])
    stats = {k: [] for k in ("actor_loss", "critic_loss", "entropy_loss", "max_ratio", "min_prob", "r_i", "l_f", "l_i")}
    B = hp["batch_size"]
    for epoch in range(hp["n_epoch"]):
        idxs = np.asarray(perms[epoch])
        for offset in range(0, NT, B):
            idx = torch.as_tensor(idxs[offset:offset + B], dtype=torch.long)
            l_ppo, aux = oppo.minibatch_loss(p, state[idx], action[idx], value[idx], ret[idx], adv[idx],
                                             log_prob_old[idx], continuous, hp["eps_clip"], hp["vf_coef"], hp["ent_coef"])
            f, phi_n, g = icm_forward(q, buf, normalize(state[idx], rms), normalize(next_state[idx], rms), a_rows[idx],
                                      ihp["batch_norm"])
            ri_b, l_f, l_i, l_icm = icm_loss(f, phi_n, g, action[idx], A, continuous, ihp["eta"], ihp["beta"])
            loss = ihp["lamb"] * l_ppo + l_icm
            opt.zero_grad(set_to_none=True)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(list(p.values()), hp["clip_grad_norm"])
            opt.step()
            for k in ("actor_loss", "critic_loss", "entropy_loss", "max_ratio", "min_prob"):
                stats[k].append(aux[k].item())
            stats["r_i"].append(ri_b.mean().item())
            stats["l_f"].append(l_f.item())
            stats["l_i"].append(l_i.item())
    result = {k: float(np.mean(stats[k])) for k in ("actor_loss", "critic_loss", "entropy_loss", "r_i", "l_f", "l_i")}
    result.update(max_ratio=max(stats["max_ratio"]), min_prob=min(stats["min_prob"]), mean_ret=float(ret.mean()))
    return {"params": {k: v.detach().clone() for k, v in p.items()}, "icm": {k: v.detach().clone() for k, v in q.items()},
            "buffers": buf, "opt_state": opt.state_dict(), "reward": mixed.view(-1), "result": result}
