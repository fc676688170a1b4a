"""Float64 CPU oracle of RND-PPO (Burda et al., 2018, arXiv:1810.12894) on PPO's rollout path, functional style.

target()          t = fc2(elu(fc1(x')))  (rnd_cnn: the target's own CNN trunk in place of x')
predictor()       p = fc3(elu(fc2(elu(BN(fc1(x'))))))  with BN in training mode (running buffers updated in place)
rnd_loss()        r_i = mean_F (p - t)^2 per row, rnd_loss = mean_B r_i
ppo_loss()        PPO's loss on the head outputs [pi | v | v_i] / [mu | log_std | v | v_i] with a second clipped critic
adv_mix()         extrinsic_coeff * adv_e + intrinsic_coeff * adv_i, then PPO's per-row standardisation
learn()           one learn: rms_obs update, the target / predictor pre-pass over the whole rollout, the filter / rms_ri /
                  scaling of r_i, the pre-pass of s and s', one GAE per stream (intrinsic: done masked out when
                  non_episodic), the mix, then n_epoch passes of injected permutations with
                  loss = L_ppo(two critics) + rnd_loss, clip_grad_norm_ on the policy network's parameters only and one torch
                  Adam over the policy + predictor parameters.  The target is never updated.
RunningMeanStd, reward_filter and normalize are ICM-PPO's (oracle/icm_ppo.py); gae is PPO's.
"""
import numpy as np
import torch
import torch.nn.functional as F
from torch.distributions import Categorical, Normal

from . import nets
from . import ppo as oppo
from .icm_ppo import BN_EPS, BN_MOMENTUM, RunningMeanStd, normalize, reward_filter   # noqa: F401  (re-exported)


def _trunk(p, x):
    if "head.conv1.weight" in p:                          # rnd_cnn: the CNN trunk on the [B, 4, 84, 84] stacks
        return nets.cnn_head(p, x.reshape(x.shape[0], 4, 84, 84))
    return x


def target(p, x):
    return F.linear(F.elu(F.linear(_trunk(p, x), p["fc1.weight"], p["fc1.bias"])), p["fc2.weight"], p["fc2.bias"])


def predictor(p, buffers, x, batch_norm=True):
    h = F.linear(_trunk(p, x), p["fc1.weight"], p["fc1.bias"])
    if batch_norm:
        h = F.batch_norm(h, buffers["bn1.running_mean"], buffers["bn1.running_var"], p["bn1.weight"], p["bn1.bias"],
                         training=True, momentum=BN_MOMENTUM, eps=BN_EPS)
        buffers["bn1.num_batches_tracked"] += 1
    h = F.elu(F.linear(F.elu(h), p["fc2.weight"], p["fc2.bias"]))
    return F.linear(h, p["fc3.weight"], p["fc3.bias"])


def rnd_loss(pred, tgt):
    r_i = ((pred - tgt) ** 2).mean(1)
    return r_i, r_i.mean()


def closed_form(pred, tgt):
    """d rnd_loss / d p in closed form (what csrc/rnd.cu computes)."""
    return 2 * (pred - tgt) / pred.numel()


def values(p, x):
    """(v, v_i) of the two-value policy network."""
    h = F.relu(F.linear(nets.head(p, x), p["l.weight"], p["l.bias"]))
    return F.linear(h, p["v.weight"], p["v.bias"]), F.linear(h, p["v_i.weight"], p["v_i.bias"])


def _clipped_critic(v, v_old, ret, eps_clip):
    v_clip = v_old + torch.clamp(v - v_old, -eps_clip, eps_clip)
    return torch.max(F.mse_loss(v, ret), F.mse_loss(v_clip, ret))


def ppo_loss(out, action, adv, ret, v_old, ret_i, v_i_old, log_prob_old, A, continuous, eps_clip, vf_coef, ent_coef):
    """PPO's minibatch loss (oracle/ppo.py minibatch_loss) on the raw head outputs, with critic_loss the sum of the
    extrinsic and the intrinsic clipped critics.  Every argument but A / continuous / coefficients is [B, .]."""
    if continuous:
        mu = torch.clamp(out[:, :A], -5.0, 5.0)
        m = Normal(mu, torch.tanh(out[:, A:2 * A]).exp())
        log_prob = m.log_prob(torch.atanh(torch.clamp(action, -1 + 1e-7, 1 - 1e-7)))
        v, v_i = out[:, 2 * A:2 * A + 1], out[:, 2 * A + 1:2 * A + 2]
    else:
        m = Categorical(torch.exp(F.log_softmax(out[:, :A], dim=-1)))
        log_prob = m.log_prob(action.long().reshape(-1)).unsqueeze(-1)
        v, v_i = out[:, A:A + 1], out[:, A + 1:A + 2]
    ratio = (log_prob - log_prob_old).sum(1, keepdim=True).exp()
    actor_loss = -torch.min(ratio * adv, torch.clamp(ratio, 1 - eps_clip, 1 + eps_clip) * adv).mean()
    critic_e = _clipped_critic(v, v_old, ret, eps_clip)
    critic_i = _clipped_critic(v_i, v_i_old, ret_i, eps_clip)
    entropy_loss = -m.entropy().mean()
    critic_loss = critic_e + critic_i
    loss = actor_loss + vf_coef * critic_loss + ent_coef * entropy_loss
    return loss, {"actor_loss": actor_loss, "critic_loss": critic_loss, "entropy_loss": entropy_loss,
                  "max_ratio": ratio.max(), "min_prob": log_prob.exp().min(), "critic_e": critic_e, "critic_i": critic_i}


def adv_mix(adv_e, adv_i, n_step, ext_coef, int_coef, standardize):
    adv = (ext_coef * adv_e + int_coef * adv_i).reshape(-1, n_step)
    if standardize:
        adv = (adv - adv.mean(dim=1, keepdim=True)) / (adv.std(dim=1, keepdim=True) + 1e-7)
    return adv.reshape(-1, 1)


def new_state(D, N):
    """The learner's persistent statistics: rms_obs, rms_ri and the filter state."""
    return {"rms_obs": RunningMeanStd((D,)), "rms_ri": RunningMeanStd(()), "rewems": np.zeros(N)}


def _forward_out(p, x, continuous):
    """The head outputs [pi logits | v | v_i] / [mu | log_std | v | v_i] as the policy network produces them."""
    h = F.relu(F.linear(nets.head(p, x), p["l.weight"], p["l.bias"]))
    names = ("mu", "log_std", "v", "v_i") if continuous else ("pi", "v", "v_i")
    return torch.cat([F.linear(h, p[f"{n}.weight"], p[f"{n}.bias"]) for n in names], 1)


def learn(params, target_params, pred_params, pred_buffers, batch, hp, rhp, perms, lr, stats_state, opt_state=None):
    """params / target_params / pred_params / pred_buffers: dicts name -> tensor; batch: dict of [N*T, ...] tensors
    (state, next_state, action, reward, done); hp: PPO's learn keys (continuous, A, n_step, gamma, lambda, standardize,
    batch_size, n_epoch, clip_grad_norm, eps_clip, vf_coef, ent_coef); rhp: the RND keys (gamma_i, extrinsic_coeff,
    intrinsic_coeff, obs_normalize, ri_normalize, batch_norm, non_episodic); stats_state: new_state(), updated in place;
    opt_state: a previous learn's.  Everything runs in float64.  Returns post-learn params, predictor params and buffers,
    the optimiser state, both streams' advantages and returns, r_i and the result dict."""
    continuous, A = hp["continuous"], hp["A"]
    dd = lambda t: t.detach().to(torch.float64)
    p = {k: dd(v).clone().requires_grad_(True) for k, v in params.items()}
    q = {k: dd(v).clone().requires_grad_(True) for k, v in pred_params.items()}
    tg = {k: dd(v) for k, v in target_params.items()}
    buf = {k: (v.detach().clone() if v.dtype == torch.int64 else dd(v).clone()) for k, v in pred_buffers.items()}
    opt = torch.optim.Adam(list(p.values()) + list(q.values()), lr=lr)
    if opt_state is not None:
        opt.load_state_dict(opt_state)
    state, next_state, action = dd(batch["state"]), dd(batch["next_state"]), dd(batch["action"])
    reward, done = dd(batch["reward"]).view(-1, 1), dd(batch["done"]).view(-1, 1)
    NT, T = state.shape[0], hp["n_step"]
    N = NT // T
    rms = stats_state["rms_obs"] if rhp["obs_normalize"] else None
    if rms is not None:
        rms.update(next_state.reshape(NT, -1).numpy())
    with torch.no_grad():
        x = normalize(next_state, rms)
        t_all = target(tg, x)
        r_i = rnd_loss(predictor(q, buf, x, rhp["batch_norm"]), t_all)[0].numpy()
    if rhp["ri_normalize"]:
        filt, stats_state["rewems"] = reward_filter(stats_state["rewems"], r_i.reshape(N, T), rhp["gamma_i"])
        stats_state["rms_ri"].update(filt.reshape(-1))
        r_i = r_i / (np.sqrt(stats_state["rms_ri"].var) + 1e-7)
    ri = torch.as_tensor(r_i).view(-1, 1)
    with torch.no_grad():
        out = _forward_out(p, state, continuous)
        nxt = _forward_out(p, next_state, continuous)
        v, v_i, nv, nv_i = out[:, -2:-1], out[:, -1:], nxt[:, -2:-1], nxt[:, -1:]
        log_prob_old = oppo.prepass(p, state, action, next_state, continuous)[2]
    adv_e, ret = oppo.gae(reward, done, v, nv, T, hp["gamma"], hp["lambda"], False)
    done_i = torch.zeros_like(done) if rhp["non_episodic"] else done
    adv_i, ret_i = oppo.gae(ri, done_i, v_i, nv_i, T, rhp["gamma_i"], hp["lambda"], False)
    adv = adv_mix(adv_e, adv_i, T, rhp["extrinsic_coeff"], rhp["intrinsic_coeff"], hp["standardize"])
    keys = ("actor_loss", "critic_loss", "entropy_loss", "max_ratio", "min_prob", "rnd_loss")
    stats = {k: [] for k in keys}
    B = hp["batch_size"]
    for epoch in range(hp["n_epoch"]):
        idxs = np.asarray(perms[epoch])
        for offset in range(0, NT, B):
            idx = torch.as_tensor(idxs[offset:offset + B], dtype=torch.long)
            o = _forward_out(p, state[idx], continuous)
            l_ppo, aux = ppo_loss(o, action[idx], adv[idx], ret[idx], v[idx], ret_i[idx], v_i[idx], log_prob_old[idx], A,
                                  continuous, hp["eps_clip"], hp["vf_coef"], hp["ent_coef"])
            pb = predictor(q, buf, normalize(next_state[idx], rms), rhp["batch_norm"])
            _, l_rnd = rnd_loss(pb, t_all[idx])
            opt.zero_grad(set_to_none=True)
            (l_ppo + l_rnd).backward()
            torch.nn.utils.clip_grad_norm_(list(p.values()), hp["clip_grad_norm"])
            opt.step()
            for k in keys[:5]:
                stats[k].append(aux[k].item())
            stats["rnd_loss"].append(l_rnd.item())
    result = {k: float(np.mean(stats[k])) for k in ("actor_loss", "critic_loss", "entropy_loss", "rnd_loss")}
    result.update(max_ratio=max(stats["max_ratio"]), min_prob=min(stats["min_prob"]), mean_ret=float(ret.mean()),
                  r_i=float(np.mean(r_i)))
    return {"params": {k: v.detach().clone() for k, v in p.items()}, "predictor": {k: v.detach().clone() for k, v in q.items()},
            "buffers": buf, "opt_state": opt.state_dict(), "adv": adv.view(-1), "ret": ret.view(-1), "ret_i": ret_i.view(-1),
            "r_i": torch.as_tensor(r_i), "result": result}
