"""RND-PPO without a GPU: the configs, the constructor's rejections, the closed-form gradients of the two-critic PPO loss
and of the distillation loss against float64 autograd, the advantage mix against numpy, and the oracle networks against
torch modules written from the spec (BatchNorm in training mode with its running buffers, ELU)."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import rnd_ppo as orr


# ------------------------------------------------------------------------------------------------------- configs
@pytest.mark.parametrize("env", ["cartpole", "mountaincar", "pendulum", "mujoco", "atari"])
def test_configs_are_ppo_rows_plus_the_rnd_keys(env):
    from jorldy_b200 import config
    d, ppo = config.load(f"config.rnd_ppo.{env}"), config.load(f"config.ppo.{env}")
    a = dict(d.agent)
    assert a.pop("name") == "rnd_ppo"
    rnd = {k: a.pop(k) for k in ("rnd_network", "gamma_i", "extrinsic_coeff", "intrinsic_coeff", "obs_normalize",
                                 "ri_normalize", "batch_norm", "non_episodic")}
    frames = env == "atari"
    assert rnd == dict(rnd_network="rnd_cnn" if frames else "rnd_mlp", gamma_i=0.99, extrinsic_coeff=2.0,
                       intrinsic_coeff=1.0, obs_normalize=not frames, ri_normalize=True, batch_norm=True,
                       non_episodic=True)
    assert a == {k: v for k, v in ppo.agent.items() if k != "name"}
    assert d.optim == ppo.optim and d.train == ppo.train and d.env == ppo.env
    assert f"config.rnd_ppo.{env}" in config.available()


def test_the_agent_factory_knows_rnd_ppo():
    from jorldy_b200.core.agent import RND_PPO, agent_dict
    assert agent_dict["rnd_ppo"] is RND_PPO


@pytest.mark.parametrize("kw,match", [
    (dict(rnd_network="rnd_icm"), "unknown rnd_network"),
    (dict(rnd_network="rnd_cnn", obs_normalize=False), "takes the observations of head='cnn', got head='mlp'"),
    (dict(rnd_network="rnd_mlp", head="cnn"), "takes the observations of head='mlp', got head='cnn'"),
    (dict(rnd_network="rnd_cnn", head="cnn", obs_normalize=True), "obs_normalize=False"),
    (dict(network="discrete_q_network"), "has no two-value variant"),
    (dict(action_size=19), "take 1 to 18 actions, got action_size=19"),
    (dict(action_size=9, network="continuous_policy_value"), "take 1 to 8 actions, got action_size=9"),
])
def test_constructor_rejects_bad_settings(kw, match):
    """The checks run before the agent allocates anything, so they need no GPU."""
    from jorldy_b200.core.agent.rnd_ppo import RND_PPO
    kw = dict(kw)
    A = kw.pop("action_size", 2)
    with pytest.raises(ValueError, match=re.escape(match)):
        RND_PPO([4, 84, 84] if kw.get("head") == "cnn" else 4, A, **kw)


def test_one_row_minibatch_with_batch_norm_is_rejected():
    from jorldy_b200.core.agent.rnd_ppo import RND_PPO
    agent = RND_PPO.__new__(RND_PPO)
    agent.batch_norm, agent.batch_size = True, 32
    with pytest.raises(ValueError, match=r"RND-PPO with batch_norm.*batch_size=32.*rollout of 65 rows"):
        agent._check_batch(65)
    agent._check_batch(64)
    agent.batch_size = 1
    with pytest.raises(ValueError, match="batch_size=1"):
        agent._check_batch(64)
    agent.batch_norm = False
    agent._check_batch(65)


# ------------------------------------------------------------------------------------------- closed-form gradients
def _ppo_closed_form(out, action, adv, ret, v_old, ret_i, v_i_old, lpo, A, cont, eps, vf, ent):
    """d loss / d out of the two-critic PPO loss in closed form, as csrc/rnd.cu computes it (jbppo::row for the policy
    and v columns, and the same clipped pair for v_i)."""
    B = out.shape[0]
    npol = 2 * A if cont else A
    g = torch.zeros_like(out)
    if cont:
        mu_raw, ls_raw = out[:, :A], out[:, A:2 * A]
        mu, ls = mu_raw.clamp(-5, 5), torch.tanh(ls_raw)
        sd = ls.exp()
        z = torch.atanh(action.clamp(-1 + 1e-7, 1 - 1e-7))
        logp = -(z - mu) ** 2 / (2 * sd ** 2) - sd.log() - 0.5 * np.log(2 * np.pi)
        ratio = (logp - lpo).sum(1, keepdim=True).exp()
    else:
        lsm = F.log_softmax(out[:, :A], 1)
        p = lsm.exp()
        logp = lsm.gather(1, action.long().view(-1, 1))
        ratio = (logp - lpo).exp()
    s1, s2 = ratio * adv, ratio.clamp(1 - eps, 1 + eps) * adv
    inr = ((ratio >= 1 - eps) & (ratio <= 1 + eps)).double()
    gr = torch.where(s1 < s2, adv, torch.where(s1 > s2, adv * inr, 0.5 * adv + 0.5 * adv * inr))
    dlogp = -gr * ratio / B
    if cont:
        d = z - mu
        dmu = dlogp * d / sd ** 2 * ((mu_raw >= -5) & (mu_raw <= 5)).double()
        dsd = dlogp * (d ** 2 / sd ** 3 - 1 / sd) + (-ent / B / A) / sd
        g[:, :A], g[:, A:2 * A] = dmu, dsd * sd * (1 - ls ** 2)
    else:
        onehot = F.one_hot(action.long().view(-1), A).double()
        H = -(p * lsm).sum(1, keepdim=True)                  # d H / d logit_j = -p_j (log p_j + H)
        g[:, :A] = dlogp * (onehot - p) + (ent / B) * p * (lsm + H)
    for col, vo, r in ((npol, v_old, ret), (npol + 1, v_i_old, ret_i)):
        v = out[:, col:col + 1]
        vc = vo + (v - vo).clamp(-eps, eps)
        c1, c2 = ((v - r) ** 2).mean(), ((vc - r) ** 2).mean()
        w1 = 1.0 if c1 > c2 else (0.5 if c1 == c2 else 0.0)
        inc = ((v - vo >= -eps) & (v - vo <= eps)).double()
        g[:, col:col + 1] = vf * (w1 * 2 * (v - r) / B + (1 - w1) * 2 * (vc - r) * inc / B)
    return g


@pytest.mark.parametrize("cont,A", [(False, 2), (False, 18), (True, 1), (True, 8)])
@pytest.mark.parametrize("regime", ["mixed", "tie"])
def test_two_critic_loss_closed_form_matches_autograd(cont, A, regime):
    rs = np.random.RandomState(A + 7 * cont + (50 if regime == "tie" else 0))
    B, eps = 33, 0.1
    nout = 2 * A + 2 if cont else A + 2
    out = torch.tensor(rs.standard_normal((B, nout)), requires_grad=True)
    action = torch.tensor(rs.uniform(-0.9, 0.9, (B, A)) if cont else rs.randint(0, A, (B, 1)).astype(np.float64))
    col = lambda k: out.detach()[:, k:k + 1]
    npol = 2 * A if cont else A
    if regime == "tie":        # every value inside its clip: v_clip = v and both critics' pairs tie
        v_old, v_i_old = col(npol) + 0.01, col(npol + 1) - 0.02
    else:
        v_old, v_i_old = col(npol) + torch.tensor(rs.uniform(-0.3, 0.3, (B, 1))), col(npol + 1) + torch.tensor(
            rs.uniform(-0.3, 0.3, (B, 1)))
    ret, ret_i = torch.tensor(rs.standard_normal((B, 1))), torch.tensor(rs.standard_normal((B, 1)))
    adv = torch.tensor(rs.standard_normal((B, 1)))
    lpo = torch.tensor(rs.uniform(-2, -0.1, (B, A if cont else 1)))
    loss, aux = orr.ppo_loss(out, action, adv, ret, v_old, ret_i, v_i_old, lpo, A, cont, eps, 0.5, 0.01)
    loss.backward()
    if regime == "tie":
        assert aux["critic_e"].item() == F.mse_loss(col(npol), ret).item()
    g = _ppo_closed_form(out.detach(), action, adv, ret, v_old, ret_i, v_i_old, lpo, A, cont, eps, 0.5, 0.01)
    torch.testing.assert_close(out.grad, g, rtol=1e-9, atol=1e-12)


def test_distillation_loss_closed_form_matches_autograd():
    rs = np.random.RandomState(1)
    p = torch.tensor(rs.standard_normal((37, 256)), requires_grad=True)
    t = torch.tensor(rs.standard_normal((37, 256)))
    r_i, loss = orr.rnd_loss(p, t)
    loss.backward()
    torch.testing.assert_close(p.grad, orr.closed_form(p.detach(), t), rtol=1e-12, atol=1e-15)
    torch.testing.assert_close(r_i, ((p.detach() - t) ** 2).sum(1) / 256, rtol=1e-12, atol=0)


@pytest.mark.parametrize("standardize", [False, True])
def test_advantage_mix_matches_numpy(standardize):
    rs = np.random.RandomState(4)
    N, T = 5, 9
    ae, ai = rs.standard_normal((N * T, 1)), rs.standard_normal((N * T, 1))
    got = orr.adv_mix(torch.tensor(ae), torch.tensor(ai), T, 2.0, 1.0, standardize).numpy()
    exp = (2.0 * ae + ai).reshape(N, T)
    if standardize:
        exp = (exp - exp.mean(1, keepdims=True)) / (exp.std(1, ddof=1, keepdims=True) + 1e-7)
    np.testing.assert_allclose(got.reshape(N, T), exp, rtol=1e-12, atol=1e-14)


# ------------------------------------------------------------------------------------------------ the networks
class SpecRND(torch.nn.Module):
    """The RND networks of the spec as torch modules (float64): target fc2(elu(fc1)), predictor
    fc3(elu(fc2(elu(bn1(fc1)))))."""

    def __init__(self, D):
        super().__init__()
        self.t1, self.t2 = torch.nn.Linear(D, 256), torch.nn.Linear(256, 256)
        self.fc1, self.bn1 = torch.nn.Linear(D, 256), torch.nn.BatchNorm1d(256)
        self.fc2, self.fc3 = torch.nn.Linear(256, 256), torch.nn.Linear(256, 256)

    def forward(self, x):
        return self.t2(F.elu(self.t1(x))), self.fc3(F.elu(self.fc2(F.elu(self.bn1(self.fc1(x))))))


def test_oracle_networks_match_the_spec_module_with_batch_norm_buffers():
    torch.manual_seed(0)
    D, B = 11, 65
    m = SpecRND(D).double().train()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    tg = {"fc1.weight": sd["t1.weight"], "fc1.bias": sd["t1.bias"], "fc2.weight": sd["t2.weight"], "fc2.bias": sd["t2.bias"]}
    pr = {k: v for k, v in sd.items() if k.split(".")[0] in ("fc1", "bn1", "fc2", "fc3") and "running" not in k
          and "num_batches" not in k}
    buf = {k: v.clone() for k, v in sd.items() if "running" in k or "num_batches" in k}
    x = torch.randn(B, D, dtype=torch.float64)
    for _ in range(2):                                    # two passes: the running buffers compound
        t_ref, p_ref = m(x)
        torch.testing.assert_close(orr.target(tg, x), t_ref, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(orr.predictor(pr, buf, x), p_ref, rtol=1e-12, atol=1e-12)
    for k, v in m.state_dict().items():
        if k in buf:
            torch.testing.assert_close(buf[k], v, rtol=1e-12, atol=1e-12)
    assert int(buf["bn1.num_batches_tracked"]) == 2
    m.bn1 = torch.nn.Identity()                           # batch_norm=False drops the layer
    torch.testing.assert_close(orr.predictor(pr, {}, x, batch_norm=False), m(x)[1], rtol=1e-12, atol=1e-12)
