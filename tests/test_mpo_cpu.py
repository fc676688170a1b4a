"""MPO without a GPU: the configs, the constructor's rejections, the float64 oracle's closed-form gradients against
autograd, and the Retrace targets against windows computed by hand."""
import math

import numpy as np
import pytest
import torch

from jorldy_b200 import config
from oracle import mpo as om

EPS = (0.01, 0.01, 5e-5)
GAMMA = 0.9


# ------------------------------------------------------------------------------------------------------------ configs
def test_configs():
    names = [f"config.mpo.{e}" for e in ("cartpole", "mountaincar", "pendulum", "mujoco")]
    assert all(n in config.available() for n in names)
    for n in names:
        c = config.load(n)
        a = c.agent
        cont = n.endswith(("pendulum", "mujoco"))
        assert a["name"] == "mpo"
        assert (a["actor"], a["critic"]) == (("continuous_policy", "continuous_q_network") if cont else
                                             ("discrete_policy", "discrete_q_network"))
        assert (a["hidden_size"], a["gamma"], a["n_step"], a["batch_size"]) == (512, 0.99, 8, 64)
        assert (a["critic_loss_type"], a["num_sample"], a["target_update_period"], a["clip_grad_norm"]) == ("retrace", 30, 100, 1.0)
        assert (a["eta"], a["alpha_mu"], a["alpha_sigma"], a["min_eta"]) == (1.0, 1.0, 1.0, 1e-8)
        assert c.optim == dict(name="adam", lr=3e-4)
        sac = config.load("config.sac." + ("cartpole" if n.endswith("mountaincar") else n.split(".")[-1]))
        assert (a["buffer_size"], a["start_train_step"]) == (sac.agent["buffer_size"], sac.agent["start_train_step"])
        if not n.endswith("mountaincar"):
            assert c.train == sac.train
    with pytest.raises(ImportError):
        config.load("config.mpo.atari")


@pytest.mark.parametrize("kwargs, exc", [
    (dict(critic_loss_type="td_lambda"), ValueError),
    (dict(n_step=0), ValueError),
    (dict(n_step=33), ValueError),
    (dict(actor="continuous_policy", critic="continuous_q_network", num_sample=65), ValueError),
    (dict(actor="continuous_policy", critic="continuous_q_network", num_sample=0), ValueError),
    (dict(action_size=19), ValueError),
    (dict(actor="continuous_policy", critic="continuous_q_network", action_size=9), ValueError),
    (dict(actor="discrete_policy", critic="continuous_q_network"), ValueError),
    (dict(actor="deterministic_policy", critic="continuous_q_network"), ValueError),
    (dict(head="cnn"), NotImplementedError),
])
def test_constructor_rejections(kwargs, exc):
    from jorldy_b200.core.agent.mpo import MPO
    args = dict(state_size=4, action_size=2)
    args.update(kwargs)
    with pytest.raises(exc):
        MPO(**args)


# ------------------------------------------------------------------------------------------ closed-form gradients
def _policy_inputs(rs, S, A, K, continuous, eta=0.7):
    nout = 2 * A if continuous else A
    t = lambda *s: torch.tensor(rs.standard_normal(s), dtype=torch.float64)
    tout = t(S, nout)
    out = tout + 0.3 * t(S, nout)
    if continuous:
        out[::5, 0] = 6.0                                   # clamped mu rows
        tq, z = t(S, K), t(S, K, A)
    else:
        tq, z = t(S, A), None
    mult = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (eta, 1.3, 0.4)]
    return out.requires_grad_(True), tout, tq, z, mult


@pytest.mark.parametrize("continuous, A", [(False, 2), (False, 18), (True, 3), (True, 8)])
def test_policy_closed_form_matches_autograd(continuous, A):
    rs = np.random.RandomState(A)
    out, tout, tq, z, mult = _policy_inputs(rs, 24, A, 30, continuous)
    loss, _ = om.policy_loss(out, tout, tq, z, *mult, EPS, A, continuous)
    for m in mult:
        m.grad = torch.zeros_like(m)
    loss.backward()
    g, dmult = om.policy_closed(out.detach(), tout, tq, z, *[m.detach() for m in mult], EPS, A, continuous)
    np.testing.assert_allclose(g.numpy(), out.grad.numpy(), rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(dmult.numpy(), [m.grad.item() for m in mult], rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("continuous", [False, True])
def test_min_eta_is_finite(continuous):
    rs = np.random.RandomState(3)
    out, tout, tq, z, mult = _policy_inputs(rs, 16, 3, 30, continuous, eta=1e-8)
    loss, aux = om.policy_loss(out, tout, tq, z, *mult, EPS, 3, continuous)
    g, dmult = om.policy_closed(out.detach(), tout, tq, z, *[m.detach() for m in mult], EPS, 3, continuous)
    assert torch.isfinite(loss) and torch.isfinite(g).all() and torch.isfinite(dmult).all()


def test_critic_target_closed_form():
    """d mean (Q - Qret)^2 / d Q = 2 (Q - Qret) / (B n), the gradient jb_mpo_critic_target writes."""
    q = torch.randn(3, 4, dtype=torch.float64, requires_grad=True)
    qret = torch.randn(3, 4, dtype=torch.float64)
    ((q - qret) ** 2).mean().backward()
    np.testing.assert_allclose(q.grad.numpy(), (2 * (q - qret) / 12).detach().numpy(), rtol=1e-12)


# --------------------------------------------------------------------------------------------------------- Retrace
def _t(x):
    return torch.tensor([x], dtype=torch.float64)


def _window(done, c):
    """A 3-step window with V'_1..3 = (1, 2, 3), Q'(s_1, a_1) = 0.5, Q'(s_2, a_2) = 1.5, r = (1, 2, 3); c = (c_1, c_2)."""
    v, qt, r = _t([1.0, 2.0, 3.0]), _t([0.5, 1.5, 0.0]), _t([1.0, 2.0, 3.0])
    return om.retrace(v, _t([c[0], c[1], 0.0]), qt, r, _t(done), GAMMA)[0].numpy()


def test_retrace_hand_computed():
    g = GAMMA
    # no done, c = (0.5, 0.25)
    q2 = 3 + g * 3
    q1 = 2 + g * (2 + 0.25 * (q2 - 1.5))
    q0 = 1 + g * (1 + 0.5 * (q1 - 0.5))
    np.testing.assert_allclose(_window([0, 0, 0], (0.5, 0.25)), [q0, q1, q2], rtol=1e-12)
    # done mid-window (d_1 = 1): Qret_1 = r_1, and Qret_0 still bootstraps through s_1
    q2 = 3 + g * 3
    q1 = 2.0
    q0 = 1 + g * (1 + 0.5 * (q1 - 0.5))
    np.testing.assert_allclose(_window([0, 1, 0], (0.5, 0.25)), [q0, q1, q2], rtol=1e-12)
    # done at the last step: Qret_2 = r_2
    q2 = 3.0
    q1 = 2 + g * (2 + 0.25 * (q2 - 1.5))
    q0 = 1 + g * (1 + 0.5 * (q1 - 0.5))
    np.testing.assert_allclose(_window([0, 0, 1], (0.5, 0.25)), [q0, q1, q2], rtol=1e-12)


def _targets(rs, B, n, A, ratio_shift=None, continuous=False, K=4):
    t = lambda *s: torch.tensor(rs.standard_normal(s), dtype=torch.float64)
    if continuous:
        tout, tq = t(B, n + 1, 2 * A), t(B, n + 1, K + 1)
        action = torch.tanh(t(B, n, A))
    else:
        tout, tq = t(B, n + 1, A), t(B, n + 1, A)
        action = torch.tensor(rs.randint(0, A, (B, n)))
    lp = om.logp(tout[:, :n], action, A, continuous)
    log_mu = lp - ratio_shift if ratio_shift is not None else t(B, n)
    reward = t(B, n)
    done = torch.tensor((rs.uniform(size=(B, n)) < 0.2).astype(np.float64))
    return tout, tq, action, log_mu, reward, done


def test_c_clipped_at_one_and_unrolled():
    """Every ratio pi'/mu above 1: c = 1 throughout, and Qret equals the recursion unrolled by hand."""
    rs = np.random.RandomState(0)
    B, n, A = 3, 4, 3
    tout, tq, action, log_mu, r, d = _targets(rs, B, n, A, ratio_shift=0.7)
    qret = om.critic_target(tout, tq, action, log_mu, r, d, GAMMA, A, False)
    v = (torch.softmax(tout, -1) * tq).sum(-1)                      # V'_0..n
    qa = tq[:, :n].gather(-1, action.unsqueeze(-1)).squeeze(-1)      # Q'(s_t, a_t)
    for b in range(B):
        exp = [0.0] * n
        exp[n - 1] = r[b, n - 1] + GAMMA * (1 - d[b, n - 1]) * v[b, n]
        for t in range(n - 2, -1, -1):
            exp[t] = r[b, t] + GAMMA * (1 - d[b, t]) * (v[b, t + 1] + 1.0 * (exp[t + 1] - qa[b, t + 1]))
        np.testing.assert_allclose(qret[b].numpy(), np.array([float(x) for x in exp]), rtol=1e-12)
    # the clip itself: c_t is exactly 1 where the ratio is exp(0.7)
    lp = om.logp(tout[:, 1:n], action[:, 1:], A, False)
    assert torch.all(torch.clamp(torch.exp(lp - log_mu[:, 1:]), max=1.0) == 1.0)


@pytest.mark.parametrize("continuous", [False, True])
def test_one_step_td_is_retrace_with_zero_c(continuous):
    rs = np.random.RandomState(1)
    B, n, A = 4, 5, 3
    tout, tq, action, log_mu, r, d = _targets(rs, B, n, A, continuous=continuous)
    td = om.critic_target(tout, tq, action, log_mu, r, d, GAMMA, A, continuous, use_retrace=False)
    if continuous:
        v = tq[:, 1:, :-1].mean(-1)
    else:
        v = (torch.softmax(tout, -1) * tq)[:, 1:].sum(-1)
    zero = torch.zeros(B, n, dtype=torch.float64)
    np.testing.assert_allclose(td.numpy(), om.retrace(v, zero, zero, r, d, GAMMA).numpy(), rtol=1e-12)
    np.testing.assert_allclose(td.numpy(), (r + GAMMA * (1 - d) * v).numpy(), rtol=1e-12)


def test_n1_is_one_step_td():
    rs = np.random.RandomState(2)
    B, A = 6, 2
    tout, tq, action, log_mu, r, d = _targets(rs, B, 1, A)
    qret = om.critic_target(tout, tq, action, log_mu, r, d, GAMMA, A, False)
    v1 = (torch.softmax(tout[:, 1], -1) * tq[:, 1]).sum(-1)
    np.testing.assert_allclose(qret[:, 0].numpy(), (r[:, 0] + GAMMA * (1 - d[:, 0]) * v1).numpy(), rtol=1e-12)


def test_logp_matches_torch_distributions():
    rs = np.random.RandomState(4)
    A = 3
    out = torch.tensor(rs.standard_normal((5, 2 * A)))
    a = torch.tanh(torch.tensor(rs.standard_normal((5, A))))
    mu, ls = out[:, :A].clamp(-5, 5), torch.tanh(out[:, A:])
    ref = torch.distributions.Normal(mu, ls.exp()).log_prob(torch.atanh(a.clamp(-1 + 1e-7, 1 - 1e-7))).sum(-1)
    np.testing.assert_allclose(om.logp(out, a, A, True).numpy(), ref.numpy(), rtol=1e-12)
    logits = torch.tensor(rs.standard_normal((5, 4)))
    ai = torch.tensor(rs.randint(0, 4, 5))
    ref = torch.distributions.Categorical(logits=logits).log_prob(ai)
    np.testing.assert_allclose(om.logp(logits, ai, 4, False).numpy(), ref.numpy(), rtol=1e-12)
    assert math.isfinite(float(om.logp(out, torch.ones(5, A), A, True).sum()))
