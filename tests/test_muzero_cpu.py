"""MuZero host-side checks without a GPU: configs, registry and rejections, the value transform, the loss and scaling
gradients against float64 autograd, the targets of hand-built windows, the oracle search on hand-solved trees, and the
support coverage of the built-in configs."""
import math

import numpy as np
import pytest
import torch

from oracle import muzero as om


def test_configs_and_registry():
    from jorldy_b200 import config as cfg
    from jorldy_b200.core.agent import agent_dict
    assert "muzero" in agent_dict
    for env in ("cartpole", "mountaincar"):
        assert f"config.muzero.{env}" in cfg.available()
        c = cfg.load(f"config.muzero.{env}")
        a = c.agent
        assert a["name"] == "muzero" and a["num_simulation"] == 50 and a["num_unroll"] == 5 and a["td_steps"] == 10
        assert a["gamma"] == 0.997 and a["hidden_size"] == 128 and a["latent_size"] == 64
        assert a["value_support"] == 20 and a["reward_support"] == 1 and a["value_loss_coef"] == 0.25
        assert a["alpha"] == 1.0 and a["beta"] == 1.0 and a["batch_size"] == 128 and a["buffer_size"] == 100000
        assert c.optim == {"name": "adam", "lr": 3e-4} and a["clip_grad_norm"] == 5
        assert c.train["update_period"] >= 1 and c.train["run_step"] == 100000


@pytest.mark.parametrize("kw, err", [
    (dict(head="cnn"), NotImplementedError),
    (dict(state_size=(4, 84, 84)), NotImplementedError),
    (dict(action_type="continuous"), ValueError),
    (dict(action_size=19), ValueError),
    (dict(num_unroll=0), ValueError),
    (dict(td_steps=0), ValueError),
    (dict(num_simulation=0), ValueError),
])
def test_rejections(kw, err):
    from jorldy_b200.core import Agent
    args = dict(state_size=4, action_size=2)
    args.update(kw)
    with pytest.raises(err):
        Agent("muzero", **args)


def test_value_transform_round_trip():
    x = torch.cat([torch.linspace(-1000, 1000, 2001, dtype=torch.float64), torch.tensor([0.0, 1e-6, -1e-6, 333.0])])
    np.testing.assert_allclose(om.value_h(om.value_h_inv(x)).numpy(), x.numpy(), rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(om.value_h_inv(om.value_h(x)).numpy(), x.numpy(), rtol=1e-10, atol=1e-9)


@pytest.mark.parametrize("V", [1, 20, 300])
def test_two_hot_matches_an_explicit_loop(V):
    rng = np.random.default_rng(V)
    xs = np.concatenate([rng.normal(0, 50, 64), [0.0, 1e9, -1e9, float(om.value_h_inv(torch.tensor(float(V))))]])
    sup = om.scalar_to_support(torch.as_tensor(xs), V).numpy()
    for i, x in enumerate(xs):
        y = min(max(float(om.value_h(torch.tensor(x, dtype=torch.float64))), -V), V)
        ref = np.zeros(2 * V + 1)
        lo = math.floor(y)
        ref[lo + V] += 1 - (y - lo)
        if lo + V + 1 <= 2 * V:
            ref[lo + V + 1] += y - lo
        np.testing.assert_allclose(sup[i], ref, atol=1e-12)
        assert abs(sup[i].sum() - 1) < 1e-12
    # inside the support the expectation of the two-hot is h(x)
    inside = np.abs(xs) < 1e3
    expect = (sup * np.arange(-V, V + 1)).sum(-1)
    np.testing.assert_allclose(expect[inside], om.value_h(torch.as_tensor(xs[inside])).clamp(-V, V).numpy(), atol=1e-9)


def test_scaling_backward_matches_autograd():
    """The kernel's closed form: dx = dy / s + (d min at the argmin) + (d max at the argmax), constant rows clamped."""
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.normal(size=(6, 16)), np.full((1, 16), 0.3), rng.normal(size=(1, 16)) * 1e-7])
    dy = rng.normal(size=x.shape)
    xt = torch.tensor(x, requires_grad=True)
    (om.scale(xt) * torch.tensor(dy)).sum().backward()
    for i in range(x.shape[0]):
        r, g = x[i], dy[i]
        imn, imx = int(np.argmin(r)), int(np.argmax(r))
        rng_ = r[imx] - r[imn]
        clamped = not rng_ >= 1e-5
        s = 1e-5 if clamped else rng_
        y = (r - r[imn]) / s
        dmn = (g * (-1 if clamped else y - 1)).sum() / s
        dmx = 0.0 if clamped else (g * -y).sum() / s
        dx = g / s
        dx[imn] += dmn
        dx[imx] += dmx
        np.testing.assert_allclose(dx, xt.grad[i].numpy(), rtol=1e-9, atol=1e-6)


def test_loss_gradient_closed_form_matches_autograd():
    """d logits = c_k w_b / B (softmax - target) (times value_loss_coef for the value head)."""
    rng = np.random.default_rng(1)
    B, K, n, A, V, R = 5, 3, 2, 3, 4, 1
    L = K + n + 1
    hp = dict(K=K, n=n, V=V, R=R, gamma=0.9, value_loss_coef=0.25, alpha=1.0, A=A)
    done = np.zeros((B, L))
    done[1, 0] = done[2, 2] = 1
    pol = rng.random((B, L, A))
    batch = dict(reward=rng.normal(size=(B, L)), done=done, root_value=rng.normal(size=(B, L)) * 3,
                 policy=pol / pol.sum(-1, keepdims=True))
    w = rng.random(B)
    pi = torch.tensor(rng.normal(size=(K + 1, B, A)), requires_grad=True)
    v = torch.tensor(rng.normal(size=(K + 1, B, 2 * V + 1)), requires_grad=True)
    r = torch.tensor(rng.normal(size=(K, B, 2 * R + 1)), requires_grad=True)
    total, stats, _ = om.loss(pi, v, r, batch, w, hp)
    total.backward()
    z, u, absorbing = om.targets(batch["reward"], done, batch["root_value"], K, n, 0.9)
    for k in range(K + 1):
        c = (1.0 if k == 0 else 1.0 / K) * w / B
        tv = om.scalar_to_support(torch.as_tensor(z[:, k]), V).numpy()
        np.testing.assert_allclose(v.grad[k].numpy(), 0.25 * c[:, None] * (torch.softmax(v[k], -1).detach().numpy() - tv),
                                   atol=1e-12)
        tp = batch["policy"][:, k] * (~absorbing[:, k])[:, None]
        cp = c * (~absorbing[:, k])
        np.testing.assert_allclose(pi.grad[k].numpy(), cp[:, None] * (torch.softmax(pi[k], -1).detach().numpy() - tp),
                                   atol=1e-12)
        if k > 0:
            tr = om.scalar_to_support(torch.as_tensor(u[:, k]), R).numpy()
            np.testing.assert_allclose(r.grad[k - 1].numpy(), c[:, None] * (torch.softmax(r[k - 1], -1).detach().numpy() - tr),
                                       atol=1e-12)
    assert abs(stats["loss"] - (stats["value_loss"] + stats["reward_loss"] + stats["policy_loss"])) < 1e-12


def test_targets_of_hand_built_windows():
    K, n, g = 2, 2, 0.5
    reward = np.array([[1.0, 2.0, 3.0, 4.0, 5.0], [1.0, 2.0, 3.0, 4.0, 5.0], [1.0, 2.0, 3.0, 4.0, 5.0]])
    rv = np.array([[10.0, 20.0, 30.0, 40.0, 50.0]] * 3)
    done = np.array([[0, 0, 0, 0, 0], [0, 1, 0, 0, 0], [1, 0, 0, 0, 0]], dtype=np.float64)
    z, u, ab = om.targets(reward, done, rv, K, n, g)
    # no done: z_k = r_k + g r_{k+1} + g^2 nu_{k+2}
    np.testing.assert_allclose(z[0], [1 + 0.5 * 2 + 0.25 * 30, 2 + 0.5 * 3 + 0.25 * 40, 3 + 0.5 * 4 + 0.25 * 50])
    np.testing.assert_allclose(u[0], [0, 1, 2])
    # done at step 1: z_0 = r_0 + g r_1 (cut), z_1 = r_1, position 2 absorbing; the terminal reward r_1 is a target
    np.testing.assert_allclose(z[1], [1 + 0.5 * 2, 2, 0])
    np.testing.assert_allclose(u[1], [0, 1, 2])
    assert ab[1].tolist() == [False, False, True]
    # done at step 0: z_0 = r_0; positions 1, 2 absorbing; the reward into position 2 follows an absorbing position
    np.testing.assert_allclose(z[2], [1, 0, 0])
    np.testing.assert_allclose(u[2], [0, 1, 0])
    assert ab[2].tolist() == [False, True, True]


def _scripted(values, rewards, pis, V=5, R=5):
    """A model whose simulation j returns value values[j], reward rewards[j] and policy logits pis[j] (logits whose
    support expectation is h of the scalar, so support_to_scalar returns it)."""
    def logits(x, W):
        t = om.scalar_to_support(torch.tensor([float(x)]), W)[0]
        return torch.log(t.clamp(min=1e-300))

    def model(sim, latent, a):
        return latent, np.asarray(pis[sim], dtype=np.float64), logits(values[sim], V), logits(rewards[sim], R)
    return model


def test_oracle_search_first_simulation_ties_at_zero_visits_and_backs_up():
    """At parent N = 0 every exploration term is 0 (sqrt(0)), so the first simulation takes action 0 whatever the
    priors.  The second sees root edge 0 at Q = 0.5 + 2 = 2.5 (the bounds are equal, so Q is not normalised), which beats
    the exploration terms, and expands node 1's action 0 (uniform priors tie -> lowest index)."""
    A, S, g = 3, 2, 1.0
    model = _scripted([2.0, 1.0], [0.5, 0.0], [[0, 0, 0], [0, 0, 0]])
    t, a, pi, rv = om.search(np.log([0.2, 0.5, 0.3]), None, model, A, S, g, 5, 5)
    assert t.n[0].tolist() == [2, 0, 0] and t.n[1].tolist() == [1, 0, 0] and t.child[1, 0] == 2
    np.testing.assert_allclose(pi, [1, 0, 0])
    assert abs(t.w[0, 0] - 3.0) < 1e-9 and abs(t.r[0, 0] - 0.5) < 1e-9 and abs(t.w[1, 0] - 1.0) < 1e-9
    assert abs(rv - 2.0) < 1e-9 and abs(t.qmin - 1.0) < 1e-9 and abs(t.qmax - 2.5) < 1e-9
    assert a == 0


def test_oracle_search_two_simulations_by_hand():
    """Uniform priors over 2 actions, gamma 1.  Sim 1 expands action 0 (tie -> lowest) with r = 0, v = 1.  Sim 2 at the
    root (parent N = 1): action 0 scores q = (1 - 1)/(1 - 1)... the bounds are equal, so q stays 1, plus pb/2; action 1
    (unvisited) scores pb: pb = (log((1 + c2 + 1) / c2) + 1.25) * 1 * 0.5, so 1 + pb/2 > pb and action 0 is taken
    again, expanding its child's action 0."""
    A, S = 2, 2
    model = _scripted([1.0, 3.0], [0.0, 0.0], [[0, 0], [0, 0]])
    t, a, pi, rv = om.search(np.zeros(2), None, model, A, S, 1.0, 5, 5)
    assert t.n[0].tolist() == [2, 0] and t.n[1].tolist() == [1, 0] and t.child[1, 0] == 2
    np.testing.assert_allclose(t.w[0, 0], 1.0 + 3.0)
    np.testing.assert_allclose(rv, 2.0)
    assert a == 0 and abs(t.qmin - 1.0) < 1e-9 and abs(t.qmax - 3.0) < 1e-9


def test_oracle_action_sampling():
    t = om.Tree(3, 4)
    t.n[0] = [1, 0, 3]
    t.w[0] = [1.0, 0.0, 3.0]
    assert t.act(1.0, False)[0] == 2
    assert t.act(1.0, True, 1.0, 0.0)[0] == 0 and t.act(1.0, True, 1.0, 0.26)[0] == 2
    assert t.act(1.0, True, 0.5, 0.09)[0] == 0 and t.act(1.0, True, 0.5, 0.11)[0] == 2


@pytest.mark.parametrize("env", ["cartpole", "mountaincar"])
def test_supports_cover_the_largest_targets(env):
    """CartPole's rewards are 0.1 and -1, MountainCar's -1 per step: |z| <= max|r| / (1 - gamma), |r| <= max|r|."""
    from jorldy_b200 import config as cfg
    a = cfg.load(f"config.muzero.{env}").agent
    z_max = 1.0 / (1.0 - a["gamma"])
    assert float(om.value_h(torch.tensor(z_max, dtype=torch.float64))) <= a["value_support"]
    assert float(om.value_h(torch.tensor(1.0, dtype=torch.float64))) <= a["reward_support"]
