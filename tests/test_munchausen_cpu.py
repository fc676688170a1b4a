"""CPU checks of the Munchausen agents: their built-in configs, and the float64 oracle (oracle/munchausen.py) the kernels
are tested against: its stable tau logpi against log_softmax, its alpha = 0, tau -> 0 limit against the DQN and IQN
targets, and the clip-then-scale order of the bonus."""
import math

import numpy as np
import pytest
import torch

from oracle import dqn as od
from oracle import munchausen as om
from oracle import quantile as oq

M_KEYS = dict(alpha=0.9, tau=0.03, l_0=-1)


def test_munchausen_configs():
    from jorldy_b200 import config as cfg
    for agent, base in (("m_dqn", "dqn"), ("m_iqn", "iqn")):
        paths = sorted(p for p in cfg.available() if p.split(".")[1] == agent)
        assert paths == [f"config.{agent}.{e}" for e in ("atari", "cartpole", "mountaincar")]
        for env in ("cartpole", "mountaincar", "atari"):
            c, ref = cfg.load(f"config.{agent}.{env}"), cfg.load(f"config.{base}.{env}")
            assert c.agent == dict(ref.agent, name=agent, **M_KEYS), (agent, env)
            assert c.env == ref.env and c.optim == ref.optim and c.train == ref.train
    assert cfg.load("config.m_iqn.atari").agent["head"] == "cnn"
    assert cfg.load("config.m_dqn.cartpole").agent["network"] == "discrete_q_network"


@pytest.mark.parametrize("tau", [0.03, 0.5, 3.0])
def test_stable_tau_logpi_matches_log_softmax(tau):
    rs = np.random.RandomState(int(tau * 100))
    q = torch.from_numpy(rs.standard_normal((64, 18)) * 0.05)      # spreads where log_softmax(q / tau) is itself exact
    want = tau * torch.log_softmax(q / tau, -1)
    np.testing.assert_allclose(om.tau_logpi(q, tau).numpy(), want.numpy(), rtol=1e-12, atol=1e-14)
    # wide spreads: pi underflows, the stable form stays finite and exact on the argmax
    wide = q * 1e4
    t = om.tau_logpi(wide, 0.03)
    assert torch.isfinite(t).all() and (t.max(-1).values == 0).all()
    assert torch.isfinite(om.soft_value(wide, wide, 0.03)).all()


def _separated(rs, B, A):
    """Q rows whose maximum is unique and at least 0.05 above the rest."""
    q = rs.standard_normal((B, A))
    top = q.argmax(1)
    q[np.arange(B), top] = q.max(1) + 0.05
    return torch.from_numpy(q)


def test_alpha_zero_small_tau_is_dqn():
    rs = np.random.RandomState(0)
    B, A, D, H, gamma = 16, 5, 4, 8, 0.99
    p = {"head.l.weight": rs.standard_normal((H, D)), "head.l.bias": rs.standard_normal(H),
         "l.weight": rs.standard_normal((H, H)), "l.bias": rs.standard_normal(H),
         "q.weight": rs.standard_normal((A, H)), "q.bias": rs.standard_normal(A)}
    p = {k: torch.from_numpy(v) for k, v in p.items()}
    tp = {k: v + 0.1 * torch.from_numpy(rs.standard_normal(tuple(v.shape))) for k, v in p.items()}
    batch = {"state": torch.from_numpy(rs.standard_normal((B, D))), "next_state": torch.from_numpy(rs.standard_normal((B, D))),
             "action": torch.from_numpy(rs.randint(A, size=B)), "reward": torch.from_numpy(rs.standard_normal(B)),
             "done": torch.from_numpy((rs.uniform(size=B) < 0.3).astype(np.float64))}
    qn = om.nets.discrete_q_network(tp, batch["next_state"])
    top2 = qn.topk(2, 1).values
    assert ((top2[:, 0] - top2[:, 1]) > 1e-3).all()
    got = om.mdqn_learn(p, tp, batch, dict(gamma=gamma, lr=1e-3, alpha=0.0, tau=1e-6, l_0=-1.0))
    want_y = batch["reward"] + (1 - batch["done"]) * gamma * qn.max(1).values
    assert torch.equal(got["y"], want_y)
    col = {k: batch[k].view(B, 1) for k in ("reward", "done")}
    ref = od.td_learn(p, tp, dict(batch, action=batch["action"].view(B, 1), **col),
                      dict(net="dqn", gamma=gamma, n_step=1, double=False, loss="huber", order="dqn", alpha=0.0,
                           action_size=A), dict(name="adam", lr=1e-3))
    assert abs(got["result"]["loss"] - ref["loss"]) < 1e-12 and got["result"]["max_Q"] == ref["max_Q"]
    for k, g in ref["grads"].items():
        np.testing.assert_allclose(got["grads"][k].numpy(), g.numpy(), rtol=1e-10, atol=1e-14, err_msg=k)


def test_alpha_zero_small_tau_is_iqn():
    rs = np.random.RandomState(1)
    B, A, Np, Nc = 8, 4, 6, 5
    tn = torch.from_numpy(rs.standard_normal((B, A, Np)))
    means = tn.mean(2)
    top = means.argmax(1)
    tn[torch.arange(B), top] += 0.1                                   # a unique argmax of the mean, >= 0.1 clear
    tc = torch.from_numpy(rs.standard_normal((B, A, Nc)))
    a = torch.from_numpy(rs.randint(A, size=B))
    r = torch.from_numpy(rs.standard_normal(B))
    d = torch.from_numpy((rs.uniform(size=B) < 0.3).astype(np.float64))
    y = om.miqn_targets(tc, tn, a, r, d, 0.99, 0.0, 1e-6, -1.0)
    _, want = oq.targets(tn, r, d, 0.99)
    assert torch.equal(y, want)


def test_bonus_clips_then_scales():
    # tau = 1, A = 2, q'(s, .) = (log(e^2 - 1), 0): tau logpi(1|s) = -2 exactly in real arithmetic
    q = torch.tensor([[math.log(math.e ** 2 - 1), 0.0]], dtype=torch.float64)
    a = torch.tensor([1])
    assert abs(om.tau_logpi(q, 1.0)[0, 1].item() + 2.0) < 1e-14
    assert abs(om.bonus(q, a, 0.9, 1.0, -1.0).item() + 0.9) < 1e-14            # 0.9 * clip(-2, -1, 0); scale-then-clip: -1
    q_mid = torch.tensor([[math.log(math.exp(0.5) - 1), 0.0]], dtype=torch.float64)   # tau logpi(1|s) = -0.5
    assert abs(om.bonus(q_mid, a, 0.9, 1.0, -1.0).item() + 0.45) < 1e-14
    assert om.bonus(q, torch.tensor([0]), 0.9, 1.0, -1.0).item() == pytest.approx(0.9 * math.log1p(-math.exp(-2)), abs=1e-14)
