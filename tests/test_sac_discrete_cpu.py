"""CPU checks of the discrete-action SAC: its two built-in configs, and the closed-form gradients the kernels implement
(oracle/sac_discrete.py) against float64 autograd, including rows whose logits lie 40 apart and rows of equal logits."""
import math

import numpy as np
import pytest
import torch

from oracle import sac_discrete as osd


def test_sac_discrete_configs():
    from jorldy_b200 import config as cfg
    paths = [p for p in cfg.available() if p.split(".")[1] == "sac_discrete"]
    assert sorted(paths) == ["config.sac_discrete.atari", "config.sac_discrete.cartpole"]
    cp = cfg.load("config.sac_discrete.cartpole")
    ref = cfg.load("config.sac.cartpole")
    assert cp.env == dict(ref.env, action_type="discrete")
    assert cp.agent == dict(ref.agent, actor="discrete_policy", critic="discrete_q_network")
    assert cp.optim == ref.optim and cp.train == ref.train
    at = cfg.load("config.sac_discrete.atari")
    assert at.agent == dict(name="sac", actor="discrete_policy", critic="discrete_q_network", head="cnn",
                            use_dynamic_alpha=True, gamma=0.99, tau=5e-3, buffer_size=1_000_000, batch_size=64,
                            start_train_step=20000)
    assert at.optim == dict(actor="adam", critic="adam", alpha="adam", actor_lr=3e-4, critic_lr=3e-4, alpha_lr=3e-4)
    assert at.env == cfg.load("config.ppo.atari").env and "name" not in at.env
    assert at.train["update_period"] == 4 and at.train["num_workers"] == 16
    assert at.train["run_step"] == cfg._TRAIN_ATARI["run_step"]


def _logits(rs, B, A):
    z = rs.standard_normal((B, A)) * 3.0
    z[0] = 0.0                          # equal logits
    z[1, :] = -20.0
    z[1, 0] = 20.0                      # 40 apart
    if A > 2:
        z[2, 1] = z[2, 0] + 40.0
    return torch.from_numpy(z)


@pytest.mark.parametrize("A", [2, 4, 18])
@pytest.mark.parametrize("alpha", [0.0, 0.37])
def test_closed_form_dz_matches_autograd(A, alpha):
    rs = np.random.RandomState(A)
    B = 7
    z = _logits(rs, B, A).requires_grad_(True)
    q1, q2 = torch.from_numpy(rs.standard_normal((B, A))), torch.from_numpy(rs.standard_normal((B, A)))
    q2[3] = q1[3]                       # ties in min(q1, q2)
    loss = osd.actor_loss(z, q1, q2, alpha)
    loss.backward()
    dz, st = osd.actor_closed(z.detach(), q1, q2, alpha, osd.target_entropy(A))
    np.testing.assert_allclose(dz.numpy(), z.grad.numpy(), rtol=1e-12, atol=1e-15)
    assert abs(st["actor_loss"] - loss.item()) < 1e-12
    assert abs(osd.target_entropy(A) - 0.98 * math.log(A)) < 1e-15
    assert abs(st["entropy_gap"] - (st["entropy"] - 0.98 * math.log(A))) < 1e-12
    # equal logits: pi uniform, entropy ln A; the 40-apart row is numerically one-hot and its gradient is finite
    lp0 = torch.log_softmax(z.detach()[0], -1)
    np.testing.assert_allclose(lp0.numpy(), np.full(A, -math.log(A)), rtol=0, atol=1e-15)
    assert torch.isfinite(dz).all()


@pytest.mark.parametrize("A", [2, 4, 18])
def test_closed_form_dq_matches_autograd(A):
    rs = np.random.RandomState(100 + A)
    B = 9
    q1 = torch.from_numpy(rs.standard_normal((B, A))).requires_grad_(True)
    q2 = torch.from_numpy(rs.standard_normal((B, A))).requires_grad_(True)
    action = torch.from_numpy(rs.randint(A, size=B))
    nz = _logits(rs, B, A)
    nq1, nq2 = torch.from_numpy(rs.standard_normal((B, A))), torch.from_numpy(rs.standard_normal((B, A)))
    r, d = torch.from_numpy(rs.standard_normal(B)), torch.from_numpy((rs.uniform(size=B) < 0.3).astype(np.float64))
    y = osd.target(nz, nq1, nq2, r, d, 0.99, 0.2)
    # the target by its definition, one row at a time
    for b in range(B):
        p = torch.softmax(nz[b], -1)
        v = sum(p[k] * (min(nq1[b, k], nq2[b, k]) - 0.2 * torch.log(p[k])) for k in range(A) if p[k] > 0)
        assert abs(y[b].item() - (r[b] + (1 - d[b]) * 0.99 * v).item()) < 1e-9
    l1, l2, dq1, dq2 = osd.critic_closed(q1.detach(), q2.detach(), action, y)
    for q, l, dq in ((q1, l1, dq1), (q2, l2, dq2)):
        loss = torch.nn.functional.mse_loss(q.gather(1, action.view(B, 1)).view(B), y)
        loss.backward()
        assert abs(loss.item() - l.item()) < 1e-12
        np.testing.assert_allclose(dq.numpy(), q.grad.numpy(), rtol=1e-12, atol=1e-15)


def test_inverse_cdf_and_greedy():
    z = torch.tensor([[0.0, 0.0, 0.0], [0.0, math.log(3.0), 0.0], [5.0, 5.0, -1.0]], dtype=torch.float64)
    u = torch.tensor([0.5, 0.3, 0.999999], dtype=torch.float64)
    assert osd.act(z, u).tolist() == [1, 1, 2]
    assert osd.act(z).tolist() == [0, 1, 0]
