"""CPU checks of the quantile agents: their built-in configs, the closed-form quantile Huber gradient the kernel
implements (oracle/quantile.py) against float64 autograd, and the oracle's IQN forward against a plain torch module."""
import math

import numpy as np
import pytest
import torch

from oracle import quantile as oq


def test_quantile_configs():
    from jorldy_b200 import config as cfg
    for agent in ("qrdqn", "iqn"):
        paths = sorted(p for p in cfg.available() if p.split(".")[1] == agent)
        assert paths == [f"config.{agent}.{e}" for e in ("atari", "cartpole", "mountaincar")]
        for env in ("cartpole", "mountaincar", "atari"):
            c, ref = cfg.load(f"config.{agent}.{env}"), cfg.load(f"config.dqn.{env}")
            extra = dict(num_support=200) if agent == "qrdqn" else \
                dict(num_sample=64, embedding_dim=64, sample_min=0.0, sample_max=1.0)
            net = "discrete_q_network" if agent == "qrdqn" else "iqn"
            assert c.agent == dict(ref.agent, name=agent, network=net, **extra), (agent, env)
            assert c.env == ref.env and c.optim == ref.optim and c.train == ref.train
    assert cfg.load("config.iqn.atari").agent["head"] == "cnn"


def _case(rs, B, N, Np):
    theta = torch.from_numpy(rs.standard_normal((B, N)) * 1.5)
    y = torch.from_numpy(rs.standard_normal((B, Np)) * 1.5)
    tau = torch.from_numpy(rs.uniform(size=(B, N)))
    y[0, 0] = theta[0, 0]                          # u exactly 0
    if Np > 1 and N > 1:
        y[0, 1] = theta[0, 1] + 1.0                # |u| = kappa
        y[0, -1] = theta[0, 0] - (1.0 - 1e-9)      # |u| just below kappa
        y[1 % B, 0] = theta[1 % B, 1] + (1.0 + 1e-9)
        tau[0, 0], tau[0, 1] = 0.0, 1.0            # tau at both ends
    return theta, y, tau


@pytest.mark.parametrize("B,N,Np", [(1, 1, 1), (3, 8, 8), (4, 16, 5), (2, 5, 32)])
def test_closed_form_gradient_matches_autograd(B, N, Np):
    rs = np.random.RandomState(B * 100 + N + Np)
    theta, y, tau = _case(rs, B, N, Np)
    t = theta.clone().requires_grad_(True)
    L = oq.loss(t, y, tau)
    L.backward()
    np.testing.assert_allclose(oq.grad_closed(theta, y, tau).numpy(), t.grad.numpy(), rtol=1e-12, atol=1e-15)
    assert abs(oq.per_sample_loss(theta, y, tau).mean().item() - L.item()) < 1e-12
    # shared fractions (QR-DQN's [N] tau) broadcast like per-sample ones
    tq = oq.qr_tau(N)
    t2 = theta.clone().requires_grad_(True)
    oq.loss(t2, y, tq).backward()
    np.testing.assert_allclose(oq.grad_closed(theta, y, tq).numpy(), t2.grad.numpy(), rtol=1e-12, atol=1e-15)


def test_loss_weights_by_the_sign_of_u():
    theta = torch.zeros(1, 1, dtype=torch.float64)
    tau = torch.tensor([[0.2]], dtype=torch.float64)
    over = oq.loss(theta, torch.tensor([[3.0]], dtype=torch.float64), tau).item()      # u > 0: weight tau
    under = oq.loss(theta, torch.tensor([[-3.0]], dtype=torch.float64), tau).item()    # u < 0: weight 1 - tau
    assert abs(over - 0.2 * 2.5) < 1e-15 and abs(under - 0.8 * 2.5) < 1e-15
    assert oq.qr_tau(4).tolist() == [0.125, 0.375, 0.625, 0.875]


def test_targets_take_the_argmax_of_the_mean():
    tn = torch.tensor([[[0.0, 3.0], [1.0, 1.0], [2.0, 1.0]]], dtype=torch.float64)   # means 1.5, 1.0, 1.5
    a, y = oq.targets(tn, torch.tensor([0.5], dtype=torch.float64), torch.tensor([0.0], dtype=torch.float64), 0.5)
    assert a.tolist() == [0] and y.tolist() == [[0.5, 2.0]]
    _, y = oq.targets(tn, torch.tensor([0.5], dtype=torch.float64), torch.tensor([1.0], dtype=torch.float64), 0.5)
    assert y.tolist() == [[0.5, 0.5]]


class _TorchIQN(torch.nn.Module):
    """The IQN of arXiv:1806.06923 as plain torch modules (MLP head)."""

    def __init__(self, D_in, A, H, D_em):
        super().__init__()
        self.D_em = D_em
        self.head = torch.nn.Linear(D_in, H)
        self.sample_embed = torch.nn.Linear(D_em, H)
        self.l = torch.nn.Linear(H, H)
        self.q = torch.nn.Linear(H, A)

    def forward(self, x, tau):
        psi = torch.relu(self.head(x))
        i_pi = torch.arange(self.D_em, dtype=torch.float64) * math.pi
        phi = torch.relu(self.sample_embed(torch.cos(tau.unsqueeze(-1) * i_pi)))
        return self.q(torch.relu(self.l(psi.unsqueeze(1) * phi)))


@pytest.mark.parametrize("N", [1, 8])
def test_oracle_iqn_forward_matches_a_torch_module(N):
    torch.manual_seed(N)
    m = _TorchIQN(5, 3, 16, 8).double()
    p = {("head.l." + k[5:] if k.startswith("head.") else k): v.detach() for k, v in m.state_dict().items()}
    x = torch.randn(4, 5, dtype=torch.float64)
    tau = torch.rand(4, N, dtype=torch.float64)
    want = m(x, tau)
    got = oq.iqn_network(p, x, tau, 8)
    assert got.shape == (4, N, 3)
    np.testing.assert_allclose(got.detach().numpy(), want.detach().numpy(), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(oq.iqn_q(p, x, tau, 8).numpy(), want.detach().mean(1).numpy(), rtol=1e-12, atol=1e-13)
