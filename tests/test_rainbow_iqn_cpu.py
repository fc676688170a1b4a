"""CPU checks of Rainbow-IQN: its built-in configs (and Rainbow's, unchanged), the oracle's n-step fold and double-Q
action (oracle/rainbow_iqn.py) against explicit loops, the closed-form IS-weighted gradient the kernel implements against
float64 autograd, and the oracle's network against a plain torch module."""
import math

import numpy as np
import pytest
import torch

from oracle import rainbow_iqn as ori


def test_rainbow_iqn_configs():
    from jorldy_b200 import config as cfg
    paths = sorted(p for p in cfg.available() if p.split(".")[1] == "rainbow_iqn")
    assert paths == [f"config.rainbow_iqn.{e}" for e in ("atari", "cartpole", "mountaincar")]
    iqn_keys = dict(num_sample=64, embedding_dim=64, sample_min=0.0, sample_max=1.0)
    for env in ("cartpole", "mountaincar", "atari"):
        c, ref = cfg.load(f"config.rainbow_iqn.{env}"), cfg.load(f"config.rainbow.{env}")
        want = {k: v for k, v in ref.agent.items() if k not in ("v_min", "v_max", "num_support")}
        assert c.agent == dict(want, name="rainbow_iqn", network="rainbow_iqn", **iqn_keys), env
        assert c.env == ref.env and c.optim == ref.optim and c.train == ref.train
    atari = cfg.load("config.rainbow_iqn.atari")
    assert atari.agent["learn_period"] == 4 and atari.agent["head"] == "cnn" and atari.optim["lr"] == 2.5e-4 / 4
    assert atari.train["run_step"] == 30000000
    # Rainbow's own configs keep their values
    r = cfg.load("config.rainbow.atari")
    assert (r.agent["learn_period"], r.optim["lr"], r.train["run_step"]) == (4, 2.5e-4 / 4, 30000000)
    assert cfg.load("config.rainbow.cartpole").agent["learn_period"] == 2
    assert cfg.load("config.iqn.atari").optim["lr"] == 1e-4


@pytest.mark.parametrize("n", [1, 3, 5])
def test_nstep_fold_matches_an_explicit_loop(n):
    rs = np.random.RandomState(n)
    B, A, N1, N2, gamma = 6, 4, 5, 7, 0.97
    nxt_on = torch.from_numpy(rs.standard_normal((B, N1, A)))
    nxt_tg = torch.from_numpy(rs.standard_normal((B, N2, A)))
    reward = torch.from_numpy(rs.standard_normal((B, n)))
    done = torch.zeros(B, n, dtype=torch.float64)
    done[0, 0] = 1.0                               # done at the first step
    done[1, n // 2] = 1.0                          # ... a middle step
    done[2, n - 1] = 1.0                           # ... the last step
    done[3, :] = 1.0
    a_star, y = ori.targets(nxt_on, nxt_tg, reward, done, gamma)
    for b in range(B):
        means = [float(nxt_on[b, :, a].mean()) for a in range(A)]
        a_b = max(range(A), key=lambda a: (means[a], -a))           # first index of the max
        assert a_star[b].item() == a_b
        for j in range(N2):
            g = float(nxt_tg[b, j, a_b])
            for s in range(n - 1, -1, -1):
                g = float(reward[b, s]) + (1.0 - float(done[b, s])) * gamma * g
            assert abs(y[b, j].item() - g) < 1e-12
    # a done at the first step cuts the bootstrap: y is r_0 on every fraction
    assert torch.all(y[0] == reward[0, 0]) and torch.all(y[3] == reward[3, 0])


def test_double_q_takes_a_star_from_the_online_net_with_first_index_ties():
    on = torch.tensor([[[1.0, 3.0, 3.0], [1.0, 1.0, 1.0]]], dtype=torch.float64)     # means 1, 2, 2: tie -> 1
    tg = torch.tensor([[[9.0, 0.5, 7.0]]], dtype=torch.float64)                     # the target net would pick 0
    z = torch.zeros(1, 1, dtype=torch.float64)
    a_star, y = ori.targets(on, tg, z, z, 0.5)
    assert a_star.tolist() == [1] and y.tolist() == [[0.25]]


@pytest.mark.parametrize("B,N,Np", [(1, 1, 1), (3, 8, 8), (4, 16, 5), (2, 5, 32)])
def test_weighted_closed_form_gradient_matches_autograd(B, N, Np):
    rs = np.random.RandomState(B * 100 + N + Np)
    theta = torch.from_numpy(rs.standard_normal((B, N)) * 1.5)
    y = torch.from_numpy(rs.standard_normal((B, Np)) * 1.5)
    tau = torch.from_numpy(rs.uniform(size=(B, N)))
    y[0, 0] = theta[0, 0]                          # u exactly 0
    if N > 1 and Np > 1:
        y[0, 1] = theta[0, 1] + 1.0                # |u| = kappa
    w = torch.from_numpy(rs.uniform(0.05, 1.0, size=B))
    t = theta.clone().requires_grad_(True)
    L = ori.loss(t, y, tau, w)
    L.backward()
    np.testing.assert_allclose(ori.grad_closed(theta, y, tau, w).numpy(), t.grad.numpy(), rtol=1e-12, atol=1e-15)
    from oracle import quantile as oq
    per = oq.per_sample_loss(theta, y, tau)
    assert abs((w * per).mean().item() - L.item()) < 1e-12
    np.testing.assert_allclose(ori.priorities(theta, y, tau, 0.5).numpy(), per.sqrt().numpy(), rtol=1e-14)


class _TorchRainbowIQN(torch.nn.Module):
    """Rainbow-IQN as plain torch modules (MLP head), with factorised noisy layers y = x (mu + sig eps) + (mu_b + sig_b eps_b)
    in the (in, out) weight layout."""

    def __init__(self, D_in, A, H, D_em):
        super().__init__()
        self.D_em = D_em
        self.noisy = torch.nn.ParameterDict()
        for lt, (i, o) in (("_a1", (H, H)), ("_v1", (H, H)), ("_a2", (H, A)), ("_v2", (H, 1))):
            self.noisy["mu_w" + lt] = torch.nn.Parameter(torch.randn(i, o) / i ** 0.5)
            self.noisy["sig_w" + lt] = torch.nn.Parameter(torch.rand(i, o) * 0.1)
            self.noisy["mu_b" + lt] = torch.nn.Parameter(torch.randn(o) * 0.1)
            self.noisy["sig_b" + lt] = torch.nn.Parameter(torch.rand(o) * 0.1)
        self.head = torch.nn.Linear(D_in, H)
        self.sample_embed = torch.nn.Linear(D_em, H)
        self.l = torch.nn.Linear(H, H)

    def _nl(self, x, lt, eps):
        n = self.noisy
        if eps is None:
            return x @ n["mu_w" + lt] + n["mu_b" + lt]
        fi, fj = (torch.sign(e) * torch.sqrt(torch.abs(e)) for e in eps)
        return x @ (n["mu_w" + lt] + n["sig_w" + lt] * torch.outer(fi, fj)) + (n["mu_b" + lt] + n["sig_b" + lt] * fj)

    def forward(self, x, tau, noise):
        psi = torch.relu(self.head(x))
        i_pi = torch.arange(self.D_em, dtype=torch.float64) * math.pi
        phi = torch.relu(self.sample_embed(torch.cos(tau.unsqueeze(-1) * i_pi)))
        f = torch.relu(self.l(psi.unsqueeze(1) * phi))
        na1, nv1, na2, nv2 = noise if noise is not None else (None,) * 4
        a = self._nl(torch.relu(self._nl(f, "_a1", na1)), "_a2", na2)
        v = self._nl(torch.relu(self._nl(f, "_v1", nv1)), "_v2", nv2)
        return v + a - a.mean(-1, keepdim=True)


@pytest.mark.parametrize("N,noisy", [(1, True), (8, True), (8, False)])
def test_oracle_network_matches_a_torch_module(N, noisy):
    torch.manual_seed(N)
    D_in, A, H, E = 5, 3, 16, 8
    m = _TorchRainbowIQN(D_in, A, H, E).double()
    p = {}
    for k, v in m.state_dict().items():
        k = k[len("noisy."):] if k.startswith("noisy.") else ("head.l." + k[5:] if k.startswith("head.") else k)
        p[k] = v.detach()
    x = torch.randn(4, D_in, dtype=torch.float64)
    tau = torch.rand(4, N, dtype=torch.float64)
    noise = [(torch.randn(H, dtype=torch.float64), torch.randn(o, dtype=torch.float64)) for o in (H, H, A, 1)] \
        if noisy else None
    want = m(x, tau, noise)
    got = ori.network(p, x, tau, E, noise)
    assert got.shape == (4, N, A)
    np.testing.assert_allclose(got.detach().numpy(), want.detach().numpy(), rtol=1e-12, atol=1e-13)
