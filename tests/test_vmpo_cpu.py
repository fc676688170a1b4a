"""CPU checks of V-MPO: the built-in configs, and the float64 oracle's closed-form gradients (what csrc/vmpo.cu
computes) against autograd of its loss, including median ties, the empty top half and the max-shifted eta loss."""
import math

import numpy as np
import pytest
import torch

from oracle import vmpo as ov

EPS = (0.01, 0.01, 5e-5)


def _case(rs, B, A, continuous, adv=None):
    nout = 2 * A + 1 if continuous else A + 1
    out = torch.from_numpy(rs.standard_normal((B, nout)))
    out_old = out + 0.3 * torch.from_numpy(rs.standard_normal((B, nout)))
    if continuous:
        out[:, 0] = 6.0                         # one clamped mu column (zero gradient through the clamp)
        action = torch.from_numpy(rs.uniform(-0.99, 0.99, (B, A)))
    else:
        action = torch.from_numpy(rs.randint(0, A, B).astype(np.float64))
    if adv is None:
        adv = torch.from_numpy(rs.standard_normal(B))
    ret = torch.from_numpy(rs.standard_normal(B))
    return out, out_old, action, adv, ret


def _autograd(out, out_old, action, adv, ret, mult, A, continuous):
    o = out.clone().requires_grad_(True)
    m = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in mult]
    loss, aux = ov.minibatch_loss(o, out_old, action, adv, ret, *m, EPS, A, continuous)
    loss.backward()
    dm = torch.stack([t.grad if t.grad is not None else torch.zeros((), dtype=torch.float64) for t in m])
    return o.grad, dm, aux


def test_vmpo_configs_extend_the_ppo_rows():
    from jorldy_b200 import config as cfg
    paths = [p for p in cfg.available() if p.split(".")[1] == "vmpo"]
    assert sorted(paths) == sorted(f"config.vmpo.{e}" for e in ("cartpole", "mountaincar", "pendulum", "mujoco", "atari"))
    for p in paths:
        v, ppo = cfg.load(p), cfg.load(p.replace("vmpo", "ppo"))
        a = v.agent
        assert a["name"] == "vmpo"
        for k in ("min_eta", "min_alpha_mu", "min_alpha_sigma", "eps_eta", "eps_alpha_mu", "eps_alpha_sigma", "eta",
                  "alpha_mu", "alpha_sigma"):
            assert k in a and a[k] > 0, (p, k)
        for k, val in ppo.agent.items():
            if k not in ("name", "epsilon_clip", "vf_coef", "ent_coef"):
                assert a[k] == val, (p, k)
        assert v.optim == ppo.optim and v.train == ppo.train and v.env == ppo.env
    assert cfg.load("config.vmpo.atari").agent["head"] == "cnn"
    assert cfg.load("config.vmpo.mujoco").agent["network"] == "continuous_policy_value"


@pytest.mark.parametrize("continuous,A", [(False, 2), (False, 18), (True, 1), (True, 3)])
@pytest.mark.parametrize("B", [1, 2, 7, 64])
def test_closed_form_gradients_equal_autograd(continuous, A, B):
    rs = np.random.RandomState(B * 31 + A)
    case = _case(rs, B, A, continuous)
    mult = (0.7, 1.3, 0.4)
    g_ref, dm_ref, _ = _autograd(*case, mult, A, continuous)
    g, dm = ov.closed_form(*case, *[torch.tensor(v, dtype=torch.float64) for v in mult], EPS, A, continuous)
    np.testing.assert_allclose(g.numpy(), g_ref.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(dm.numpy(), dm_ref.numpy(), rtol=1e-10, atol=1e-12)
    if not continuous:
        assert dm[2] == 0.0


def test_max_shifted_eta_loss_equals_the_literal_form_where_finite():
    rs = np.random.RandomState(3)
    adv = torch.from_numpy(rs.standard_normal(256))
    _, top = ov.top_half(adv)
    n = int(top.sum())
    for eta in (10.0, 1.0, 0.1, 0.02):
        literal = eta * 0.01 + eta * torch.log(torch.mean(torch.exp(adv[top] / eta)))
        z = adv[top] / eta
        shifted = eta * 0.01 + eta * (z.max() + torch.log(torch.exp(z - z.max()).sum()) - math.log(n))
        assert torch.isfinite(literal)
        np.testing.assert_allclose(float(shifted), float(literal), rtol=1e-12)
    # at eta = min_eta the literal form overflows even in float64; the shifted one stays finite (and ~ max top advantage)
    eta = 1e-8
    assert not torch.isfinite(torch.log(torch.mean(torch.exp(adv[top] / eta))))
    out, out_old, action, _, ret = _case(rs, 256, 2, False)
    loss, aux = ov.minibatch_loss(out, out_old, action, adv, ret, torch.tensor(eta, dtype=torch.float64),
                                  torch.tensor(1.0, dtype=torch.float64), torch.tensor(1.0, dtype=torch.float64), EPS, 2,
                                  False)
    assert torch.isfinite(loss) and abs(float(aux["eta_loss"]) - float(adv.max())) < 1e-6


def test_median_ties_are_excluded_from_the_top_half():
    adv = torch.tensor([0.5, -1.0, 0.5, 0.5, 2.0, 0.5], dtype=torch.float64)
    m, top = ov.top_half(adv)
    assert float(m) == 0.5                                  # element (B-1)//2 = 2 of the sorted values
    assert top.tolist() == [False, False, False, False, True, False]
    rs = np.random.RandomState(5)
    case = _case(rs, 6, 3, False, adv=adv)
    g_ref, dm_ref, aux = _autograd(*case, (1.0, 1.0, 1.0), 3, False)
    g, dm = ov.closed_form(*case, *[torch.tensor(1.0, dtype=torch.float64)] * 3, EPS, 3, False)
    assert aux["n"] == 1
    np.testing.assert_allclose(g.numpy(), g_ref.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(dm.numpy(), dm_ref.numpy(), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("continuous,A", [(False, 4), (True, 2)])
@pytest.mark.parametrize("B", [1, 5])
def test_empty_top_half_keeps_the_kl_and_critic_terms(continuous, A, B):
    rs = np.random.RandomState(B)
    case = _case(rs, B, A, continuous, adv=torch.full((B,), 0.25, dtype=torch.float64))
    g_ref, dm_ref, aux = _autograd(*case, (0.5, 2.0, 3.0), A, continuous)
    assert aux["n"] == 0 and float(aux["actor_loss"]) == 0.0 and float(aux["eta_loss"]) == 0.0
    assert dm_ref[0] == 0.0 and torch.all(torch.isfinite(g_ref))
    assert torch.any(g_ref[:, :-1] != 0)                    # the KL terms still move the policy head
    g, dm = ov.closed_form(*case, *[torch.tensor(v, dtype=torch.float64) for v in (0.5, 2.0, 3.0)], EPS, A, continuous)
    np.testing.assert_allclose(g.numpy(), g_ref.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(dm.numpy(), dm_ref.numpy(), rtol=1e-10, atol=1e-12)
