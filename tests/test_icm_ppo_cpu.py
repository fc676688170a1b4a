"""ICM-PPO without a GPU: the configs, the closed-form ICM loss gradients against float64 autograd, the oracle network
against a torch module written from the spec (BatchNorm in training mode with its running buffers, ELU), and the
running statistics / reward filter against a numpy restatement."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import icm_ppo as oi


# ------------------------------------------------------------------------------------------------------- configs
@pytest.mark.parametrize("env", ["cartpole", "mountaincar", "pendulum", "mujoco", "atari"])
def test_configs_are_ppo_rows_plus_the_icm_keys(env):
    from jorldy_b200 import config
    d, ppo = config.load(f"config.icm_ppo.{env}"), config.load(f"config.ppo.{env}")
    a = dict(d.agent)
    assert a.pop("name") == "icm_ppo"
    icm = {k: a.pop(k) for k in ("icm_network", "beta", "lamb", "eta", "extrinsic_coeff", "intrinsic_coeff",
                                 "obs_normalize", "ri_normalize", "batch_norm")}
    frames = env == "atari"
    assert icm == dict(icm_network="icm_cnn" if frames else "icm_mlp", beta=0.2, lamb=1.0, eta=0.01, extrinsic_coeff=1.0,
                       intrinsic_coeff=1.0, obs_normalize=not frames, ri_normalize=True, batch_norm=True)
    assert a == {k: v for k, v in ppo.agent.items() if k != "name"}
    assert d.optim == ppo.optim and d.train == ppo.train and d.env == ppo.env
    assert f"config.icm_ppo.{env}" in config.available()


@pytest.mark.parametrize("kw,match", [
    (dict(icm_network="icm_rnd"), "unknown icm_network"),
    (dict(icm_network="icm_cnn", obs_normalize=False), "takes the observations of head='cnn', got head='mlp'"),
    (dict(icm_network="icm_mlp", head="cnn"), "takes the observations of head='mlp', got head='cnn'"),
    (dict(icm_network="icm_cnn", head="cnn", obs_normalize=True), "obs_normalize=False"),
])
def test_constructor_rejects_mismatched_icm_settings(kw, match):
    """The checks run before the agent allocates anything, so they need no GPU."""
    from jorldy_b200.core.agent.icm_ppo import ICM_PPO
    with pytest.raises(ValueError, match=re.escape(match)):
        ICM_PPO([4, 84, 84] if kw.get("head") == "cnn" else 4, 2, **kw)


def test_one_row_minibatch_with_batch_norm_is_rejected():
    from jorldy_b200.core.agent.icm_ppo import ICM_PPO
    agent = ICM_PPO.__new__(ICM_PPO)
    agent.batch_norm, agent.batch_size = True, 32
    with pytest.raises(ValueError, match=r"batch_size=32.*rollout of 65 rows"):
        agent._check_batch(65)
    agent._check_batch(64)
    agent.batch_size = 1
    with pytest.raises(ValueError, match="batch_size=1"):
        agent._check_batch(64)
    agent.batch_norm = False
    agent._check_batch(65)


# ------------------------------------------------------------------------------------------- closed-form gradients
@pytest.mark.parametrize("cont,A", [(False, 2), (False, 18), (True, 1), (True, 8)])
@pytest.mark.parametrize("beta", [0.0, 0.2, 1.0])
def test_closed_form_icm_gradients_match_autograd(cont, A, beta):
    rs = np.random.RandomState(A + int(10 * beta))
    B = 37
    f = torch.tensor(rs.standard_normal((B, 256)), requires_grad=True)
    phi_n = torch.tensor(rs.standard_normal((B, 256)), requires_grad=True)
    g = torch.tensor(rs.standard_normal((B, A)), requires_grad=True)
    action = torch.tensor(rs.uniform(-1, 1, (B, A)) if cont else rs.randint(0, A, (B, 1)).astype(np.float64))
    _, _, _, loss = oi.icm_loss(f, phi_n, g, action, A, cont, 0.01, beta)
    loss.backward()
    df, dg = oi.closed_form(f.detach(), phi_n.detach(), g.detach(), action, A, cont, beta)
    torch.testing.assert_close(f.grad, df, rtol=1e-12, atol=1e-15)
    torch.testing.assert_close(g.grad, dg, rtol=1e-12, atol=1e-15)
    assert phi_n.grad is None or torch.count_nonzero(phi_n.grad) == 0       # phi(s') is a detached target in l_f


# ------------------------------------------------------------------------------------------------ the network
class SpecICM(torch.nn.Module):
    """The ICM of the spec as torch modules (float64)."""

    def __init__(self, D, A):
        super().__init__()
        self.fc1, self.fc2 = torch.nn.Linear(D, 256), torch.nn.Linear(256, 256)
        self.bn1, self.bn1_next = torch.nn.BatchNorm1d(256), torch.nn.BatchNorm1d(256)
        self.fc_f1, self.fc_f2 = torch.nn.Linear(256 + A, 256), torch.nn.Linear(256 + A, 256)
        self.inv, self.pi = torch.nn.Linear(512, 256), torch.nn.Linear(256, A)

    def phi(self, x, bn):
        return F.elu(self.fc2(F.elu(bn(self.fc1(x)))))

    def forward(self, s, s_next, a):
        phi, phi_n = self.phi(s, self.bn1), self.phi(s_next, self.bn1_next)
        f = self.fc_f2(torch.cat([F.relu(self.fc_f1(torch.cat([phi, a], 1))), a], 1))
        g = self.pi(F.relu(self.inv(torch.cat([phi, phi_n], 1))))
        return f, phi_n, g


def test_oracle_network_matches_the_spec_module_with_batch_norm_buffers():
    torch.manual_seed(0)
    D, A, B = 11, 3, 65
    m = SpecICM(D, A).double().train()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items() if v.is_floating_point() and "running" not in k}
    buf = {k: v.clone() for k, v in sd.items() if "running" in k or "num_batches" in k}
    s, s_n = torch.randn(B, D, dtype=torch.float64), torch.randn(B, D, dtype=torch.float64)
    a = torch.randn(B, A, dtype=torch.float64)
    for _ in range(2):                                    # two passes: the running buffers compound
        ref = m(s, s_n, a)
        got = oi.icm_forward(p, buf, s, s_n, a)
        for x, y in zip(got, ref):
            torch.testing.assert_close(x, y, rtol=1e-12, atol=1e-12)
    for k, v in m.state_dict().items():
        if k in buf:
            torch.testing.assert_close(buf[k], v, rtol=1e-12, atol=1e-12)
    assert int(buf["bn1.num_batches_tracked"]) == 2


# ------------------------------------------------------------------------------------------ statistics
def test_running_mean_std_and_the_reward_filter_match_numpy():
    rs = np.random.RandomState(3)
    rms = oi.RunningMeanStd((5,))
    mean, var, count = np.zeros(5), np.ones(5), 1e-4
    for _ in range(3):
        x = rs.standard_normal((40, 5)) * 3 + 1
        rms.update(x)
        # the parallel merge restated: the moments of the pooled samples, with the prior as `count` pseudo-samples
        bm, bv, n = x.mean(0), x.var(0), len(x)
        tot = count + n
        new_mean = (mean * count + bm * n) / tot
        new_var = (count * (var + (mean - new_mean) ** 2) + n * (bv + (bm - new_mean) ** 2)) / tot
        mean, var, count = new_mean, new_var, tot
        np.testing.assert_allclose(rms.mean, mean, rtol=1e-12)
        np.testing.assert_allclose(rms.var, var, rtol=1e-12)
        assert rms.count == count
    ri = rs.uniform(0, 1, (3, 7))
    filt, e = oi.reward_filter(np.array([0.5, 0.0, 1.0]), ri, 0.9)
    exp = np.empty_like(ri)
    acc = np.array([0.5, 0.0, 1.0])
    for t in range(7):
        acc = 0.9 * acc + ri[:, t]
        exp[:, t] = acc
    np.testing.assert_allclose(filt, exp, rtol=1e-15)
    np.testing.assert_array_equal(e, filt[:, -1])


# ---------------------------------------------------------------------------------------- frame-ring residency
def _next_refs_resident(T, F, done, rollouts=3):
    """Pushes `rollouts` rollouts of T steps into one lane's ring of F frames the way FrameStore.start / push do
    (csrc/frame_ring.cu) and checks, when learn_rollout() reads each rollout, that every stack it references is resident:
    the T states and, as ICM-PPO's next_ref column keeps them, all T next states (the terminal stack at done steps).  A
    stack at position p reaches back to max(p - 3, first[p]); it is resident while that is >= head - F.  done(r, t)."""
    first = []                                           # first[p]: episode-first position of the frame at p

    push = first.append
    push(0)                                              # start(): the reset frame
    for r in range(rollouts):
        h0, refs = len(first), []
        for t in range(T):
            s = len(first) - 1                           # the stack acted on
            push(first[s])                               # the newest frame continues its episode
            refs += [s, len(first) - 1]                  # state_ref and next_ref of step t
            if done(r, t):
                push(len(first))                         # auto-reset: an episode-first frame
        h = len(first)
        for p in refs:
            lo = max(p - 3, first[p])
            assert h0 - 4 <= lo and p < h0 + 2 * T       # the window frames_per_rollout sizes the ring for
            if not (p < h and lo >= h - F):
                return False
    return True


def _patterns(T):
    table = np.random.RandomState(T).rand(3, T) < 0.3
    return {"every": lambda r, t: True, "never": lambda r, t: False,
            "alternating": lambda r, t: (r * T + t) % 2 == 0, "random": lambda r, t: bool(table[r, t]),
            "never_then_every": lambda r, t: r > 0}


@pytest.mark.parametrize("T", [1, 5, 128])
@pytest.mark.parametrize("pattern", ["every", "never", "alternating", "random", "never_then_every"])
def test_every_next_ref_stays_resident_in_the_rollout_ring(T, pattern):
    from jorldy_b200.core.buffer.frame_store import frames_per_rollout
    assert _next_refs_resident(T, frames_per_rollout(T), _patterns(T)[pattern])


@pytest.mark.parametrize("T", [5, 128])
def test_a_shorter_ring_evicts_next_refs(T):
    """One frame less than frames_per_rollout(T) loses a reference once a rollout that starts mid-episode ends one at
    every step: the ring is sized by the window, with no slack."""
    assert not _next_refs_resident(T, 2 * T + 3, _patterns(T)["never_then_every"])
