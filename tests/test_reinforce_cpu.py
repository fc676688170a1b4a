"""REINFORCE without a GPU: the configs, the constructor's rejections, the float64 oracle's closed-form gradient against
autograd of the reference expression, the oracle's batched ring-to-rows mapping against the reference's per-episode
loop, and the episode ring's capacity argument."""
import numpy as np
import pytest
import torch

from jorldy_b200 import config
from jorldy_b200.core.buffer import EpisodeRing
from oracle import reinforce as orf

ENVS = ("cartpole", "mountaincar", "pendulum", "mujoco")


# ------------------------------------------------------------------------------------------------------------ configs
def test_configs():
    names = [f"config.reinforce.{e}" for e in ENVS]
    assert all(n in config.available() for n in names)
    for e, n in zip(ENVS, names):
        c, ppo = config.load(n), config.load(f"config.ppo.{e}")
        assert c.agent == dict(name="reinforce", network=ppo.agent["network"].replace("_value", ""), gamma=0.99,
                               use_standardization=True, lr_decay=True)
        assert c.env == ppo.env and c.optim == ppo.optim
        assert "distributed_batch_size" not in c.train
        assert c.train == {k: v for k, v in ppo.train.items() if k != "distributed_batch_size"}
    assert config.load("config.reinforce.pendulum").agent["network"] == "continuous_policy"
    assert config.load("config.reinforce.cartpole").agent["network"] == "discrete_policy"
    with pytest.raises(ImportError):
        config.load("config.reinforce.atari")


def test_registered():
    from jorldy_b200.core.agent import agent_dict
    from jorldy_b200.core.agent.reinforce import REINFORCE
    assert agent_dict["reinforce"] is REINFORCE


@pytest.mark.parametrize("kwargs, exc", [
    (dict(action_size=19), ValueError),
    (dict(action_size=0), ValueError),
    (dict(network="continuous_policy", action_size=9), ValueError),
    (dict(network="discrete_policy_value"), ValueError),
    (dict(head="cnn"), NotImplementedError),
])
def test_constructor_rejections(kwargs, exc):
    from jorldy_b200.core.agent.reinforce import REINFORCE
    args = dict(state_size=4, action_size=2)
    args.update(kwargs)
    with pytest.raises(exc):
        REINFORCE(**args)


def test_collector_rejects_envs_without_a_ring_bound():
    from jorldy_b200.core.collect import EpisodeCollector

    class NoLimit:
        max_steps = None

    class Frames:
        frame_stack = True

    with pytest.raises(ValueError):
        EpisodeCollector(NoLimit(), None, 8)
    with pytest.raises(NotImplementedError):
        EpisodeCollector(Frames(), None, 8)


# ------------------------------------------------------------------------------------------ closed-form gradients
def _loss_inputs(rs, M, A, continuous, extreme=False):
    nout = 2 * A if continuous else A
    out = torch.as_tensor(rs.standard_normal((M, nout)) * 2, dtype=torch.float64)
    if continuous:
        a = torch.as_tensor(np.tanh(rs.standard_normal((M, A))), dtype=torch.float64)
        if extreme:     # raw mu at exactly +-5 and beyond, actions at +-1
            out[0, 0], out[-1, 0] = 5.0, -5.0
            if M > 2:
                out[1, 0], out[2, A - 1] = 7.5, -6.0
            a[0, 0], a[-1, A - 1] = 1.0, -1.0
    else:
        a = torch.as_tensor(rs.randint(0, A, M), dtype=torch.int64)
    ret = torch.as_tensor(rs.standard_normal(M), dtype=torch.float64)
    return out, a, ret


@pytest.mark.parametrize("continuous, A", [(False, 2), (False, 18), (True, 1), (True, 3), (True, 8)])
@pytest.mark.parametrize("M", [1, 2, 7, 300])
def test_closed_form_matches_autograd(continuous, A, M):
    rs = np.random.RandomState(17 * M + A)
    out, a, ret = _loss_inputs(rs, M, A, continuous, extreme=True)
    leaf = out.clone().requires_grad_(True)
    orf.loss(leaf, a, ret, A, continuous).backward()
    g = orf.closed_form(out, a, ret, A, continuous)
    np.testing.assert_allclose(g.numpy(), leaf.grad.numpy(), rtol=0, atol=1e-10)


# ------------------------------------------------------------------------------------------ the batched mapping
def _simulate(rs, N, L, rounds, T, p_done, max_steps=None, gamma=0.9, standardize=True):
    """Runs N envs in lockstep for `rounds` rounds of T steps with random rewards and dones, learning after every
    round with the oracle's ring mapping.  Checks every learn against the reference loop applied to each env's episodes
    taken from the plain (unwrapped) time series, episode by episode, env-major and oldest first."""
    reward = np.zeros((N, L))
    done = np.zeros((N, L))
    series_r = [[] for _ in range(N)]
    series_d = [[] for _ in range(N)]
    head = np.zeros(N, np.int64)
    learned = np.zeros(N, np.int64)             # episodes of each env already learned (the reference's side)
    elapsed = np.zeros(N, np.int64)
    pos = 0
    n_learns = 0
    for _ in range(rounds):
        for _ in range(T):
            r = rs.standard_normal(N)
            d = p_done(rs, N)
            elapsed += 1
            if max_steps is not None:
                d = np.where(elapsed >= max_steps, 1.0, d)
            elapsed = np.where(d != 0, 0, elapsed)
            col = pos % L
            reward[:, col], done[:, col] = r, d
            for e in range(N):
                series_r[e].append(r[e])
                series_d[e].append(d[e])
            pos += 1
        idx, ret, count, new_head = orf.ring_rows(reward, done, pos, head, gamma, standardize)
        # the reference, episode by episode
        exp_idx, exp_ret = [], []
        for e in range(N):
            ends = [t for t, dd in enumerate(series_d[e]) if dd != 0]
            starts = [0] + [t + 1 for t in ends[:-1]]
            for k in range(learned[e], len(ends)):
                ts = range(starts[k], ends[k] + 1)
                exp_idx += [e * L + t % L for t in ts]
                exp_ret += list(orf.reference_returns([series_r[e][t] for t in ts], gamma, standardize))
            learned[e] = len(ends)
        np.testing.assert_array_equal(idx, np.array(exp_idx, np.int64))
        np.testing.assert_allclose(ret, np.array(exp_ret), rtol=0, atol=1e-12)
        assert count.sum() == len(exp_idx)
        head = new_head
        n_learns += int(len(idx) > 0)
    return n_learns


def _bernoulli(p):
    return lambda rs, N: (rs.random_sample(N) < p).astype(np.float64)


@pytest.mark.parametrize("standardize", [True, False])
@pytest.mark.parametrize("case", ["random", "length1", "cross_rounds", "several_per_round", "none_complete", "wrap"])
def test_ring_mapping_matches_reference_loop(case, standardize):
    rs = np.random.RandomState(["random", "length1", "cross_rounds", "several_per_round", "none_complete", "wrap"].index(case))
    N, T = 5, 8
    if case == "random":
        _simulate(rs, N, 64, 3, T, _bernoulli(0.2), standardize=standardize)
    elif case == "length1":         # every step ends an episode
        _simulate(rs, N, T, 3, T, lambda rs, N: np.ones(N), standardize=standardize)
    elif case == "cross_rounds":    # episodes of 20 steps over rounds of 8
        _simulate(rs, N, 19 + T, 5, T, lambda rs, N: np.zeros(N), max_steps=20, standardize=standardize)
    elif case == "several_per_round":
        _simulate(rs, N, 64, 2, T, _bernoulli(0.6), standardize=standardize)
    elif case == "none_complete":   # env 0 never completes within the run
        def p(rs, N):
            d = _bernoulli(0.3)(rs, N)
            d[0] = 0.0
            return d
        _simulate(rs, N, 64, 3, T, p, standardize=standardize)
    else:                           # a ring of L = max_steps - 1 + T wrapped many times over
        n = _simulate(rs, N, 6 - 1 + T, 12, T, _bernoulli(0.1), max_steps=6, standardize=standardize)
        assert n == 12


# ------------------------------------------------------------------------------------------ ring capacity
def _max_unlearned_overwritten(L, max_steps, T, done_fn, rounds=60, seed=0):
    """Models the ring positions: returns True if a write ever lands on an unlearned step (one that was written but
    not yet consumed by a learn and is older than L steps)."""
    rs = np.random.RandomState(seed)
    N = max_steps           # env e may first end at step e (the "never" pattern), so every phase occurs
    head = np.zeros(N, np.int64)
    elapsed = np.zeros(N, np.int64)
    last_done = np.full(N, -1, np.int64)
    pos = 0
    for rnd in range(rounds):
        for _ in range(T):
            # writing step `pos` into column pos % L overwrites step pos - L: unlearned if pos - L >= head
            if np.any(pos - L >= head):
                return True
            d = done_fn(rs, N, pos, rnd)
            elapsed += 1
            d = np.where(elapsed >= max_steps, 1, d)
            last_done = np.where(d != 0, pos, last_done)
            elapsed = np.where(d != 0, 0, elapsed)
            pos += 1
        head = np.maximum(head, last_done + 1)      # the learn consumes every completed step
    return False


@pytest.mark.parametrize("pattern", ["every", "never", "alternating", "random"])
@pytest.mark.parametrize("max_steps, T", [(5, 3), (10, 8), (200, 128), (7, 16)])
def test_ring_capacity(pattern, max_steps, T):
    fns = {"every": lambda rs, N, pos, r: np.ones(N, np.int64),
           "never": lambda rs, N, pos, r: (np.arange(N) == pos).astype(np.int64),   # time-limit episodes, staggered
           "alternating": lambda rs, N, pos, r: np.full(N, pos % 2, np.int64),
           "random": lambda rs, N, pos, r: (rs.random_sample(N) < 0.05).astype(np.int64)}
    L = max_steps - 1 + T
    assert L == EpisodeRing.capacity(max_steps, T)
    assert not _max_unlearned_overwritten(L, max_steps, T, fns[pattern])
    if pattern == "never":          # with episodes that run to the time limit, one step less of ring is overwritten
        assert _max_unlearned_overwritten(L - 1, max_steps, T, fns[pattern])
