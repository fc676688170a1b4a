"""TicTacToe and MuZero's masked root on the GPU: the env against the numpy oracle (oracle/tictactoe.py) bit for bit, the
opponent's laws, the masked tree kernels against the float64 oracle (oracle/muzero_legal.py) and against the unmasked
kernels, the masked search with real networks, the agent's masked act, the other collectors on the env, and end-to-end
runs of `jorldy_b200.main` on `config.muzero.tictactoe`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import muzero as om
from oracle import muzero_legal as ol
from oracle import tictactoe as ot

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"


def _C():
    from jorldy_b200.core.dev import C
    return C


def ptr(t):
    return 0 if t is None else t.data_ptr()


def _env(N, seed=0, **kw):
    from jorldy_b200.core import Env
    return Env("tictactoe", num_envs=N, seed=seed, **kw)


# ------------------------------------------------------------------------------------------- 1. env vs oracle
def _assert_env_equal(env, ref, tag):
    assert np.array_equal(env.boards.cpu().numpy(), ref.boards), tag
    assert np.array_equal(env.obs.cpu().numpy(), ref.obs), tag
    assert np.array_equal(env.legal.cpu().numpy(), ref.legal), tag
    assert np.array_equal(env.elapsed.cpu().numpy(), ref.elapsed), tag
    assert np.array_equal(env.episode.cpu().numpy(), ref.episode), tag
    assert np.array_equal(env._score.cpu().numpy(), ref.score), tag


def _actions(rng, legal, N):
    """Random actions: mostly a legal cell, sometimes an occupied cell or one outside 0..8."""
    a = np.array([rng.choice(np.flatnonzero(l)) if l.any() else 0 for l in legal], dtype=np.int64)
    bad = rng.random(N) < 0.15
    a[bad] = rng.integers(-2, 11, int(bad.sum()))
    return a


@pytest.mark.parametrize("N", [1, 7, 4096])
@pytest.mark.parametrize("auto_reset", [True, False])
@pytest.mark.parametrize("graph", [False, True])
def test_env_matches_the_oracle_bit_for_bit(N, auto_reset, graph):
    """64 steps of random legal and illegal actions.  Under a graph, one captured step is replayed every step, so each
    replay must draw from the advanced episode and move counters."""
    env = _env(N, seed=5, id=1, auto_reset=auto_reset)
    ref = ot.TicTacToeBatch(N, seed=5, id=1, auto_reset=auto_reset)
    env.reset_device()
    ref.reset()
    _assert_env_equal(env, ref, "reset")
    rng = np.random.default_rng(N)
    act = torch.zeros(N, dtype=torch.int64, device=DEV)
    g = None
    for t in range(64):
        a = _actions(rng, ref.legal, N)
        if not auto_reset and t % 8 == 7:           # without auto-reset, reset the finished boards by mask
            mask = torch.as_tensor(ref_done.astype(np.uint8), device=DEV)
            env.reset_device(mask)
            ref.reset(ref_done.astype(bool))
        act.copy_(torch.as_tensor(a))
        if graph:
            if g is None:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    env.step_device(act)
            g.replay()                              # capture does not run the step: the first replay is step 0
        else:
            env.step_device(act)
        ns, r, d = ref.step(a)
        ref_done = d > 0
        torch.cuda.synchronize()
        assert np.array_equal(env.next_obs.cpu().numpy(), ns), t
        assert np.array_equal(env.reward.cpu().numpy(), r), t
        assert np.array_equal(env.done.cpu().numpy(), d), t
        _assert_env_equal(env, ref, t)
    assert np.array_equal(env.stats.cpu().numpy(), ref.stats)
    if auto_reset:
        assert ref.stats[0] > 0


def test_numpy_api_and_action_kinds():
    env = _env(3, seed=2)
    obs = env.reset()
    assert obs.shape == (3, 18) and obs.dtype == np.float32
    assert env.state_size == 18 and env.action_size == 9 and env.action_type == "discrete" and env.max_steps == 5
    legal = env.legal.cpu().numpy()
    a = np.array([[int(np.flatnonzero(l)[0])] for l in legal])
    ns, r, d = env.step(a)
    assert ns.shape == (3, 18) and r.shape == (3, 1) and r.dtype == np.float64 and d.shape == (3, 1) and d.dtype == bool
    with pytest.raises(ValueError):
        env.step(np.array([[0], [9], [1]]))
    with pytest.raises(TypeError):
        env.step_device(torch.zeros(3, device=DEV))
    # int32 actions step exactly like int64
    e1, e2 = _env(64, seed=4), _env(64, seed=4)
    e1.reset_device()
    e2.reset_device()
    a = torch.randint(0, 9, (64,), device=DEV, generator=torch.Generator(DEV).manual_seed(0))
    e1.step_device(a)
    e2.step_device(a.to(torch.int32))
    assert torch.equal(e1.obs, e2.obs) and torch.equal(e1.reward, e2.reward) and torch.equal(e1.next_obs, e2.next_obs)


# ------------------------------------------------------------------------------------------- 2. opponent law
def test_opening_and_opponent_cell_laws():
    """10^5 boards: the opening happens with probability 1/2 on a uniform cell, and the reply to the agent's centre move
    on a board the opponent did not open is uniform over the 8 empty cells (chi-square)."""
    from scipy import stats
    N = 100000
    env = _env(N, seed=11)
    env.reset_device()
    op = env.obs[:, 9:].cpu().numpy()
    opened = op.sum(1) > 0
    assert stats.binomtest(int(opened.sum()), N, 0.5).pvalue > 1e-3
    cells = op[opened].argmax(1)
    assert stats.chisquare(np.bincount(cells, minlength=9)).pvalue > 1e-3
    fresh = ~opened
    env.step_device(torch.full((N,), 4, dtype=torch.int64, device=DEV))
    reply = env.next_obs[:, 9:].cpu().numpy()[fresh].argmax(1)
    counts = np.bincount(reply, minlength=9)
    assert counts[4] == 0
    assert stats.chisquare(np.delete(counts, 4)).pvalue > 1e-3


# ------------------------------------------------------------------------------------------- 3-4. masked tree kernels
def _tree(N, A, S, Hs):
    f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)
    i = lambda *s: torch.zeros(*s, dtype=torch.int32, device=DEV)
    return {"n": i(N, S + 1, A), "w": f(N, S + 1, A), "p": f(N, S + 1, A), "r": f(N, S + 1, A),
            "child": i(N, S + 1, A), "latent": f(N, S + 1, Hs), "count": i(N), "bounds": f(N, 2), "path": i(N, S + 1),
            "path_len": i(N)}


def _scripted_search(N, A, S, gamma, seed, legal, training=False, gamma_in=None, masked=True):
    """The tree kernels with a scripted model (random logits per simulation); masked: the _legal entry points with
    `legal` u8 [N, A].  Returns the tree dict and the actions."""
    C, Hs, V, R = _C(), 8, 5, 2
    g = torch.Generator().manual_seed(seed)
    root_pi, root_v = torch.randn(N, A, generator=g), torch.randn(N, 2 * V + 1, generator=g)
    sims = {"pi": torch.randn(S, N, A, generator=g), "v": torch.randn(S, N, 2 * V + 1, generator=g),
            "r": torch.randn(S, N, 2 * R + 1, generator=g), "s": torch.rand(S, N, Hs, generator=g)}
    lat0 = torch.rand(N, Hs, generator=g)
    t = _tree(N, A, S, Hs)
    tree = [ptr(t[k]) for k in ("n", "w", "p", "r", "child", "latent", "count", "bounds", "path", "path_len")]
    dev = {k: v.to(DEV).contiguous() for k, v in sims.items()}
    leaf_n, leaf_a = torch.zeros(N, dtype=torch.int32, device=DEV), torch.zeros(N, dtype=torch.int32, device=DEV)
    dyn = torch.zeros(N, Hs + A, device=DEV)
    gin = None if gamma_in is None else torch.as_tensor(gamma_in, dtype=torch.float64, device=DEV)
    ctr = torch.zeros(N, dtype=torch.int64, device=DEV)
    lg = torch.as_tensor(np.asarray(legal, dtype=np.uint8), device=DEV).contiguous()
    root_d = [x.to(DEV) for x in (root_pi, root_v, lat0)]
    root_args = (*(ptr(x) for x in root_d), N, A, S, Hs, V, int(training), 0.25, 0.25, ptr(gin), 7, ptr(ctr), *tree, 0)
    if masked:
        C.jb_mcts_root_legal(*root_args, ptr(lg), 0)
    else:
        C.jb_mcts_root(*root_args, 0)
    for j in range(S):
        sel = (N, A, S, Hs, gamma, *tree, ptr(leaf_n), ptr(leaf_a), ptr(dyn))
        if masked:
            C.jb_mcts_select_legal(*sel, ptr(lg), 0)
        else:
            C.jb_mcts_select(*sel, 0)
        C.jb_mcts_expand_backup(ptr(dev["s"][j]), ptr(dev["pi"][j]), ptr(dev["v"][j]), ptr(dev["r"][j]), N, A, S, Hs, V,
                                R, gamma, ptr(leaf_n), ptr(leaf_a), *tree, 0)
    action = torch.zeros(N, dtype=torch.int64, device=DEV)
    pi, rv = torch.zeros(N, A, device=DEV), torch.zeros(N, device=DEV)
    C.jb_mcts_act(N, A, S, gamma, 0, 0, 0, 11, 0, ptr(t["n"]), ptr(t["w"]), ptr(t["r"]), ptr(action), ptr(pi), ptr(rv), 0)
    torch.cuda.synchronize()
    t["action"], t["pi"], t["rv"] = action, pi, rv
    return t, root_pi, lat0, sims


def _masks(kind, N, A, rng):
    if kind == "all":
        return np.ones((N, A), dtype=np.uint8)
    if kind == "single":
        m = np.zeros((N, A), dtype=np.uint8)
        m[np.arange(N), rng.integers(0, A, N)] = 1
        return m
    m = (rng.random((N, A)) < 0.5).astype(np.uint8)
    m[0] = 0                                          # a row with no legal action searches unmasked
    return m


@pytest.mark.parametrize("A", [2, 9, 18])
@pytest.mark.parametrize("kind", ["random", "single", "all"])
@pytest.mark.parametrize("training", [False, True])
def test_masked_kernels_vs_oracle(A, kind, training):
    N, S, gamma = 64, 24, 0.997
    rng = np.random.default_rng(A * 10 + len(kind))
    legal = _masks(kind, N, A, rng)
    gam = rng.gamma(0.25, size=(N, A)) + 1e-3 if training else None
    t, root_pi, lat0, sims = _scripted_search(N, A, S, gamma, seed=A, legal=legal, training=training, gamma_in=gam)
    n, p0 = t["n"].cpu().numpy(), t["p"][:, 0].cpu().numpy()
    for e in range(N):
        model = lambda sim, lat, a, e=e: (sims["s"][sim, e].double(), sims["pi"][sim, e].double(),
                                          sims["v"][sim, e].double(), sims["r"][sim, e].double())
        tr, a, pi, rv = ol.search_legal(root_pi[e].double().numpy(), lat0[e].double(), model, A, S, gamma, 5, 2,
                                        legal[e], noise=None if gam is None else gam[e], training=False)
        np.testing.assert_allclose(p0[e], tr.p[0], rtol=1e-5, atol=1e-7, err_msg=f"env {e}")
        np.testing.assert_array_equal(n[e], tr.n, err_msg=f"env {e}")
        assert int(t["action"][e]) == a
        ok = legal[e].astype(bool) if legal[e].any() else np.ones(A, dtype=bool)
        assert n[e, 0][~ok].sum() == 0 and p0[e][~ok].sum() == 0


@pytest.mark.parametrize("A", [2, 9, 18])
@pytest.mark.parametrize("training", [False, True])
def test_all_legal_mask_is_bit_identical_to_the_unmasked_kernels(A, training):
    """With every action legal, the Philox-drawn noise, the priors and every tree array equal the unmasked kernels'."""
    N, S = 256, 32
    legal = np.ones((N, A), dtype=np.uint8)
    a, *_ = _scripted_search(N, A, S, 0.997, seed=A + 1, legal=legal, training=training, masked=True)
    b, *_ = _scripted_search(N, A, S, 0.997, seed=A + 1, legal=legal, training=training, masked=False)
    for k in ("n", "w", "p", "r", "child", "latent", "count", "bounds", "path", "path_len", "action", "pi", "rv"):
        assert torch.equal(a[k], b[k]), k


def test_masked_kernels_reject_a_null_mask():
    from jorldy_b200._lib import JbError
    C, N, A, S, Hs = _C(), 2, 3, 2, 4
    t = _tree(N, A, S, Hs)
    tree = [ptr(t[k]) for k in ("n", "w", "p", "r", "child", "latent", "count", "bounds", "path", "path_len")]
    z = torch.zeros(N, 2 * A + 8, device=DEV)
    i = torch.zeros(N, dtype=torch.int32, device=DEV)
    with pytest.raises(JbError):
        C.jb_mcts_root_legal(ptr(z), ptr(z), ptr(z), N, A, S, Hs, 1, 0, 0.25, 0.25, 0, 1, 0, *tree, 0, 0, 0)
    with pytest.raises(JbError):
        C.jb_mcts_select_legal(N, A, S, Hs, 1.0, *tree, ptr(i), ptr(i), ptr(z), 0, 0)


# ------------------------------------------------------------------------------------------- 5. search, real networks
def _agent(**kw):
    from jorldy_b200.core import Agent
    args = dict(state_size=18, action_size=9, hidden_size=32, latent_size=16, num_simulation=12, num_unroll=3,
                td_steps=5, gamma=1.0, value_support=1, reward_support=1, batch_size=16, buffer_size=512,
                start_train_step=0, optim_config={"name": "adam", "lr": 1e-3}, run_step=1000, lr_decay=False,
                device=DEV, seed=3)
    args.update(kw)
    return Agent("muzero", **args)


def test_masked_search_with_networks_vs_oracle():
    N = 64
    env = _env(N, seed=3)
    env.reset_device()
    for _ in range(2):                                # boards with a few marks on them
        env.step_device(torch.as_tensor([int(np.flatnonzero(l)[-1]) for l in env.legal.cpu().numpy()], device=DEV))
    agent = _agent(use_cuda_graph=False)
    agent.attach_legal(env.legal)
    with torch.no_grad():
        agent.network.p["f.pi.weight"].mul_(300.0)
        agent.network.p["f.v.weight"].mul_(30.0)
        agent.network.p["g.r.weight"].mul_(30.0)
    x = env.obs.clone()
    action, _ = agent.act_device(x, training=False)
    n = agent._search_state(N)["n"].cpu().numpy()
    legal = env.legal.cpu().numpy()
    p = {k: v.double().cpu() for k, v in agent.network.state_dict().items()}
    model = om.network_model(p, 9)
    s0 = om.represent(p, x.double().cpu())
    pi0, _ = om.predict(p, s0)
    qualify = 0
    for e in range(N):
        assert legal[e, int(action[e])] == 1 and n[e, 0][legal[e] == 0].sum() == 0
        margins = []
        tr, a, _, _ = ol.search_legal(pi0[e].numpy(), s0[e], model, 9, 12, 1.0, 1, 1, legal[e], margins=margins)
        if not margins or min(margins) > 1e-3:
            qualify += 1
            np.testing.assert_array_equal(n[e], tr.n, err_msg=f"env {e}")
            assert int(action[e]) == a
    assert qualify >= 0.8 * N, qualify


# ------------------------------------------------------------------------------------------- 6. agent
def test_graph_act_is_bit_identical_to_eager_with_the_mask():
    res = []
    for graph in (True, False):
        env = _env(32, seed=8)
        env.reset_device()
        agent = _agent(use_cuda_graph=graph)
        agent.attach_legal(env.legal)
        steps = []
        for _ in range(6):
            a, v = agent.act_device(env.obs, training=True)
            steps.append((a.clone(), v.clone(), agent.step_inputs["policy"].clone(), env.legal.clone()))
            env.step_device(a)
        res.append(steps)
        if graph:
            assert (32, True) in agent._graphs
    for (a1, v1, p1, l1), (a2, v2, p2, l2) in zip(*res):
        assert torch.equal(a1, a2) and torch.equal(v1, v2) and torch.equal(p1, p2) and torch.equal(l1, l2)
        assert bool((l1.gather(1, a1.view(-1, 1)) == 1).all())          # every sampled action is legal
        assert float(p1[l1 == 0].abs().sum()) == 0.0


def test_attach_after_capture_drops_the_graph_and_rows_must_match():
    env = _env(16, seed=1)
    env.reset_device()
    agent = _agent(use_cuda_graph=True)
    agent.act_device(env.obs, training=True)
    assert (16, True) in agent._graphs
    agent.attach_legal(env.legal)
    assert not agent._graphs
    a, _ = agent.act_device(env.obs, training=True)
    assert bool((env.legal.gather(1, a.view(-1, 1)) == 1).all())
    with pytest.raises(RuntimeError):
        agent.act_device(torch.zeros(8, 18, device=DEV), training=True)
    with pytest.raises(ValueError):
        agent.attach_legal(torch.ones(16, 9, device=DEV))


def _greedy_games(agent, N=10000, seed=0):
    """N greedy games against the env's opponent; returns the forfeit count and the outcomes."""
    env = _env(N, seed=seed, auto_reset=False)
    env.reset_device()
    agent.attach_legal(env.legal)
    live = torch.ones(N, dtype=torch.bool, device=DEV)
    forfeits = torch.zeros(N, dtype=torch.bool, device=DEV)
    outcome = torch.zeros(N, device=DEV)
    for _ in range(5):
        a, _ = agent.act_device(env.obs, training=False)
        illegal = env.legal.gather(1, a.view(-1, 1)).view(-1) == 0
        forfeits |= live & illegal
        env.step_device(a)
        outcome = torch.where(live & (env.done > 0), env.reward, outcome)
        live &= env.done == 0
    assert not bool(live.any())
    return int(forfeits.sum()), outcome


def test_greedy_agent_never_forfeits_trained_or_not():
    from jorldy_b200.core.collect import ReplayCollector
    agent = _agent(num_simulation=8, use_cuda_graph=True)
    f0, _ = _greedy_games(agent)
    assert f0 == 0
    env = _env(16, seed=2)
    agent.attach_legal(env.legal)
    col = ReplayCollector(env, agent, update_period=4)
    step, learns = 0, 0
    for _ in range(30):
        step, res = col.run_round(step)
        learns += bool(res)
    assert learns > 0
    f1, _ = _greedy_games(agent, seed=1)
    assert f1 == 0


# ------------------------------------------------------------------------------------------- 7. other collectors
def _cfg_agent(config_path, env, **override):
    from jorldy_b200 import config as builtin
    from jorldy_b200.core import Agent
    cfg = builtin.load(config_path)
    kw = dict(cfg.agent, state_size=env.state_size, action_size=env.action_size, optim_config=cfg.optim,
              run_step=1000, device=DEV)
    kw.update(override)
    return Agent(**kw)


def test_ppo_rollout_and_learn():
    from jorldy_b200.core.collect import RolloutCollector
    env = _env(8, seed=1)
    agent = _cfg_agent("config.ppo.cartpole", env, hidden_size=64, n_step=16, batch_size=32, n_epoch=1)
    before = agent.network.flat.clone()
    res = agent.learn_rollout(RolloutCollector(env, agent, use_cuda_graph=False).collect())
    assert res and all(np.isfinite(v) for v in res.values()) and not torch.equal(before, agent.network.flat)


def test_dqn_replay_round_and_learn():
    from jorldy_b200.core.collect import ReplayCollector
    env = _env(8, seed=1)
    agent = _cfg_agent("config.dqn.cartpole", env, hidden_size=64, batch_size=32, buffer_size=1024, start_train_step=0)
    before = agent.network.flat.clone()
    _, res = ReplayCollector(env, agent, update_period=8).run_round(0)
    assert res and all(np.isfinite(v) for v in res.values()) and not torch.equal(before, agent.network.flat)


def test_reinforce_episode_round():
    from jorldy_b200.core.collect import EpisodeCollector
    env = _env(8, seed=1)
    agent = _cfg_agent("config.reinforce.cartpole", env, hidden_size=64)
    col = EpisodeCollector(env, agent, 16, use_cuda_graph=False)
    assert col.ring.L == 5 - 1 + 16
    res = agent.learn_episodes(col.collect())           # 16 steps finish at least 8 games of at most 5 moves
    assert res and all(np.isfinite(v) for v in res.values())


# ------------------------------------------------------------------------------------------- 8. drivers
@pytest.mark.parametrize("mode,extra,final", [
    ("--single", [], 300),
    ("--sync", ["--train.num_workers", "32", "--train.update_period", "4"], 800),
])
def test_training_run_with_save_and_load(tmp_path, mode, extra, final):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base = [sys.executable, "-m", "jorldy_b200.main", mode, "--config", "config.muzero.tictactoe", "--train.run_step",
            str(final), "--train.print_period", str(final // 2), "--train.save_period", str(final),
            "--agent.start_train_step", "200", "--agent.batch_size", "32", "--agent.num_simulation", "8",
            "--agent.hidden_size", "64", "--agent.latent_size", "32", *extra]
    r = subprocess.run(base, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith(f"{final} step |") for line in r.stdout.splitlines()), out[-4000:]
    assert any("policy_loss" in line for line in r.stdout.splitlines() if " step |" in line), out[-4000:]
    ckpts = [d for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    r2 = subprocess.run(base + ["--train.load_path", ckpts[0]], cwd=tmp_path / "logs", env=env, capture_output=True,
                        text=True, timeout=900)
    out2 = r2.stdout + r2.stderr
    assert "Traceback" not in out2 and "Load model from" in out2, out2[-4000:]
