"""Every registered task trains (pytest -m gpu): each game of core/env/frames.py::_ACTIONS under config.ppo.atari and
each MuJoCo name of core/env/synth.py::_DIMS under PPO, DDPG, TD3 and SAC runs one collect and one learn at small
sizes, with finite results and moved parameters; jb_mlp_in_fwd takes every observation width up to 32."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from jorldy_b200.core.env.frames import _ACTIONS
from jorldy_b200.core.env.synth import _DIMS

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _agent_for(config_path, env, **override):
    """The agent `main` builds for this config and env (run_mode._agent_config), with small sizes."""
    from jorldy_b200 import config as builtin
    from jorldy_b200.core import Agent
    cfg = builtin.load(config_path)
    kw = dict(cfg.agent, state_size=env.state_size, action_size=env.action_size, optim_config=cfg.optim,
              run_step=1000, device=DEV)
    kw.update(override)
    return Agent(**kw)


def _params(agent):
    nets = [agent.network] if hasattr(agent, "network") else [agent.actor, *agent.critics]
    return [n.flat.detach().clone() for n in nets]


def _moved_and_finite(agent, before, res):
    assert res, "no learn happened"
    assert all(np.isfinite(v) for v in res.values()), res
    after = _params(agent)
    assert all(bool(torch.isfinite(a).all()) for a in after)
    assert any(not torch.equal(a, b) for a, b in zip(after, before))   # TD3 delays its actor's first update


@pytest.mark.parametrize("game", sorted(_ACTIONS))
def test_ppo_atari_collect_and_learn(game):
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import RolloutCollector
    env = Env(game, num_envs=8, seed=1, device=DEV)
    agent = _agent_for("config.ppo.atari", env, hidden_size=64, n_step=8, batch_size=16, n_epoch=1)
    assert agent.action_size == _ACTIONS[game]
    before = _params(agent)
    ro = RolloutCollector(env, agent, use_cuda_graph=False).collect()
    assert int(ro.action.max().item()) < _ACTIONS[game]
    _moved_and_finite(agent, before, agent.learn_rollout(ro))


@pytest.mark.parametrize("task", sorted(_DIMS))
def test_ppo_mujoco_collect_and_learn(task):
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import RolloutCollector
    env = Env(task, num_envs=8, seed=1, device=DEV)
    agent = _agent_for("config.ppo.mujoco", env, hidden_size=64, n_step=16, batch_size=32, n_epoch=1)
    assert (agent.state_size, agent.action_size) == _DIMS[task]
    before = _params(agent)
    _moved_and_finite(agent, before, agent.learn_rollout(RolloutCollector(env, agent, use_cuda_graph=False).collect()))


@pytest.mark.parametrize("task", sorted(_DIMS))
@pytest.mark.parametrize("algo", ["ddpg", "td3", "sac"])
def test_off_policy_mujoco_act_fill_and_learn(algo, task):
    """8 envs x 8 steps into the replay, then one process() that learns once on a batch of 32."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    env = Env(task, num_envs=8, seed=1, device=DEV)
    agent = _agent_for(f"config.{algo}.mujoco", env, hidden_size=64, batch_size=32, buffer_size=1024,
                       start_train_step=0)
    before = _params(agent)
    _, res = ReplayCollector(env, agent, update_period=8).run_round(0)
    _moved_and_finite(agent, before, res)


@pytest.mark.parametrize("D", [1, 16, 17, 32])
@pytest.mark.parametrize("gather", [False, True])
def test_mlp_in_fwd_widths_vs_float64(D, gather):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(D)
    R, M, H = 300, 257, 200
    x = torch.as_tensor(rs.standard_normal((R, D)).astype(np.float32), device=DEV)
    w = torch.as_tensor((rs.standard_normal((H, D)) / np.sqrt(D)).astype(np.float32), device=DEV)
    b = torch.as_tensor((0.1 * rs.standard_normal(H)).astype(np.float32), device=DEV)
    idx = torch.as_tensor(rs.randint(0, R, M).astype(np.int32), device=DEV) if gather else None
    h1, xg = torch.empty(M, H, device=DEV), torch.empty(M, D, device=DEV)
    C.jb_mlp_in_fwd(ptr(x), ptr(idx), ptr(w), ptr(b), M, D, H, ptr(h1), ptr(xg), stream_ptr())
    torch.cuda.synchronize()
    rows = x[idx.long()] if gather else x[:M]
    ref = torch.relu(rows.double() @ w.double().T + b.double())
    assert torch.equal(xg, rows)
    torch.testing.assert_close(h1.double(), ref, rtol=1e-5, atol=1e-5)


def test_mlp_in_fwd_rejects_33_inputs():
    from jorldy_b200._lib import JbError
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    x, w, b, h = (torch.zeros(n, device=DEV) for n in (33, 33 * 4, 4, 4))
    with pytest.raises(JbError):
        C.jb_mlp_in_fwd(ptr(x), 0, ptr(w), ptr(b), 1, 33, 4, ptr(h), 0, stream_ptr())


@pytest.mark.parametrize("config_path, task, extra", [
    ("config.sac.mujoco", "half_cheetah", ["--agent.batch_size", "32", "--agent.start_train_step", "256",
                                           "--agent.hidden_size", "64"]),
    ("config.ppo.mujoco", "walker", ["--agent.n_step", "32", "--agent.batch_size", "64", "--agent.hidden_size", "64"]),
])
def test_sync_training_run_on_17_dim_tasks(tmp_path, config_path, task, extra):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable, "-m", "jorldy_b200.main", "--sync", "--config", config_path, "--env.name", task,
           "--train.num_workers", "16", "--train.run_step", "1024", "--train.print_period", "512",
           "--train.save_period", "1024", "--train.update_period", "32", "--train.distributed_batch_size", "64", *extra]
    r = subprocess.run(cmd, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith("1024 step |") for line in r.stdout.splitlines()), out[-4000:]
