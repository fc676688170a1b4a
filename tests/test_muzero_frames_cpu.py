"""MuZero on Atari frames, host side: `config.muzero.atari`, the registry and the rejections, the oracle's action planes
on a hand-built example across an episode start, the oracle's CNN representation against a torch module written from
the spec, and a pure-Python model of the frame rings showing that frames_per_window keeps every frame a live replay
window references resident (jorldy_b200/core/buffer/frame_store.py)."""
import numpy as np
import pytest
import torch

from jorldy_b200.core.buffer.frame_store import frames_per_window
from oracle import muzero_frames as omf


def test_muzero_atari_config():
    from jorldy_b200 import config as cfg
    from jorldy_b200.manager import ConfigManager
    assert "config.muzero.atari" in cfg.available()
    c = cfg.load("config.muzero.atari")
    assert c.env == cfg._ATARI_ENV
    a = c.agent
    assert a["name"] == "muzero" and a["head"] == "cnn"
    assert a["gamma"] == 0.997 and a["num_unroll"] == 5 and a["td_steps"] == 10 and a["num_simulation"] == 50
    assert a["root_dirichlet_alpha"] == 0.25 and a["root_exploration_fraction"] == 0.25
    assert a["alpha"] == 1.0 and a["beta"] == 1.0 and a["value_loss_coef"] == 0.25 and a["batch_size"] == 1024
    assert a["buffer_size"] == 1000000 and a["hidden_size"] == 512 and a["latent_size"] == 256
    assert c.optim == {"name": "adam", "lr": 3e-4}
    assert c.train == dict(cfg._TRAIN_ATARI, update_period=8, num_workers=32)
    learns = c.train["run_step"] // c.train["update_period"]
    assert a["temperature_learns"] == (learns // 2, learns * 3 // 4)
    m = ConfigManager("config.muzero.atari", ["--env.name", "breakout", "--agent.batch_size", "64"])
    assert m.config.env.name == "breakout" and m.config.agent.head == "cnn" and m.config.agent.batch_size == 64
    # the flat configs are unchanged
    for env in ("cartpole", "mountaincar"):
        assert "head" not in cfg.load(f"config.muzero.{env}").agent


@pytest.mark.parametrize("kw, err, match", [
    (dict(state_size=[4, 84, 84]), NotImplementedError, "head='cnn'"),           # frame stacks need the CNN head
    (dict(state_size=4, head="cnn"), NotImplementedError, "frame stacks"),
    (dict(state_size=[8, 84, 84], head="cnn"), ValueError, "stack_frame 4"),
    (dict(state_size=[4, 64, 64], head="cnn"), ValueError, r"\[4, 84, 84\]"),
    (dict(state_size=[4, 84, 84], head="cnn", action_size=19), ValueError, "at most 18"),
    (dict(state_size=[4, 84, 84], head="cnn", action_type="continuous"), ValueError, "discrete"),
])
def test_frame_rejections(kw, err, match):
    from jorldy_b200.core import Agent
    args = dict(action_size=4)
    args.update(kw)
    with pytest.raises(err, match=match):
        Agent("muzero", **args)


def test_action_planes_hand_built_across_an_episode_start():
    """One lane: frames 0..5 of an episode, then a reset at position 6 (the episode-first frame), then frames 7, 8.
    Frame q > 0 of the first episode was produced by action q % 3; the second episode's by 2, then 1."""
    A = 3
    # (stack position p, episode-first f, the lane's last four actions before the act at p) -> the planes * A
    cases = [
        (0, 0, [0, 0, 0, 0], [0, 0, 0, 0]),         # the reset stack: frame 0 tiled x4, no action before any of it
        (2, 0, [0, 0, 1, 2], [0, 0, 1, 2]),         # frames 0, 0, 1, 2: the repeated first frame has no plane
        (5, 0, [2, 0, 1, 2], [2, 0, 1, 2]),         # frames 2..5, all produced in this episode
        (6, 6, [0, 1, 2, 0], [0, 0, 0, 0]),         # the reset frame: every plane zero, whatever came before
        (7, 6, [1, 2, 0, 2], [0, 0, 0, 2]),         # frames 6, 6, 6, 7: only frame 7 follows an action
        (8, 6, [2, 0, 2, 1], [0, 0, 2, 1]),         # frames 6, 6, 7, 8
    ]
    for p, f, hist, want in cases:
        got = omf.action_planes(np.array([hist]), np.array([p]), np.array([f]), A)
        np.testing.assert_array_equal(got.numpy(), np.array([want], dtype=np.float64) / A, err_msg=str((p, f)))
    stacks = np.random.default_rng(0).integers(0, 256, (2, 4, 84, 84), dtype=np.uint8)
    planes = omf.action_planes(np.array([[0, 1, 2, 0], [2, 2, 2, 2]]), np.array([7, 9]), np.array([6, 0]), A)
    x = omf.frame_action_input(stacks, planes)
    assert x.shape == (2, 8, 84, 84) and x.dtype == torch.float64
    np.testing.assert_array_equal(x[:, :4].numpy(), stacks / 255.0)
    assert torch.equal(x[0, 4:7], torch.zeros(3, 84, 84)) and torch.all(x[0, 7] == 0.0)
    assert torch.all(x[1, 4:] == 2 / 3)


def test_oracle_cnn_representation_vs_torch_module():
    Hs, g = 32, torch.Generator().manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Conv2d(8, 32, 8, 4), torch.nn.ReLU(), torch.nn.Conv2d(32, 64, 4, 2),
                              torch.nn.ReLU(), torch.nn.Conv2d(64, 64, 3, 1), torch.nn.ReLU(), torch.nn.Flatten(),
                              torch.nn.Linear(3136, Hs)).double()
    names = ["head.conv1", "head.conv2", "head.conv3", "h.l"]
    layers = [m for m in net if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear))]
    p = {}
    for name, m in zip(names, layers):
        p[f"{name}.weight"], p[f"{name}.bias"] = m.weight.detach(), m.bias.detach()
    stacks = torch.randint(0, 256, (5, 4, 84, 84), generator=g, dtype=torch.uint8)
    planes = omf.action_planes(torch.randint(0, 6, (5, 4), generator=g).numpy(), np.arange(5) + 3, np.zeros(5), 6)
    x = omf.frame_action_input(stacks.numpy(), planes)
    y = net(x)
    ref = (y - y.min(1, keepdim=True).values) / (y.max(1, keepdim=True).values - y.min(1, keepdim=True).values)
    got = omf.represent(p, x)
    np.testing.assert_allclose(got.detach().numpy(), ref.detach().numpy(), rtol=1e-12, atol=1e-12)
    assert float(got.min()) == 0.0 and float(got.max()) == 1.0


def _windows_resident(C, N, L, F, done, steps):
    """Pushes `steps` env steps of N lanes into rings of F frames the way FrameStore.start / push do, emits one window
    per lane and step once L steps are pushed (SequenceAssembler with period 1), keeps the newest C windows (the
    replay ring), and checks after every step that each live window's first stack is resident by the kernels' rule.
    done(lane, t) -> bool."""
    first = [[0] for _ in range(N)]                     # first[e][p]: episode-first position of lane e's frame at p
    states = [[] for _ in range(N)]                     # the stack each step acted on
    live = []                                           # (lane, first step) of the stored windows, oldest first
    for t in range(steps):
        for e in range(N):
            s = len(first[e]) - 1
            states[e].append(s)
            first[e].append(first[e][s])                # the newest frame continues its episode
            if done(e, t):
                first[e].append(len(first[e]))          # auto-reset: an episode-first frame
        if t >= L - 1:
            live = (live + [(e, t - L + 1) for e in range(N)])[-C:]
        for e, t0 in live:
            p, h = states[e][t0], len(first[e])
            lo = max(p - 3, first[e][p])
            if not (p < h and lo >= h - F):
                return False
    return True


def _patterns(C, N, L):
    rs = np.random.RandomState(C + N)
    table = rs.rand(N, 4 * (C // N + L)) < 0.3
    t_last = -(-C // N)                                 # the live windows' first steps start about here
    return {"every": lambda e, t: True, "never": lambda e, t: False, "random": lambda e, t: bool(table[e, t]),
            "never_then_every": lambda e, t: t >= t_last}


@pytest.mark.parametrize("C,N,L", [(64, 4, 16), (60, 8, 7), (33, 1, 3)])
@pytest.mark.parametrize("pattern", ["every", "never", "random", "never_then_every"])
def test_frames_per_window_keeps_every_reference_resident(C, N, L, pattern):
    F = frames_per_window(C, N, L)
    assert F == max(2 * (-(-C // N) + L) + 2, 8)
    assert _windows_resident(C, N, L, F, _patterns(C, N, L)[pattern], steps=3 * (C // N + L))


@pytest.mark.parametrize("C,N,L", [(64, 4, 16), (60, 8, 7)])
def test_a_shorter_ring_loses_a_reference(C, N, L):
    """One frame fewer is not enough once a lane that ran its episode through the oldest live window's stack then ends
    an episode at every step."""
    F = frames_per_window(C, N, L)
    steps = 3 * (C // N + L)
    table = np.zeros((N, steps), dtype=bool)
    table[:, C // N + L + 3:] = True                      # no dones, then one at every step
    done = lambda e, t: bool(table[e, t])
    assert _windows_resident(C, N, L, F, done, steps)
    assert not _windows_resident(C, N, L, F - 1, done, steps)
