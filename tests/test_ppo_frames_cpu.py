"""PPO on Atari frames, host side: the built-in `config.ppo.atari`, and a pure-Python model of the frame ring's push
positions showing that frames_per_rollout(T) never lets a frame a rollout references be overwritten before it is learned
from (jorldy_b200/core/buffer/frame_store.py)."""
import numpy as np
import pytest

from jorldy_b200.core.buffer.frame_store import frames_per_rollout


def test_ppo_atari_config():
    from jorldy_b200 import config as cfg
    from jorldy_b200.manager import ConfigManager
    assert "config.ppo.atari" in cfg.available()
    c = cfg.load("config.ppo.atari")
    assert c.env == cfg._ATARI_ENV
    assert c.agent == dict(name="ppo", network="discrete_policy_value", head="cnn", gamma=0.99, batch_size=32, n_step=128,
                           n_epoch=3, _lambda=0.95, epsilon_clip=0.1, vf_coef=1.0, ent_coef=0.01, clip_grad_norm=1.0,
                           use_standardization=True, lr_decay=True)
    assert c.optim == dict(name="adam", lr=2.5e-4)
    assert c.train == dict(cfg._TRAIN_ATARI, run_step=30000000, eval_iteration=5, distributed_batch_size=256,
                           update_period=128, num_workers=8)
    m = ConfigManager("config.ppo.atari", ["--env.name", "breakout", "--train.num_workers", "16"])
    assert m.config.env.name == "breakout" and m.config.train.num_workers == 16 and m.config.agent.head == "cnn"


def _rollouts_resident(T, F, done, rollouts=3):
    """Pushes `rollouts` rollouts of T steps into one lane's ring of F frames the way FrameStore.start / push do
    (csrc/frame_ring.cu), and checks at the end of each rollout, when learn_rollout() reads it, that every stack it
    references (the T states and the last next state) is resident by the kernels' rule.  done(r, t) -> bool."""
    first = []                                           # first[p]: episode-first position of the frame at p

    def push(f):
        first.append(f)

    push(0)                                              # start(): the reset frame
    for r in range(rollouts):
        refs = []
        for t in range(T):
            s = len(first) - 1                           # the stack acted on
            push(first[s])                               # the newest frame continues its episode
            nxt = len(first) - 1
            refs.append(s)
            if done(r, t):
                push(len(first))                         # auto-reset: an episode-first frame
        refs.append(nxt)
        h = len(first)
        for p in refs:
            lo = max(p - 3, first[p])
            if not (p < h and lo >= h - F):
                return False
    return True


def _patterns(T):
    rs = np.random.RandomState(T)
    table = rs.rand(3, T) < 0.3
    return {"every": lambda r, t: True, "never": lambda r, t: False,
            "alternating": lambda r, t: (r * T + t) % 2 == 0, "random": lambda r, t: bool(table[r, t]),
            "never_then_every": lambda r, t: r > 0}


@pytest.mark.parametrize("T", [1, 5, 128])
@pytest.mark.parametrize("pattern", ["every", "never", "alternating", "random", "never_then_every"])
def test_frames_per_rollout_keeps_every_reference_resident(T, pattern):
    F = frames_per_rollout(T)
    assert F == max(2 * T + 4, 8)
    assert _rollouts_resident(T, F, _patterns(T)[pattern])


@pytest.mark.parametrize("T", [5, 128])
def test_shorter_rings_lose_references(T):
    """T + 3 frames (one step's frame per state and the stack's three older ones) are not enough once every step ends
    an episode, and 2T + 3 are not enough when a rollout that starts mid-episode then ends one at every step."""
    assert not _rollouts_resident(T, T + 3, _patterns(T)["every"])
    assert not _rollouts_resident(T, 2 * T + 3, _patterns(T)["never_then_every"])
    assert _rollouts_resident(T, 2 * T + 4, _patterns(T)["never_then_every"])
