"""Synthetic Atari-shaped env (csrc/env_frames.cu): the observation contract of
jorldy/core/env/atari.py — state (N, 4, 84, 84) uint8 with the newest frame last, sign-clipped reward,
episodic done, first state = first frame tiled x4 — fed by a Philox frame generator instead of ALE
(north star: "Atari paths fed by a synthetic 84x84x4 uint8 frame generator of identical dtype/layout").
Registered under the reference's Atari env names so `--env.name breakout` style configs resolve; the
action set size per game follows ALE's minimal action sets."""
import numpy as np
import torch

from ..dev import C, ptr, require_cuda, stream_ptr
from .base import BaseEnv

_ACTIONS = {"breakout": 4, "pong": 6, "asterix": 9, "assault": 7, "seaquest": 18, "spaceinvaders": 6, "alien": 18,
            "crazy_climber": 9, "enduro": 9, "qbert": 6, "private_eye": 18, "montezuma_revenge": 18}


class SyntheticAtari(BaseEnv):
    action_type = "discrete"
    # frame-stack contract: obs / next_obs are [N,4,84,84] stacks whose slot 3 is the newest frame and slots 0..2 the
    # previous stack's 1..3, and a reset stack is its first frame tiled x4, so a replay can store each frame once
    # (buffer/frame_store.py)
    frame_stack = True

    def __init__(self, name="breakout", num_envs=1, seed=0, id=0, device=None, auto_reset=None, img_width=84,
                 img_height=84, stack_frame=4, action_size=None, train_mode=True, **kwargs):
        assert img_width == 84 and img_height == 84 and stack_frame == 4, "generator is fixed at 4x84x84"
        self.device = require_cuda(device)
        self.name = name
        self.num_envs = int(num_envs)
        self.seed = int(seed)
        self.id = int(id) if id is not None else 0
        self.stream_base = self.id << 32
        self.auto_reset = (self.num_envs > 1) if auto_reset is None else bool(auto_reset)
        self.state_size = [4, 84, 84]
        self.action_size = int(action_size) if action_size else _ACTIONS.get(name, 4)
        n, dev = self.num_envs, self.device
        self.obs = torch.zeros(n, 4, 84, 84, dtype=torch.uint8, device=dev)
        self.next_obs = torch.zeros(n, 4, 84, 84, dtype=torch.uint8, device=dev)
        self.fcount = torch.zeros(n, dtype=torch.int64, device=dev)
        self._score = torch.zeros(n, dtype=torch.float32, device=dev)
        self.reward = torch.zeros(n, dtype=torch.float32, device=dev)
        self.done = torch.zeros(n, dtype=torch.float32, device=dev)
        self.stats = torch.zeros(2, dtype=torch.float32, device=dev)

    def reset_device(self, mask=None):
        C.jb_env_frames_reset(ptr(self.obs), ptr(self.fcount), ptr(self._score), self.seed, self.stream_base,
                              self.num_envs, stream_ptr())
        return self.obs

    def step_device(self, action=None):
        C.jb_env_frames_step(ptr(self.obs), ptr(self.fcount), ptr(self._score), ptr(self.next_obs), ptr(self.reward),
                             ptr(self.done), ptr(self.stats), int(self.auto_reset), self.seed, self.stream_base,
                             self.num_envs, stream_ptr())
        return self.next_obs, self.reward, self.done

    @property
    def score(self):
        s = self._score.cpu().numpy()
        return float(s[0]) if self.num_envs == 1 else s

    def reset(self):
        return self.reset_device().cpu().numpy()

    def step(self, action):
        next_obs, reward, done = self.step_device(None)
        n = self.num_envs
        return (next_obs.cpu().numpy(), reward.view(n, 1).cpu().numpy().astype(np.float64),
                done.view(n, 1).cpu().numpy() > 0.5)

    def close(self):
        pass
