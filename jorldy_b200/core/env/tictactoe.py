"""Batched TicTacToe on the GPU (csrc/env_tictactoe.cu), registered as `tictactoe`.

The reference ships a `tictactoe` env for MuZero, but its source is not available here: the rules below are this
project's contract (DESIGN.md 5i, "MuZero on TicTacToe").
"""
import numpy as np
import torch

from ..dev import C, ptr, require_cuda, stream_ptr
from .classic import _Classic


class TicTacToe(_Classic):
    """The agent plays one side against a uniform-random opponent; `num_envs` boards are stepped by one kernel launch.

    - obs f32 [N, 18]: cells 0..8 are 1 where the agent has a mark, 9..17 where the opponent has one (row-major 3x3).
    - legal u8 [N, 9]: the empty cells of `obs`, updated in place by every reset and step (a captured graph reads it by
      pointer).
    - reset: an empty board; one Philox draw decides, with probability 1/2, whether the opponent opens, on a uniform cell.
    - step(a): an occupied cell or an action outside 0..8 forfeits (reward -1, done).  Otherwise the agent's mark: a line
      gives +1 and done, a full board 0 and done.  Otherwise the opponent marks a uniform empty cell (the k-th empty one,
      k = floor(u n_empty)): its line gives -1 and done, a full board 0 and done.  Otherwise the reward is 0.
    - Draws come from the env's own Philox stream (id << 32 | env) at a counter built from the episode and the move, so
      every episode, and every replay of a captured collect, draws fresh numbers.
    - Every game ends within the agent's 5th move (max_steps = 5).

    Auto-reset, next_obs (the terminal board at done), stats, the int64 / int32 device actions and the numpy
    reset() / step() shapes are those of the classic envs.  The numpy step() raises ValueError on an action outside
    0..8; the device step cannot raise, so such an action forfeits.
    """
    action_type = "discrete"
    action_size = 9
    state_size = 18
    max_steps = 5

    def __init__(self, num_envs=1, seed=0, id=0, device=None, auto_reset=None, render=False, train_mode=True,
                 **kwargs):
        self.device = require_cuda(device)
        self.num_envs, self.seed = int(num_envs), int(seed)
        self.id = int(id) if id is not None else 0
        self.stream_base = self.id << 32
        self.auto_reset = (self.num_envs > 1) if auto_reset is None else bool(auto_reset)
        n, dev = self.num_envs, self.device
        self.boards = torch.zeros(n, 2, dtype=torch.int32, device=dev)       # the agent's and the opponent's bitboards
        self.obs = torch.zeros(n, self.state_size, dtype=torch.float32, device=dev)
        self.legal = torch.zeros(n, self.action_size, dtype=torch.uint8, device=dev)
        self.elapsed = torch.zeros(n, dtype=torch.int32, device=dev)
        self.episode = torch.zeros(n, dtype=torch.int64, device=dev)
        self._score = torch.zeros(n, dtype=torch.float32, device=dev)
        self.next_obs = torch.zeros(n, self.state_size, dtype=torch.float32, device=dev)
        self.reward = torch.zeros(n, dtype=torch.float32, device=dev)
        self.done = torch.zeros(n, dtype=torch.float32, device=dev)
        self.stats = torch.zeros(2, dtype=torch.float32, device=dev)   # episodes finished, sum of scores
        self.render = render

    def reset_device(self, mask=None):
        C.jb_env_tictactoe_reset(ptr(self.boards), ptr(self.obs), ptr(self.legal), ptr(self.elapsed), ptr(self.episode),
                                 ptr(self._score), ptr(mask), self.seed, self.stream_base, self.num_envs, stream_ptr())
        return self.obs

    def _action_kind(self, action):
        if action.dtype == torch.int64:
            return 0
        if action.dtype == torch.int32:
            return 1
        raise TypeError(f"unsupported action dtype {action.dtype}: TicTacToe takes int64 or int32 cells")

    def step_device(self, action):
        """action: int64 / int32 device tensor [N] / [N, 1].  Returns (next_obs, reward, done), overwritten by the next
        call; `self.obs` and `self.legal` then hold the board to act on next (post auto-reset where done)."""
        C.jb_env_tictactoe_step(ptr(self.boards), ptr(self.obs), ptr(self.legal), ptr(self.elapsed), ptr(self.episode),
                                ptr(self._score), ptr(action), self._action_kind(action), ptr(self.next_obs),
                                ptr(self.reward), ptr(self.done), ptr(self.stats), int(self.auto_reset), self.seed,
                                self.stream_base, self.num_envs, stream_ptr())
        return self.next_obs, self.reward, self.done

    def step(self, action):
        a = np.asarray(action).reshape(self.num_envs)
        if not np.all((a >= 0) & (a <= 8)):
            raise ValueError(f"action {a.tolist()}: TicTacToe takes cells 0..8")
        return super().step(a)
