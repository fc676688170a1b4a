"""Batched TicTacToe on the GPU (csrc/env_tictactoe.cu), registered as `tictactoe`.

The reference ships a `tictactoe` env for MuZero, but its source is not available here: the rules below are this
project's contract (DESIGN.md 5i, "MuZero on TicTacToe").

solve()   the game solved exactly by negamax: the value and the optimal moves of every position, from the side to move
"""
import functools

import numpy as np
import torch

from ..dev import C, ptr, require_cuda, stream_ptr
from .classic import _Classic

LINES = (0x007, 0x038, 0x1C0, 0x049, 0x092, 0x124, 0x111, 0x054)
FULL = 0x1FF
OPPONENTS = {"random": 0, "perfect": 1, "self": 2}          # csrc/env_tictactoe.cu's Opponent


def _line(b):
    return any(b & m == m for m in LINES)


def position(mover, other):
    """The base-3 index of a board from the side to move: digit c (weight 3^c) is 1 for its mark on cell c, 2 for the
    other side's."""
    return sum(3 ** c * (((mover >> c) & 1) + 2 * ((other >> c) & 1)) for c in range(9))


@functools.lru_cache(maxsize=None)
def solve():
    """TicTacToe solved by a memoised negamax from the empty board over the 4 520 non-terminal positions a game can
    reach.  Returns (value int8 [3^9], best uint16 [3^9]), indexed by position(): the negamax value for the side to move
    (win 1 > draw 0 > loss -1, quicker and slower wins alike) and the 9-bit mask of the moves that reach it.  Both are 0
    at terminal, unreachable and malformed indices.  Computed once per process; the arrays are read-only."""
    value, best = np.zeros(3 ** 9, dtype=np.int8), np.zeros(3 ** 9, dtype=np.uint16)
    seen = set()

    def negamax(me, op):               # a non-terminal position, `me` to move
        idx = position(me, op)
        if idx in seen:
            return int(value[idx])
        outcome = {}
        for a in range(9):
            if (me | op) >> a & 1:
                continue
            m = me | 1 << a
            outcome[a] = 1 if _line(m) else 0 if (m | op) == FULL else -negamax(op, m)
        v = max(outcome.values())
        value[idx], best[idx] = v, sum(1 << a for a, x in outcome.items() if x == v)
        seen.add(idx)
        return v

    negamax(0, 0)
    value.setflags(write=False)
    best.setflags(write=False)
    return value, best


class TicTacToe(_Classic):
    """`num_envs` boards stepped by one kernel launch.  `opponent` picks who plays against the agent:

    "random" (the default): the agent plays one side against a uniform-random opponent.

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

    "perfect": as "random", but the opponent plays a uniform optimal move: the k-th of the moves solve() marks optimal,
    k = floor(u n_optimal), u the random opponent's draw at the same counter.  Every cell of the empty board is optimal,
    so its openings are the random opponent's.  Each env uploads solve()'s u16 [3^9] mask table (39 KB).

    "self": two-player self-play.  The agent plays both sides: obs is the board from the side to move (its marks
    first), so a network sees the board as it does against an opponent.  reset: an empty board.  step(a): an occupied
    cell or an action outside 0..8 forfeits (-1 to the mover, done); a line gives +1 and done, a full board 0 and done;
    otherwise 0.  The reward is the mover's.  After any move the sides swap, and next_obs is the board seen by the side
    that did not just move, at done too.  elapsed counts plies (max_steps = 9), and the score (stats[1]) is the first
    player's outcome, +1, 0 or -1.  two_player is True in this mode only.

    Auto-reset, next_obs (the terminal board at done), stats, the int64 / int32 device actions and the numpy
    reset() / step() shapes are those of the classic envs.  The numpy step() raises ValueError on an action outside
    0..8; the device step cannot raise, so such an action forfeits.
    """
    action_type = "discrete"
    action_size = 9
    state_size = 18

    def __init__(self, num_envs=1, seed=0, id=0, device=None, auto_reset=None, render=False, train_mode=True,
                 opponent="random", **kwargs):
        if opponent not in OPPONENTS:
            raise ValueError(f"opponent {opponent!r}: TicTacToe takes one of {sorted(OPPONENTS)}")
        self.device = require_cuda(device)
        self.opponent, self._opp = opponent, OPPONENTS[opponent]
        self.two_player = opponent == "self"
        self.max_steps = 9 if self.two_player else 5
        # the u16 table as int16 (its masks are below 512, so the bits are the same)
        self.best = torch.as_tensor(solve()[1].astype(np.int16), device=self.device) if opponent == "perfect" else None
        self.num_envs, self.seed = int(num_envs), int(seed)
        self.id = int(id) if id is not None else 0
        self.stream_base = self.id << 32
        self.auto_reset = (self.num_envs > 1) if auto_reset is None else bool(auto_reset)
        n, dev = self.num_envs, self.device
        self.boards = torch.zeros(n, 2, dtype=torch.int32, device=dev)   # the agent's / mover's and the other bitboard
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
        args = (ptr(self.boards), ptr(self.obs), ptr(self.legal), ptr(self.elapsed), ptr(self.episode), ptr(self._score),
                ptr(mask), self.seed, self.stream_base, self.num_envs, stream_ptr())
        if self.opponent == "random":
            C.jb_env_tictactoe_reset(*args)
        else:
            C.jb_env_tictactoe_reset_opp(self._opp, ptr(self.best), *args)
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
        args = (ptr(self.boards), ptr(self.obs), ptr(self.legal), ptr(self.elapsed), ptr(self.episode), ptr(self._score),
                ptr(action), self._action_kind(action), ptr(self.next_obs), ptr(self.reward), ptr(self.done),
                ptr(self.stats), int(self.auto_reset), self.seed, self.stream_base, self.num_envs, stream_ptr())
        if self.opponent == "random":
            C.jb_env_tictactoe_step(*args)
        else:
            C.jb_env_tictactoe_step_opp(self._opp, ptr(self.best), *args)
        return self.next_obs, self.reward, self.done

    def step(self, action):
        a = np.asarray(action).reshape(self.num_envs)
        if not np.all((a >= 0) & (a <= 8)):
            raise ValueError(f"action {a.tolist()}: TicTacToe takes cells 0..8")
        return super().step(a)
