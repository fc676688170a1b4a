"""numpy batch TicTacToe — TEST INFRASTRUCTURE, never imported by the product.

Restates the rules of jorldy_b200/core/env/tictactoe.py (csrc/env_tictactoe.cu) with the same state and the same Philox
draws (oracle/philox.py), so the GPU env can be checked against it bit for bit.

LINES                     the 8 winning lines as 9-bit masks (bit c = cell c, row-major)
opening(u_open, u_cell)   the opponent's opening cell, or -1 when it does not open
opponent_cell(empty, u)   the k-th empty cell, k = floor(u n_empty)
TicTacToeBatch            N boards: reset(mask), step(action) -> (next_obs, reward, done), obs / legal / stats
"""
import numpy as np

from .philox import philox4x32, u01_double

LINES = (0x007, 0x038, 0x1C0, 0x049, 0x092, 0x124, 0x111, 0x054)
FULL = 0x1FF


def has_line(b):
    return any((int(b) & m) == m for m in LINES)


def opening(u_open, u_cell):
    return min(int(u_cell * 9.0), 8) if u_open < 0.5 else -1


def opponent_cell(empty, u):
    cells = [c for c in range(9) if (int(empty) >> c) & 1]
    return cells[min(int(u * len(cells)), len(cells) - 1)]


def draws(seed, stream, episode, move):
    """The two uniforms of Philox (seed, stream) at counter (episode << 4) | move; array arguments broadcast."""
    ctr = (np.asarray(episode).astype(np.uint64) << np.uint64(4)) | np.asarray(move).astype(np.uint64)
    x, y, z, w = philox4x32(seed, np.asarray(stream, dtype=np.uint64), ctr)
    return u01_double(x, y), u01_double(z, w)


def board_obs(me, op):
    return np.array([(int(me) >> c) & 1 for c in range(9)] + [(int(op) >> c) & 1 for c in range(9)], dtype=np.float32)


class TicTacToeBatch:
    def __init__(self, n, seed=0, id=0, auto_reset=True):
        self.n, self.seed, self.stream_base, self.auto_reset = n, seed, id << 32, auto_reset
        self.boards = np.zeros((n, 2), dtype=np.int32)
        self.elapsed = np.zeros(n, dtype=np.int32)
        self.episode = np.zeros(n, dtype=np.int64)
        self.score = np.zeros(n, dtype=np.float32)
        self.stats = np.zeros(2, dtype=np.float32)

    @property
    def obs(self):
        return np.stack([board_obs(me, op) for me, op in self.boards])

    @property
    def legal(self):
        return (1 - (self.obs[:, :9] + self.obs[:, 9:])).astype(np.uint8)

    def _streams(self, idx):
        return np.uint64(self.stream_base) | np.asarray(idx).astype(np.uint64)

    def _new_games(self, idx):
        idx = np.asarray(idx, dtype=np.int64)
        self.episode[idx] += 1
        u_open, u_cell = draws(self.seed, self._streams(idx), self.episode[idx], 0)
        for j, i in enumerate(idx):
            c = opening(u_open[j], u_cell[j])
            self.boards[i] = (0, 0 if c < 0 else 1 << c)
            self.elapsed[i], self.score[i] = 0, 0.0

    def _reply_uniforms(self):
        """The uniform of every board's opponent reply to the move it is about to take."""
        idx = np.arange(self.n)
        return draws(self.seed, self._streams(idx), self.episode, self.elapsed.astype(np.int64) + 1)[0]

    def reset(self, mask=None):
        self._new_games([i for i in range(self.n) if mask is None or mask[i]])
        return self.obs

    def step(self, action):
        action = np.asarray(action).reshape(self.n)
        next_obs = np.zeros((self.n, 18), dtype=np.float32)
        reward, done = np.zeros(self.n, dtype=np.float32), np.zeros(self.n, dtype=np.float32)
        u_reply, finished = self._reply_uniforms(), []
        for i in range(self.n):
            me, op = (int(v) for v in self.boards[i])
            a = int(action[i])
            el = int(self.elapsed[i]) + 1
            r, d = 0.0, True
            if a < 0 or a > 8 or ((me | op) >> a) & 1:
                r = -1.0
            else:
                me |= 1 << a
                if has_line(me):
                    r = 1.0
                elif (me | op) != FULL:
                    op |= 1 << opponent_cell(FULL & ~(me | op), u_reply[i])
                    if has_line(op):
                        r = -1.0
                    else:
                        d = (me | op) == FULL
            sc = np.float32(self.score[i] + np.float32(r))
            next_obs[i] = board_obs(me, op)
            reward[i], done[i] = r, float(d)
            self.boards[i] = (me, op)
            self.elapsed[i], self.score[i] = el, sc
            if d and self.auto_reset:
                self.stats += np.array([1.0, sc], dtype=np.float32)
                finished.append(i)
        self._new_games(finished)
        return next_obs, reward, done
