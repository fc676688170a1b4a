"""numpy TicTacToe self-play, the perfect opponent and two-player MuZero search in float64 — TEST INFRASTRUCTURE, never
imported by the product.

Restates the `opponent="self"` and `opponent="perfect"` modes of jorldy_b200/core/env/tictactoe.py
(csrc/env_tictactoe.cu) with the same state and the same Philox draws as oracle/tictactoe.py, which it leaves unchanged,
and the two-player search the way the MuZero pseudocode (arXiv:1911.08265) writes it, with the value flipped to the
parent's side at every ply, so that the product's "single-player kernels at -gamma" can be checked against it.

position(mover, other)      base-3 index from the side to move: digit c (weight 3^c) is 1 for its mark, 2 for the other's
enumerate_solution()        every reachable position's negamax value and optimal-move mask by a full game-tree walk
                            (no memo, no shared code with the product's solve())
SelfPlayBatch               N self-play boards: reset(mask), step(action) -> (next_obs, reward, done), obs / legal / stats
PerfectBatch                oracle/tictactoe.py's TicTacToeBatch whose opponent plays the k-th optimal cell
TwoPlayerTree               oracle/muzero.py's Tree with the pseudocode's negamax backup; TwoPlayerLegalTree adds the
                            masked root of oracle/muzero_legal.py
search_two_player()         oracle/muzero_legal.py's search_legal() on the two-player tree
targets_two_player()        the n-step value targets with the side flipped at every ply
game_step(), exact_search() the true game as a search model: exact rewards, value 0 at every leaf
"""
import numpy as np
import torch

from . import muzero as om
from . import muzero_legal as ol
from .tictactoe import FULL, TicTacToeBatch, board_obs, has_line


def position(mover, other):
    idx = 0
    for c in range(9):
        if (mover >> c) & 1:
            idx += 3 ** c
        elif (other >> c) & 1:
            idx += 2 * 3 ** c
    return idx


# ------------------------------------------------------------------------------------------------------ the solution
def enumerate_solution():
    """Walks every game from the empty board (x moves first).  Returns (positions, value, best): the set of (mover,
    other) boards reached, including terminal ones, and dicts {(mover, other): value / optimal mask} over the
    non-terminal ones, value in {-1, 0, 1} for the side to move."""
    positions, value, best = set(), {}, {}

    def walk(x, o, x_moves):
        mover, other = (x, o) if x_moves else (o, x)
        positions.add((mover, other))
        if has_line(x) or has_line(o) or (x | o) == FULL:
            return None
        results = []
        for a in range(9):
            if (x | o) >> a & 1:
                continue
            nx, no = (x | 1 << a, o) if x_moves else (x, o | 1 << a)
            child = walk(nx, no, not x_moves)
            moved = nx if x_moves else no
            results.append((a, 1 if has_line(moved) else 0 if child is None else -child))
        v = max(r for _, r in results)
        value[(mover, other)] = v
        best[(mover, other)] = sum(1 << a for a, r in results if r == v)
        return v

    walk(0, 0, True)
    return positions, value, best


# ------------------------------------------------------------------------------------------------------ the envs
class SelfPlayBatch:
    """boards[i] = (side to move, other side); elapsed counts plies; score is the first player's outcome."""

    def __init__(self, n, auto_reset=True):
        self.n, self.auto_reset = n, auto_reset
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

    def _new_games(self, idx):
        for i in idx:
            self.episode[i] += 1
            self.boards[i] = (0, 0)
            self.elapsed[i], self.score[i] = 0, 0.0

    def reset(self, mask=None):
        self._new_games([i for i in range(self.n) if mask is None or mask[i]])
        return self.obs

    def step(self, action):
        action = np.asarray(action).reshape(self.n)
        next_obs = np.zeros((self.n, 18), dtype=np.float32)
        reward, done = np.zeros(self.n, dtype=np.float32), np.zeros(self.n, dtype=np.float32)
        finished = []
        for i in range(self.n):
            me, op = (int(v) for v in self.boards[i])
            a, el = int(action[i]), int(self.elapsed[i]) + 1
            if a < 0 or a > 8 or ((me | op) >> a) & 1:
                r, d = -1.0, True
            else:
                me |= 1 << a
                r, d = (1.0, True) if has_line(me) else (0.0, (me | op) == FULL)
            first = r if el % 2 == 1 else -r              # the first player moves on odd plies
            sc = np.float32(self.score[i] + np.float32(first))
            me, op = op, me                               # the other side moves next
            next_obs[i] = board_obs(me, op)
            reward[i], done[i] = r, float(d)
            self.boards[i] = (me, op)
            self.elapsed[i], self.score[i] = el, sc
            if d and self.auto_reset:
                self.stats += np.array([1.0, sc], dtype=np.float32)
                finished.append(i)
        self._new_games(finished)
        return next_obs, reward, done


def perfect_cell(best_mask, u):
    """The k-th optimal cell, k = floor(u n_optimal)."""
    cells = [c for c in range(9) if (int(best_mask) >> c) & 1]
    return cells[min(int(u * len(cells)), len(cells) - 1)]


class PerfectBatch(TicTacToeBatch):
    """TicTacToeBatch whose opponent plays perfect_cell(best[position(opponent, agent)], u) with the random opponent's
    uniform u.  best: {(mover, other): optimal mask} (enumerate_solution()).  The opening is the random opponent's: every
    cell of the empty board is optimal.  A board stepped after its game ended is not in `best`: the opponent then
    chooses among the empty cells."""

    def __init__(self, n, best, seed=0, id=0, auto_reset=True):
        super().__init__(n, seed=seed, id=id, auto_reset=auto_reset)
        assert best[(0, 0)] == FULL
        self.best = best

    def step(self, action):
        action = np.asarray(action).reshape(self.n)
        next_obs = np.zeros((self.n, 18), dtype=np.float32)
        reward, done = np.zeros(self.n, dtype=np.float32), np.zeros(self.n, dtype=np.float32)
        u_reply, finished = self._reply_uniforms(), []
        for i in range(self.n):
            me, op = (int(v) for v in self.boards[i])
            a, el = int(action[i]), int(self.elapsed[i]) + 1
            r, d = 0.0, True
            if a < 0 or a > 8 or ((me | op) >> a) & 1:
                r = -1.0
            else:
                me |= 1 << a
                if has_line(me):
                    r = 1.0
                elif (me | op) != FULL:
                    op |= 1 << perfect_cell(self.best.get((op, me), 0) or FULL & ~(me | op), u_reply[i])
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


# ------------------------------------------------------------------------------------------------------ the search
class TwoPlayerTree(om.Tree):
    """The pseudocode's two-player backup: every value is the mover's, and an edge's W holds its child's value seen
    from the parent's side, so the value is negated at each ply."""

    def expand_backup(self, latent, pi_logits, reward, value, gamma):
        nn = self.count
        node, a = self.path[-1]
        self.latent[nn] = latent
        self.p[nn] = om._softmax(pi_logits)
        self.child[node, a] = nn
        self.r[node, a] = reward
        self.count += 1
        g = value                                   # the leaf mover's value
        for node, a in reversed(self.path):
            self.w[node, a] += -g                   # seen by the parent's mover
            self.n[node, a] += 1
            q = self.r[node, a] + gamma * self.w[node, a] / self.n[node, a]
            self.qmin, self.qmax = min(self.qmin, q), max(self.qmax, q)
            g = self.r[node, a] - gamma * g         # the parent mover's return


class TwoPlayerLegalTree(TwoPlayerTree, ol.LegalTree):
    """TwoPlayerTree with oracle/muzero_legal.py's masked root."""


def search_two_player(root_pi_logits, root_latent, model, A, S, gamma, V, R, legal, noise=None, frac=0.25,
                      training=False, temperature=1.0, u=None, margins=None):
    """oracle/muzero_legal.py's search_legal() on TwoPlayerLegalTree; same arguments and returns."""
    t = TwoPlayerLegalTree(A, S, legal)
    t.p[0] = ol.root_prior(root_pi_logits, t.legal, noise, frac)
    t.latent[0] = root_latent
    for sim in range(S):
        node, a, scores = t.select(gamma)
        finite = np.sort(np.asarray([x for x in scores if np.isfinite(x)]))[::-1]
        if margins is not None and sim > 0 and finite.size > 1:
            margins.append(finite[0] - finite[1])
        latent, pi_l, v_l, r_l = model(sim, t.latent[node], a)
        r = float(om.support_to_scalar(torch.as_tensor(r_l), R))
        v = float(om.support_to_scalar(torch.as_tensor(v_l), V))
        t.expand_backup(latent, pi_l, r, v, gamma)
    a, pi, rv = t.act(gamma, training, temperature, u)
    return t, a, pi, rv


def targets_two_player(reward, done, root_value, K, n, gamma):
    """oracle/muzero.py targets() with the side flipped at every ply: the value at step k + i + 1 is the opponent's, so
    it enters the mover's return negated.  z = r_k - gamma r_{k+1} + ... + (-gamma)^n v_{k+n}, cut at the first done."""
    reward, done, root_value = (np.asarray(t, dtype=np.float64) for t in (reward, done, root_value))
    B = reward.shape[0]
    z, u = np.zeros((B, K + 1)), np.zeros((B, K + 1))
    absorbing = np.zeros((B, K + 1), dtype=bool)
    for b in range(B):
        for k in range(K + 1):
            absorbing[b, k] = bool(np.any(done[b, :k] != 0))
            if not absorbing[b, k]:
                g = root_value[b, k + n]                 # the mover's at step k + n
                for i in reversed(range(n)):
                    g = reward[b, k + i] if done[b, k + i] else reward[b, k + i] - gamma * g
                z[b, k] = g
            if k > 0 and not (k >= 2 and absorbing[b, k - 1]):
                u[b, k] = reward[b, k - 1]
    return z, u, absorbing


# ------------------------------------------------------------------------------------------------------ exact model
def game_step(state, a):
    """The true self-play game as a search model.  state (mover, other, terminal) -> (next state from the next mover's
    side, the mover's reward).  A terminal state is absorbing with reward 0; an occupied cell forfeits (-1)."""
    me, op, term = state
    if term:
        return (op, me, True), 0.0
    if (me | op) >> a & 1:
        return (op, me, True), -1.0
    me |= 1 << a
    if has_line(me):
        return (op, me, True), 1.0
    return (op, me, (me | op) == FULL), 0.0


def exact_search(me, op, S, gamma, two_player):
    """The masked-root search of the non-terminal board (me to move) with the true game as its model: uniform priors,
    exact rewards and value 0 at every leaf.  two_player: the pseudocode's two-player tree, else the single-player
    backup.  Returns the greedy action."""
    legal = [not ((me | op) >> a & 1) for a in range(9)]
    t = (TwoPlayerLegalTree if two_player else ol.LegalTree)(9, S, legal)
    t.p[0] = ol.root_prior(np.zeros(9), legal)
    t.latent[0] = (me, op, False)
    zeros = np.zeros(9)
    for _ in range(S):
        node, a, _ = t.select(gamma)
        latent, r = game_step(t.latent[node], a)
        t.expand_backup(latent, zeros, r, 0.0, gamma)
    return t.act(gamma, False)[0]


def optimal_move_rate(best, S, gamma, two_player):
    """The share of the non-terminal positions of `best` ({(mover, other): optimal mask}) where exact_search() picks
    an optimal move."""
    hits = sum((best[key] >> exact_search(*key, S, gamma, two_player)) & 1 for key in best)
    return hits / len(best)

