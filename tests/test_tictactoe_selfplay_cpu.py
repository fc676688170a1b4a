"""Two-player TicTacToe without a GPU: `config.muzero.tictactoe_selfplay`, the self-play rules of the oracle env on
scripted games, the product's solve() against an independent full game-tree walk, the identity between the two-player
search and targets and the single-player ones at -gamma (bit for bit in float64), and the optimal-move rate of the
search with the true game as its model."""
import itertools

import numpy as np
import pytest
import torch

from oracle import muzero as om
from oracle import muzero_legal as ol
from oracle import tictactoe as ot
from oracle import tictactoe_selfplay as ts


def test_config_and_registry():
    from jorldy_b200 import config as cfg
    assert "config.muzero.tictactoe_selfplay" in cfg.available()
    c, base = cfg.load("config.muzero.tictactoe_selfplay"), cfg.load("config.muzero.tictactoe")
    assert c.env == {"name": "tictactoe", "render": False, "opponent": "self"}
    assert c.agent["two_player"] is True and c.agent["td_steps"] == 9 and c.agent["gamma"] == 1.0
    changed = {k for k in set(base.agent) | set(c.agent) if base.agent.get(k) != c.agent.get(k)}
    assert changed == {"two_player", "td_steps"}
    assert c.optim == base.optim and c.train == base.train
    assert base.env == {"name": "tictactoe", "render": False} and "two_player" not in base.agent


def test_env_rejects_an_unknown_opponent():
    from jorldy_b200.core.env.tictactoe import TicTacToe
    with pytest.raises(ValueError):
        TicTacToe(opponent="minimax")


# ------------------------------------------------------------------------------------------- self-play rules
def _selfplay(moves):
    """Plays `moves` (alternating sides, the first player first) on one board; returns the per-ply (next_obs, reward,
    done) and the env."""
    env = ts.SelfPlayBatch(1, auto_reset=False)
    env.reset()
    out = []
    for a in moves:
        ns, r, d = env.step([a])
        out.append((ns[0], float(r[0]), bool(d[0])))
        if d[0]:
            break
    return out, env


def _cells(mask):
    return [c for c in range(9) if (mask >> c) & 1]


def _filler(line, k):
    """k cells off `line` that hold no line of their own."""
    for cells in itertools.combinations([c for c in range(9) if not (line >> c) & 1], k):
        if not ot.has_line(sum(1 << c for c in cells)):
            return list(cells)


@pytest.mark.parametrize("line", ot.LINES)
@pytest.mark.parametrize("first", [True, False])
def test_every_line_wins_for_either_player(line, first):
    win = _cells(line)
    other = _filler(line, 2 if first else 3)
    pairs = itertools.zip_longest(win, other) if first else zip(other, win)
    moves = [c for pair in pairs for c in pair if c is not None]
    out, env = _selfplay(moves)
    assert len(out) == (5 if first else 6)
    assert [r for _, r, _ in out] == [0.0] * (len(out) - 1) + [1.0]          # the mover's reward
    assert [d for _, _, d in out] == [False] * (len(out) - 1) + [True]
    assert env.score[0] == (1.0 if first else -1.0)                           # the first player's outcome
    assert env.elapsed[0] == len(out)
    ns = out[-1][0]                                                           # seen by the side that did not move
    assert sum(int(ns[9 + c]) << c for c in range(9)) & line == line
    assert ns[:9].sum() == len(other)


def test_draw():
    moves = [0, 4, 8, 1, 7, 6, 2, 5, 3]
    out, env = _selfplay(moves)
    assert len(out) == 9 and all(r == 0.0 for _, r, _ in out)
    assert [d for _, _, d in out] == [False] * 8 + [True]
    assert env.score[0] == 0.0 and env.elapsed[0] == 9
    assert out[-1][0].sum() == 9 and out[-1][0][9:].sum() == 5               # the first player moved last


@pytest.mark.parametrize("moves,score", [([9], -1.0), ([-1], -1.0), ([4, 4], 1.0), ([0, 4, 0], -1.0),
                                         ([0, 4, 8, 8], 1.0)])
def test_forfeit_by_either_side(moves, score):
    out, env = _selfplay(moves)
    assert len(out) == len(moves)
    assert out[-1][1:] == (-1.0, True) and all(r == 0.0 and not d for _, r, d in out[:-1])
    assert env.score[0] == score
    ns = out[-1][0]                                  # the board is unchanged, seen by the side that did not forfeit
    before = moves[:-1]
    mover_cells = before[len(before) % 2::2]          # the forfeiting side's earlier marks
    assert sorted(np.flatnonzero(ns[9:]).tolist()) == sorted(mover_cells)
    assert ns.sum() == len(before)


def test_perspective_swaps_every_ply():
    env = ts.SelfPlayBatch(1, auto_reset=False)
    assert env.reset()[0].sum() == 0
    ns, r, d = env.step([4])
    assert ns[0][13] == 1 and ns[0][:9].sum() == 0 and np.array_equal(env.obs, ns)     # the second player to move
    assert np.array_equal(env.legal[0], 1 - ns[0][:9] - ns[0][9:])
    ns, r, d = env.step([0])
    assert ns[0][4] == 1 and ns[0][9] == 1 and ns[0].sum() == 2                       # the first player again
    assert env.elapsed[0] == 2


def test_auto_reset_and_stats():
    env = ts.SelfPlayBatch(2, auto_reset=True)
    env.reset()
    for a in ([0, 0], [3, 9], [1, 1], [4, 4], [2, 2]):      # board 1: the second player forfeits at ply 2
        env.step(a)
    assert env.stats.tolist() == [2.0, 2.0]                  # board 0: the first player's top row; board 1: +1 too
    assert env.episode.tolist() == [2, 2] and env.elapsed.tolist() == [0, 3]


# ------------------------------------------------------------------------------------------- the solution
@pytest.fixture(scope="module")
def solution():
    return ts.enumerate_solution()


def test_solve_matches_the_full_tree_walk(solution):
    from jorldy_b200.core.env.tictactoe import position, solve
    positions, value, best = solution
    assert len(positions) == 5478 and len(positions) - len(best) == 958 and len(best) == 4520
    v, b = solve()
    assert v.shape == b.shape == (3 ** 9,) and b.dtype == np.uint16 and v.dtype == np.int8
    assert not v.flags.writeable and not b.flags.writeable
    for key in best:
        idx = ts.position(*key)
        assert position(*key) == idx
        assert int(b[idx]) == best[key] and int(v[idx]) == value[key], key
    assert int((b > 0).sum()) == 4520 and int(np.abs(v).sum()) == sum(abs(x) for x in value.values())
    terminal = [ts.position(*k) for k in positions if k not in best]
    assert not b[terminal].any() and not v[terminal].any()
    assert solve() is solve()                                 # computed once per process


def test_solution_facts():
    from jorldy_b200.core.env.tictactoe import position, solve
    v, b = solve()
    assert v[0] == 0 and b[0] == 0x1FF                       # the empty board is a draw, every opening keeps it
    # x: 0, 1; o: 3, 4; x to move: 2 wins (and blocks nothing else needed)
    assert v[position(0b000000011, 0b000011000)] == 1 and b[position(0b000000011, 0b000011000)] == 1 << 2
    # o: 4 to move against x: 0, 1 must block at 2
    idx = position(0b000010000, 0b000000011)
    assert v[idx] == 0 and b[idx] == 1 << 2
    # x: 0, 4 against o: 1, 2, x to move: 8 completes the diagonal at once
    idx = position(0b000010001, 0b000000110)
    assert v[idx] == 1 and (b[idx] >> 8) & 1
    # o: 1, 7 to move against x: 0, 2, 4, which threatens 6 and 8: lost, so every empty cell reaches the value
    idx = position(0b010000010, 0b000010101)
    assert v[idx] == -1 and b[idx] == ot.FULL & ~0b010010111


def test_perfect_opponent_blocks_and_wins(solution):
    _, _, best = solution
    env = ts.PerfectBatch(1, best, auto_reset=False)
    env.boards[0] = (0b000000001, 0b000010000)                # the agent's 1 threatens 2: the only move that holds
    ns, r, d = env.step([1])
    assert r[0] == 0.0 and not d[0] and ns[0][9 + 2] == 1
    env.boards[0] = (0b100000010, 0b000011000)                # the agent's 2 threatens 5, where the opponent wins
    ns, r, d = env.step([2])
    assert r[0] == -1.0 and d[0] and ns[0][9 + 5] == 1


# ------------------------------------------------------------------------------------------- the -gamma identity
def _scripted(seed, A=9, S=60, V=1, R=1):
    g = torch.Generator().manual_seed(seed)
    sims = {"pi": torch.randn(S, A, generator=g).double(), "v": torch.randn(S, 2 * V + 1, generator=g).double(),
            "r": torch.randn(S, 2 * R + 1, generator=g).double(), "s": torch.rand(S, 4, generator=g).double()}
    root_pi = torch.randn(A, generator=g).double().numpy()
    model = lambda sim, lat, a: (sims["s"][sim], sims["pi"][sim], sims["v"][sim], sims["r"][sim])
    return root_pi, model


@pytest.mark.parametrize("gamma", [1.0, 0.997])
def test_two_player_search_is_the_single_player_search_at_minus_gamma(gamma):
    rng = np.random.default_rng(0)
    for seed in range(100):
        root_pi, model = _scripted(seed)
        legal = np.ones(9, dtype=bool) if seed % 2 else rng.random(9) < 0.6
        a, act_a, pi_a, rv_a = ts.search_two_player(root_pi, None, model, 9, 60, gamma, 1, 1, legal)
        b, act_b, pi_b, rv_b = ol.search_legal(root_pi, None, model, 9, 60, -gamma, 1, 1, legal)
        assert np.array_equal(a.n, b.n) and np.array_equal(a.w, -b.w) and np.array_equal(a.child, b.child), seed
        assert (a.qmin, a.qmax, act_a, rv_a) == (b.qmin, b.qmax, act_b, rv_b) and np.array_equal(pi_a, pi_b), seed
        if seed % 2:                                      # an all-legal root is oracle/muzero.py's search
            c, act_c, _, rv_c = om.search(root_pi, None, model, 9, 60, -gamma, 1, 1)
            assert np.array_equal(c.n, b.n) and (act_c, rv_c) == (act_b, rv_b)
    # the single-player backup at +gamma is a different search
    root_pi, model = _scripted(1)
    assert not np.array_equal(ts.search_two_player(root_pi, None, model, 9, 60, gamma, 1, 1, np.ones(9))[0].n,
                              om.search(root_pi, None, model, 9, 60, gamma, 1, 1)[0].n)


@pytest.mark.parametrize("gamma", [1.0, 0.997])
def test_two_player_targets_are_the_targets_at_minus_gamma(gamma):
    rng = np.random.default_rng(1)
    for _ in range(300):
        B, K, n = 3, int(rng.integers(1, 6)), int(rng.integers(1, 10))
        L = K + n + 1
        rew = rng.choice([-1.0, 0.0, 1.0], size=(B, L))
        done = (rng.random((B, L)) < 0.15).astype(np.float64)
        rv = rng.standard_normal((B, L))
        z, u, ab = ts.targets_two_player(rew, done, rv, K, n, gamma)
        z2, u2, ab2 = om.targets(rew, done, rv, K, n, -gamma)
        assert np.array_equal(z, z2) and np.array_equal(u, u2) and np.array_equal(ab, ab2)
    # the alternating sum written out, at gamma 1 with integer values
    rew, done, rv = np.array([[1.0, -1.0, 0.0, 1.0, 0.0]]), np.zeros((1, 5)), np.array([[0, 0, 0, 0, 3.0]])
    assert ts.targets_two_player(rew, done, rv, 1, 3, 1.0)[0][0].tolist() == [1 + 1 + 0 - 0, -1 - 0 + 1 - 3]


# ------------------------------------------------------------------------------------------- exact-model search
# The masked-root search with the true game as its model (uniform priors, exact rewards, value 0 at every leaf, gamma 1)
# over the 4 520 non-terminal positions: the share of positions where it picks an optimal move.  The single-player
# backup at +gamma reads the opponent's wins as its own.
EXACT_RATES = {50: (3901, 3701), 200: (4318, 3667)}    # S: (two-player, single-player) optimal picks of 4 520


@pytest.mark.parametrize("S", sorted(EXACT_RATES))
def test_exact_model_search_plays_better_with_the_two_player_backup(solution, S):
    _, _, best = solution
    two, one = EXACT_RATES[S]
    assert round(ts.optimal_move_rate(best, S, 1.0, True) * len(best)) == two
    assert round(ts.optimal_move_rate(best, S, 1.0, False) * len(best)) == one
    assert two > one + 150
