"""TicTacToe and MuZero's masked root without a GPU: the config and the registry, the oracle env's rules on scripted
games, the opponent's cell choice under injected uniforms, the masked oracle search on hand-solved trees, and the support
coverage of `config.muzero.tictactoe`."""
import numpy as np
import pytest
import torch

from oracle import muzero as om
from oracle import muzero_legal as ol
from oracle import tictactoe as ot


def test_config_and_registry():
    from jorldy_b200 import config as cfg
    from jorldy_b200.core.env import env_dict
    assert "tictactoe" in env_dict
    assert "config.muzero.tictactoe" in cfg.available()
    c, base = cfg.load("config.muzero.tictactoe"), cfg.load("config.muzero.cartpole")
    assert c.env == {"name": "tictactoe", "render": False}
    assert c.agent["gamma"] == 1.0 and c.agent["td_steps"] == 5 and c.agent["value_support"] == 1
    assert c.agent["reward_support"] == 1
    changed = {k for k in base.agent if base.agent[k] != c.agent[k]}
    assert changed == {"gamma", "td_steps", "value_support"}
    assert c.optim == base.optim and c.train == base.train
    assert cfg.load("config.muzero.cartpole").agent["gamma"] == 0.997       # the base table is not modified


# ------------------------------------------------------------------------------------------- the oracle env's rules
class _Scripted(ot.TicTacToeBatch):
    """One board whose opening and opponent replies are scripted instead of drawn."""

    def __init__(self, opening=-1):
        super().__init__(1, auto_reset=False)
        self._opening, self.u_next = opening, 0.0

    def _new_games(self, idx):
        for i in idx:
            self.episode[i] += 1
            self.boards[i] = (0, 0 if self._opening < 0 else 1 << self._opening)
            self.elapsed[i], self.score[i] = 0, 0.0

    def _reply_uniforms(self):
        return np.array([self.u_next])


def _play(moves, replies, opening=-1):
    """Plays the agent's moves; the opponent takes the scripted reply cells, through the uniform that picks each one
    as the k-th empty cell.  Returns the per-step (reward, done) and the env."""
    env = _Scripted(opening)
    env.reset()
    replies, out = list(replies), []
    for a in moves:
        me, op = (int(v) for v in env.boards[0])
        empty = ot.FULL & ~(me | op | (1 << a if 0 <= a <= 8 else 0))
        cells = [c for c in range(9) if (empty >> c) & 1]
        if replies and replies[0] in cells:
            env.u_next = (cells.index(replies.pop(0)) + 0.5) / len(cells)
        _, r, d = env.step([a])
        out.append((float(r[0]), bool(d[0])))
        if d[0]:
            break
    return out, env


@pytest.mark.parametrize("line", range(8))
def test_each_line_wins_for_the_agent(line):
    cells = [c for c in range(9) if (ot.LINES[line] >> c) & 1]
    others = [c for c in range(9) if c not in cells]
    # the opponent's replies avoid the line and never complete one of their own in two moves
    out, env = _play(cells, others[:2])
    assert out[-1] == (1.0, True) and all(o == (0.0, False) for o in out[:-1])
    assert env.score[0] == 1.0 and ot.has_line(env.boards[0, 0])


@pytest.mark.parametrize("line", range(8))
def test_each_line_wins_for_the_opponent(line):
    cells = [c for c in range(9) if (ot.LINES[line] >> c) & 1]
    others = [c for c in range(9) if c not in cells]
    # the agent plays off the line without completing one of its own in three moves: pick three non-collinear cells
    for trio in __import__("itertools").combinations(others, 3):
        if not ot.has_line(sum(1 << c for c in trio)):
            break
    out, env = _play(list(trio), cells)
    assert out[-1] == (-1.0, True) and all(o == (0.0, False) for o in out[:-1])
    assert ot.has_line(env.boards[0, 1]) and env.score[0] == -1.0


def test_draw_on_a_full_board():
    #  X O X
    #  X O O      agent X: 0, 2, 3, 7, 8 ; opponent O: 1, 4, 5, 6
    #  O X X
    out, env = _play([0, 2, 3, 7, 8], [1, 4, 5, 6])
    assert [o[0] for o in out] == [0.0] * 5 and out[-1][1] and not any(o[1] for o in out[:-1])
    assert (int(env.boards[0, 0]) | int(env.boards[0, 1])) == ot.FULL and env.score[0] == 0.0


def test_draw_when_the_opponent_fills_the_board():
    #  O X O
    #  O X X      the opponent O opens on 0 and fills the board with its 5th mark (cell 8)
    #  X O O
    me = (1 << 1) | (1 << 4) | (1 << 5) | (1 << 6)
    op = (1 << 0) | (1 << 2) | (1 << 3) | (1 << 7) | (1 << 8)
    assert not ot.has_line(me) and not ot.has_line(op)
    out, env = _play([1, 4, 5, 6], [2, 3, 7, 8], opening=0)
    assert out == [(0.0, False)] * 3 + [(0.0, True)]


def test_forfeit_on_an_occupied_cell_and_out_of_range():
    out, env = _play([4, 4], [0])
    assert out == [(0.0, False), (-1.0, True)]
    assert int(env.boards[0, 0]) == 1 << 4 and int(env.boards[0, 1]) == 1          # the board is unchanged
    out, env = _play([0], [], opening=0)                                            # the opponent's opening cell
    assert out == [(-1.0, True)]
    for bad in (-1, 9, 100):
        out, _ = _play([bad], [])
        assert out == [(-1.0, True)]


def test_opponent_opening():
    assert ot.opening(0.49, 0.0) == 0 and ot.opening(0.49, 0.999) == 8 and ot.opening(0.5, 0.3) == -1
    assert [ot.opening(0.0, (c + 0.5) / 9) for c in range(9)] == list(range(9))
    env = ot.TicTacToeBatch(512, seed=3)
    obs = env.reset()
    opened = obs[:, 9:].sum(1)
    assert set(opened.tolist()) == {0.0, 1.0} and 180 < opened.sum() < 332
    assert obs[:, :9].sum() == 0 and np.array_equal(env.legal, (1 - obs[:, 9:]).astype(np.uint8))
    assert np.all(env.episode == 1)


def test_opponent_cell_under_injected_uniforms():
    empty = 0b101010101                          # cells 0, 2, 4, 6, 8
    assert [ot.opponent_cell(empty, u) for u in (0.0, 0.19, 0.2, 0.5, 0.79, 0.8, 1 - 2 ** -53)] == [0, 0, 2, 4, 6, 8, 8]
    assert ot.opponent_cell(1 << 7, 0.999) == 7
    for n in range(1, 10):
        m = (1 << n) - 1
        assert [ot.opponent_cell(m, (k + 0.5) / n) for k in range(n)] == list(range(n))


def test_oracle_auto_reset_and_stats():
    env = ot.TicTacToeBatch(64, seed=1, auto_reset=True)
    env.reset()
    rng = np.random.default_rng(0)
    finished = 0
    for _ in range(40):
        ns, r, d = env.step(rng.integers(0, 9, 64))
        finished += int(d.sum())
        assert set(np.unique(r)) <= {-1.0, 0.0, 1.0}
        assert np.all(env.elapsed <= 5)
    assert env.stats[0] == finished and finished > 0 and np.all(env.episode >= 1)


# ------------------------------------------------------------------------------------------- the masked search
def _scripted(values, rewards, pis, V=5, R=5):
    def logits(x, W):
        t = om.scalar_to_support(torch.tensor([float(x)]), W)[0]
        return torch.log(t.clamp(min=1e-300))

    def model(sim, latent, a):
        return latent, np.asarray(pis[sim], dtype=np.float64), logits(values[sim], V), logits(rewards[sim], R)
    return model


def test_masked_first_simulation_takes_the_lowest_legal_action():
    """At parent N = 0 every legal score is 0, so the first simulation takes the lowest legal action, not action 0."""
    model = _scripted([1.0], [0.0], [[0, 0, 0]])
    t, a, pi, rv = ol.search_legal(np.log([0.6, 0.3, 0.1]), None, model, 3, 1, 1.0, 5, 5, legal=[0, 1, 1])
    assert t.n[0].tolist() == [0, 1, 0] and a == 1
    np.testing.assert_allclose(t.p[0], [0.0, 0.75, 0.25])
    np.testing.assert_allclose(pi, [0, 1, 0])


def test_masked_search_never_selects_an_illegal_root_edge():
    """A huge prior and a high value on illegal action 0 would win every unmasked selection; masked, it gets no visit,
    while below the root every action, action 0 included, stays allowed."""
    S, A = 12, 3
    model = _scripted([5.0] * S, [0.0] * S, [[10.0, 0.0, 0.0]] * S)
    t, a, pi, rv = ol.search_legal(np.array([10.0, 0.0, 0.0]), None, model, A, S, 1.0, 5, 5, legal=[0, 1, 1])
    assert t.n[0, 0] == 0 and t.n[0].sum() == S and a in (1, 2) and pi[0] == 0.0
    assert (t.n[1:, 0] > 0).any()                     # below the root action 0 is taken
    t2, *_ = om.search(np.array([10.0, 0.0, 0.0]), None, model, A, S, 1.0, 5, 5)
    assert t2.n[0, 0] > 0


def test_single_legal_move_gets_every_visit():
    S = 6
    model = _scripted([0.3] * S, [0.1] * S, [[0.0] * 4] * S)
    t, a, pi, rv = ol.search_legal(np.zeros(4), None, model, 4, S, 1.0, 5, 5, legal=[0, 0, 1, 0],
                                   noise=[1.0, 2.0, 3.0, 4.0], training=True, u=0.3)
    assert t.n[0].tolist() == [0, 0, S, 0] and a == 2
    np.testing.assert_allclose(t.p[0], [0, 0, 1, 0])


@pytest.mark.parametrize("seed", range(4))
def test_all_legal_and_no_legal_masks_match_the_unmasked_search(seed):
    rng = np.random.default_rng(seed)
    A, S = 5, 10
    sims = [(rng.normal(size=A), rng.normal(), rng.normal()) for _ in range(S)]
    model = _scripted([s[1] for s in sims], [s[2] for s in sims], [s[0] for s in sims])
    root = rng.normal(size=A)
    noise = rng.gamma(0.25, size=A) + 1e-3
    ref = om.search(root, None, model, A, S, 0.997, 5, 5, noise=noise, training=True, u=0.4)
    for legal in (np.ones(A), np.zeros(A)):
        got = ol.search_legal(root, None, model, A, S, 0.997, 5, 5, legal=legal, noise=noise, training=True, u=0.4)
        np.testing.assert_array_equal(got[0].n, ref[0].n)
        np.testing.assert_allclose(got[0].p, ref[0].p, rtol=1e-15)
        assert got[1] == ref[1]


def test_masked_root_noise_is_normalised_over_legal_moves():
    prior = ol.root_prior(np.zeros(4), [1, 0, 1, 0], noise=[1.0, 100.0, 3.0, 100.0], frac=0.25)
    np.testing.assert_allclose(prior, [0.75 * 0.5 + 0.25 * 0.25, 0, 0.75 * 0.5 + 0.25 * 0.75, 0])


# ------------------------------------------------------------------------------------------- supports
def test_supports_cover_the_largest_targets():
    """gamma 1 and td_steps 5 (the longest game): every value target is the outcome, |z| <= 1, and |r| <= 1."""
    from jorldy_b200 import config as cfg
    a = cfg.load("config.muzero.tictactoe").agent
    h1 = float(om.value_h(torch.tensor(1.0, dtype=torch.float64)))
    assert abs(h1 - 0.415) < 1e-3
    assert h1 <= a["value_support"] and h1 <= a["reward_support"]
    # an oracle game of at most 5 agent moves: a 5-step target from any position ends in the done
    z, _, _ = om.targets(np.array([[0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0]], dtype=np.float64),
                         np.array([[0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0]], dtype=np.float64),
                         np.full((1, 11), 7.0), 5, a["td_steps"], a["gamma"])
    assert z[0, :5].tolist() == [1.0] * 5
