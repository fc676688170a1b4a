"""Two-player TicTacToe on the GPU: the self-play and perfect-opponent env modes against the numpy oracle
(oracle/tictactoe_selfplay.py) bit for bit, the perfect opponent's table and laws, the unchanged tree and loss kernels at
-gamma against the pseudocode's two-player search and targets in float64, the search with the true game as its model,
one two-player learn, the graph act, the driver's player checks, the other collectors against the perfect opponent, and
end-to-end runs of `jorldy_b200.main` on `config.muzero.tictactoe_selfplay`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import muzero as om
from oracle import muzero_legal as ol
from oracle import tictactoe_selfplay as ts

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
TREE = ("n", "w", "p", "r", "child", "latent", "count", "bounds", "path", "path_len")


def _C():
    from jorldy_b200.core.dev import C
    return C


def ptr(t):
    return 0 if t is None else t.data_ptr()


def _env(N, opponent, seed=0, **kw):
    from jorldy_b200.core import Env
    return Env("tictactoe", num_envs=N, seed=seed, opponent=opponent, **kw)


@pytest.fixture(scope="module")
def best():
    return ts.enumerate_solution()[2]


# ------------------------------------------------------------------------------------------- 1. env modes vs oracle
def _assert_env_equal(env, ref, tag):
    for k, v in (("boards", ref.boards), ("obs", ref.obs), ("legal", ref.legal), ("elapsed", ref.elapsed),
                 ("episode", ref.episode), ("_score", ref.score)):
        assert np.array_equal(getattr(env, k).cpu().numpy(), v), (tag, k)


def _actions(rng, legal, N):
    """Random actions: mostly a legal cell, sometimes an occupied cell or one outside 0..8."""
    a = np.array([rng.choice(np.flatnonzero(l)) if l.any() else 0 for l in legal], dtype=np.int64)
    bad = rng.random(N) < 0.1
    a[bad] = rng.integers(-2, 11, int(bad.sum()))
    return a


@pytest.mark.parametrize("opponent", ["self", "perfect"])
@pytest.mark.parametrize("N", [1, 7, 4096])
@pytest.mark.parametrize("auto_reset", [True, False])
@pytest.mark.parametrize("graph", [False, True])
def test_env_modes_match_the_oracle_bit_for_bit(best, opponent, N, auto_reset, graph):
    env = _env(N, opponent, seed=5, id=1, auto_reset=auto_reset)
    ref = ts.SelfPlayBatch(N, auto_reset=auto_reset) if opponent == "self" else \
        ts.PerfectBatch(N, best, seed=5, id=1, auto_reset=auto_reset)
    assert env.two_player == (opponent == "self") and env.max_steps == (9 if opponent == "self" else 5)
    env.reset_device()
    ref.reset()
    _assert_env_equal(env, ref, "reset")
    rng = np.random.default_rng(N + len(opponent))
    act = torch.zeros(N, dtype=torch.int64, device=DEV)
    g, ref_done = None, np.zeros(N, dtype=bool)
    for t in range(64):
        a = _actions(rng, ref.legal, N)
        if not auto_reset and t % 10 == 9:           # without auto-reset, reset the finished boards by mask
            env.reset_device(torch.as_tensor(ref_done.astype(np.uint8), device=DEV))
            ref.reset(ref_done)
        act.copy_(torch.as_tensor(a))
        if graph:
            if g is None:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    env.step_device(act)
            g.replay()
        else:
            env.step_device(act)
        ns, r, d = ref.step(a)
        ref_done = d > 0
        torch.cuda.synchronize()
        assert np.array_equal(env.next_obs.cpu().numpy(), ns), t
        assert np.array_equal(env.reward.cpu().numpy(), r), t
        assert np.array_equal(env.done.cpu().numpy(), d), t
        _assert_env_equal(env, ref, t)
    assert np.array_equal(env.stats.cpu().numpy(), ref.stats)
    if auto_reset:
        assert ref.stats[0] > 0


def test_entry_points_reject_a_bad_opponent_or_table():
    from jorldy_b200._lib import JbError
    env = _env(4, "perfect")
    C = _C()
    args = (ptr(env.boards), ptr(env.obs), ptr(env.legal), ptr(env.elapsed), ptr(env.episode), ptr(env._score), 0, 0, 0,
            4, 0)
    for opp, table in ((3, 0), (-1, 0), (1, 0), (0, ptr(env.best)), (2, ptr(env.best))):
        with pytest.raises(JbError):
            C.jb_env_tictactoe_reset_opp(opp, table, *args)
        with pytest.raises(JbError):
            C.jb_env_tictactoe_step_opp(opp, table, *args[:6], ptr(env.reward), 0, ptr(env.next_obs), ptr(env.reward),
                                        ptr(env.done), 0, 0, 0, 0, 4, 0)
    with pytest.raises(ValueError):
        _env(4, "minimax")


# ------------------------------------------------------------------------------------------- 2. the perfect opponent
def test_device_table_is_solve():
    from jorldy_b200.core.env.tictactoe import solve
    env = _env(2, "perfect")
    assert env.best.shape == (3 ** 9,)
    assert np.array_equal(env.best.cpu().numpy().astype(np.uint16), solve()[1])
    assert _env(2, "self").best is None and _env(2, "random").best is None


def test_a_random_agent_never_beats_the_perfect_opponent():
    N = 100000
    env = _env(N, "perfect", seed=3, auto_reset=False)
    env.reset_device()
    gen = torch.Generator(DEV).manual_seed(0)
    live = torch.ones(N, dtype=torch.bool, device=DEV)
    outcome = torch.zeros(N, device=DEV)
    for _ in range(env.max_steps):
        a = torch.multinomial(env.legal.float() + (env.legal.sum(1, keepdim=True) == 0), 1, generator=gen).view(-1)
        env.step_device(a)
        outcome = torch.where(live & (env.done > 0), env.reward, outcome)
        live &= env.done == 0
    assert not bool(live.any())
    o = outcome.cpu().numpy()
    assert (o == 1).sum() == 0 and (o == -1).sum() > N // 2 and (o == 0).sum() > 0


def test_perfect_choice_is_uniform_over_the_optimal_cells():
    """10^5 boards: on the boards the opponent did not open, its reply to the agent's centre is one of the four corners
    (an edge loses), uniformly (chi-square); the openings are the random opponent's, bit for bit."""
    from scipy import stats
    N = 100000
    env, rnd = _env(N, "perfect", seed=11), _env(N, "random", seed=11)
    env.reset_device()
    rnd.reset_device()
    assert torch.equal(env.obs, rnd.obs)
    fresh = env.obs[:, 9:].sum(1).cpu().numpy() == 0
    env.step_device(torch.full((N,), 4, dtype=torch.int64, device=DEV))
    reply = env.next_obs[:, 9:].cpu().numpy()[fresh].argmax(1)
    counts = np.bincount(reply, minlength=9)
    assert counts[[1, 3, 4, 5, 7]].sum() == 0
    assert stats.chisquare(counts[[0, 2, 6, 8]]).pvalue > 1e-3


# ------------------------------------------------------------------------------------------- 3. tree kernels at -gamma
def _tree(N, A, S, Hs):
    f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)
    i = lambda *s: torch.zeros(*s, dtype=torch.int32, device=DEV)
    return {"n": i(N, S + 1, A), "w": f(N, S + 1, A), "p": f(N, S + 1, A), "r": f(N, S + 1, A),
            "child": i(N, S + 1, A), "latent": f(N, S + 1, Hs), "count": i(N), "bounds": f(N, 2), "path": i(N, S + 1),
            "path_len": i(N)}


class _Search:
    """The product's tree kernels at `discount` over N trees, driven from the host one simulation at a time."""

    def __init__(self, N, A, S, Hs, V, R, discount, legal=None):
        self.N, self.A, self.S, self.Hs, self.V, self.R, self.g = N, A, S, Hs, V, R, discount
        self.t = _tree(N, A, S, Hs)
        self.tree = [ptr(self.t[k]) for k in TREE]
        self.leaf_n = torch.zeros(N, dtype=torch.int32, device=DEV)
        self.leaf_a = torch.zeros(N, dtype=torch.int32, device=DEV)
        self.dyn = torch.zeros(N, Hs + A, device=DEV)
        self.legal = None if legal is None else torch.as_tensor(np.asarray(legal, dtype=np.uint8), device=DEV)

    def root(self, pi, v, lat0):
        d = [x.to(DEV).contiguous() for x in (pi, v, lat0)]
        args = (*(ptr(x) for x in d), self.N, self.A, self.S, self.Hs, self.V, 0, 0.25, 0.25, 0, 7, 0, *self.tree, 0)
        if self.legal is None:
            _C().jb_mcts_root(*args, 0)
        else:
            _C().jb_mcts_root_legal(*args, ptr(self.legal), 0)

    def select(self):
        args = (self.N, self.A, self.S, self.Hs, self.g, *self.tree, ptr(self.leaf_n), ptr(self.leaf_a), ptr(self.dyn))
        if self.legal is None:
            _C().jb_mcts_select(*args, 0)
        else:
            _C().jb_mcts_select_legal(*args, ptr(self.legal), 0)
        return self.dyn

    def expand(self, s, pi, v, r):
        d = [x.to(DEV).contiguous() for x in (s, pi, v, r)]
        _C().jb_mcts_expand_backup(*(ptr(x) for x in d), self.N, self.A, self.S, self.Hs, self.V, self.R, self.g,
                                   ptr(self.leaf_n), ptr(self.leaf_a), *self.tree, 0)

    def act(self):
        action = torch.zeros(self.N, dtype=torch.int64, device=DEV)
        pi, rv = torch.zeros(self.N, self.A, device=DEV), torch.zeros(self.N, device=DEV)
        _C().jb_mcts_act(self.N, self.A, self.S, self.g, 0, 0, 0, 11, 0, ptr(self.t["n"]), ptr(self.t["w"]),
                         ptr(self.t["r"]), ptr(action), ptr(pi), ptr(rv), 0)
        torch.cuda.synchronize()
        return action, pi, rv


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("N,A,S,gamma", [(1, 2, 1, 1.0), (7, 9, 50, 1.0), (256, 9, 50, 0.997), (64, 18, 24, 1.0)])
def test_tree_kernels_at_minus_gamma_vs_the_two_player_oracle(masked, N, A, S, gamma):
    Hs, V, R = 8, 5, 2
    g = torch.Generator().manual_seed(N * 31 + A * 7 + S)
    root_pi, root_v, lat0 = torch.randn(N, A, generator=g), torch.randn(N, 2 * V + 1, generator=g), torch.rand(N, Hs)
    sims = {"pi": torch.randn(S, N, A, generator=g), "v": torch.randn(S, N, 2 * V + 1, generator=g),
            "r": torch.randn(S, N, 2 * R + 1, generator=g), "s": torch.rand(S, N, Hs, generator=g)}
    legal = (np.random.default_rng(A).random((N, A)) < 0.6).astype(np.uint8) if masked else np.ones((N, A), np.uint8)
    run = _Search(N, A, S, Hs, V, R, -gamma, legal if masked else None)
    run.root(root_pi, root_v, lat0)
    for j in range(S):
        run.select()
        run.expand(sims["s"][j], sims["pi"][j], sims["v"][j], sims["r"][j])
    action, pi, rv = run.act()
    n, w, bounds = (run.t[k].cpu().numpy() for k in ("n", "w", "bounds"))
    for e in range(N):
        model = lambda sim, lat, a, e=e: (sims["s"][sim, e].double(), sims["pi"][sim, e].double(),
                                          sims["v"][sim, e].double(), sims["r"][sim, e].double())
        tr, a, p, v = ts.search_two_player(root_pi[e].double().numpy(), lat0[e], model, A, S, gamma, V, R, legal[e])
        np.testing.assert_array_equal(n[e], tr.n, err_msg=f"env {e}")
        np.testing.assert_allclose(w[e], -tr.w, rtol=1e-5, atol=1e-5)        # the kernels keep the child's side
        np.testing.assert_allclose(bounds[e], [tr.qmin, tr.qmax], rtol=1e-5, atol=1e-5)
        assert int(action[e]) == a
        np.testing.assert_allclose(pi[e].cpu().numpy(), p, atol=1e-6)
        np.testing.assert_allclose(float(rv[e]), v, rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------- 4. exact-model search
def _support(x, W):
    """Logits [len(x), 2W + 1] whose support expectation is h(x) for x in {-1, 0, 1}: the mass h(|x|) on the atom
    sign(x) and the rest on the centre; x = 0 puts all of it on the centre, so the value is exactly 0."""
    h1 = np.sqrt(2.0) - 1.0 + 0.001
    out = np.full((len(x), 2 * W + 1), -1e4, dtype=np.float32)
    out[:, W] = 0.0
    nz = x != 0
    out[nz, W] = np.log(1.0 - h1)
    out[nz, W + np.sign(x[nz]).astype(int)] = np.log(h1)
    return out


def test_exact_model_search_on_the_gpu(best):
    """The 4 520 non-terminal positions, searched by the kernels at -1 with the true game as the model (the latent holds
    the board): the same visit counts and action as the oracle wherever its pUCT margins exceed rounding, and the
    optimal-move rate of the CPU test."""
    keys = sorted(best)
    N, A, S, Hs, W = len(keys), 9, 50, 4, 1
    legal = np.array([[not ((me | op) >> a & 1) for a in range(9)] for me, op in keys], dtype=np.uint8)
    lat0 = torch.tensor([[me, op, 0, 0] for me, op in keys], dtype=torch.float32)
    run = _Search(N, A, S, Hs, W, W, -1.0, legal)
    run.root(torch.zeros(N, A), torch.as_tensor(_support(np.zeros(N), W)), lat0)
    zeros_v = torch.as_tensor(_support(np.zeros(N), W))
    for _ in range(S):
        dyn = run.select().cpu().numpy()
        nxt, rew = np.zeros((N, Hs), dtype=np.float32), np.zeros(N)
        for e in range(N):
            (me, op, term), r = ts.game_step((int(dyn[e, 0]), int(dyn[e, 1]), bool(dyn[e, 2])), int(dyn[e, Hs:].argmax()))
            nxt[e, :3], rew[e] = (me, op, term), r
        run.expand(torch.as_tensor(nxt), torch.zeros(N, A), zeros_v, torch.as_tensor(_support(rew, W)))
    action = run.act()[0].cpu().numpy()
    n = run.t["n"].cpu().numpy()
    hits = sum((best[k] >> int(action[e])) & 1 for e, k in enumerate(keys))
    assert abs(hits - 3901) <= 45, hits            # CPU test: 3 901 of 4 520 with exact rewards, vs 3 701 single-player

    def model(sim, latent, a):
        nxt, r = ts.game_step(latent, a)
        return nxt, np.zeros(A), _support(np.zeros(1), W)[0].astype(np.float64), \
            _support(np.array([r]), W)[0].astype(np.float64)
    qualify, rng = 0, np.random.default_rng(0)
    for e in rng.choice(N, 600, replace=False):
        margins = []
        tr, a, _, _ = ts.search_two_player(np.zeros(A), (*keys[e], False), model, A, S, 1.0, W, W, legal[e],
                                           margins=margins)
        if all(m == 0 or m > 1e-3 for m in margins):
            qualify += 1
            np.testing.assert_array_equal(n[e], tr.n, err_msg=f"position {keys[e]}")
            assert int(action[e]) == a
    assert qualify >= 300, qualify


# ------------------------------------------------------------------------------------------- 5. loss at -gamma
@pytest.mark.parametrize("K,n", [(2, 4), (3, 9), (2, 9), (3, 4)])
@pytest.mark.parametrize("gamma", [1.0, 0.997])
def test_loss_kernel_at_minus_gamma_vs_two_player_targets(K, n, gamma):
    """Rewards in {-1, 0, 1}; row b has its done at position b mod (L + 1) (none when b mod (L + 1) = L)."""
    C, V, R, A = _C(), 1, 1, 9
    L = K + n + 1
    B = 4 * (L + 1)
    rng = np.random.default_rng(K * 10 + n)
    done = np.zeros((B, L), dtype=np.float32)
    for b in range(B):
        if b % (L + 1) < L:
            done[b, b % (L + 1)] = 1
    pol = rng.random((B, L, A)).astype(np.float32)
    bt = dict(reward=rng.choice([-1.0, 0.0, 1.0], size=(B, L)).astype(np.float32), done=done,
              root_value=rng.uniform(-1, 1, (B, L)).astype(np.float32), policy=pol / pol.sum(-1, keepdims=True))
    z2, u2, ab2 = ts.targets_two_player(bt["reward"], bt["done"], bt["root_value"], K, n, gamma)
    z, u, ab = om.targets(bt["reward"], bt["done"], bt["root_value"], K, n, -gamma)
    assert np.array_equal(z, z2) and np.array_equal(u, u2) and np.array_equal(ab, ab2)
    g = torch.Generator().manual_seed(B)
    pi, v, r = torch.randn(K + 1, B, A, generator=g), torch.randn(K + 1, B, 2 * V + 1, generator=g), \
        torch.randn(K, B, 2 * R + 1, generator=g)
    w = np.random.default_rng(B).random(B)
    d = {k: torch.as_tensor(bt[k]).to(DEV).contiguous() for k in ("reward", "done", "root_value", "policy")}
    dpi, dv, dr = (torch.empty(t.shape, device=DEV) for t in (pi, v, r))
    prio, stats = torch.empty(B, dtype=torch.float64, device=DEV), torch.empty(4, device=DEV)
    scratch = torch.empty(3 * B * (K + 1), dtype=torch.float64, device=DEV)
    wd = torch.as_tensor(w, dtype=torch.float64, device=DEV)
    pi_d, v_d, r_d = pi.to(DEV), v.to(DEV), r.to(DEV)
    C.jb_muzero_loss(ptr(pi_d), ptr(v_d), ptr(r_d), ptr(d["reward"]), ptr(d["done"]), ptr(d["root_value"]),
                     ptr(d["policy"]), ptr(wd), B, K, n, A, V, R, -gamma, 0.25, 1.0, ptr(dpi), ptr(dv), ptr(dr),
                     ptr(prio), ptr(stats), ptr(scratch), 0)
    hp = dict(K=K, n=n, V=V, R=R, gamma=-gamma, value_loss_coef=0.25, alpha=1.0, A=A)
    pt, vt, rt = (t.double().requires_grad_(True) for t in (pi, v, r))
    total, st, pr = om.loss(pt, vt, rt, bt, w, hp)
    total.backward()
    torch.cuda.synchronize()
    np.testing.assert_allclose(stats.cpu().numpy(), [st["loss"], st["value_loss"], st["reward_loss"], st["policy_loss"]],
                               rtol=1e-5, atol=1e-6)
    for got, ref in ((dpi, pt.grad), (dv, vt.grad), (dr, rt.grad)):
        np.testing.assert_allclose(got.cpu().numpy(), ref.numpy(), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(prio.cpu().numpy(), pr.numpy(), rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------- 6. the agent
def _agent(**kw):
    from jorldy_b200.core import Agent
    args = dict(state_size=18, action_size=9, hidden_size=32, latent_size=16, num_simulation=12, num_unroll=3,
                td_steps=9, gamma=1.0, value_support=1, reward_support=1, batch_size=16, buffer_size=512,
                start_train_step=0, optim_config={"name": "adam", "lr": 1e-3}, run_step=1000, lr_decay=False,
                device=DEV, seed=3, two_player=True)
    args.update(kw)
    return Agent("muzero", **args)


def test_one_two_player_learn_vs_oracle():
    agent = _agent()
    K, n, A, B = agent.K, agent.n_step, 9, 64
    L = K + n + 1
    rng = np.random.default_rng(0)
    done = np.zeros((B, L), dtype=np.float32)
    done[np.arange(B), np.arange(B) % L] = 1
    pol = rng.random((B, L, A)).astype(np.float32)
    bt = dict(reward=rng.choice([-1.0, 0.0, 1.0], size=(B, L)).astype(np.float32), done=done,
              root_value=rng.uniform(-1, 1, (B, L)).astype(np.float32),
              policy=(pol / pol.sum(-1, keepdims=True)).astype(np.float32), action=rng.integers(0, A, (B, L)),
              state=rng.integers(0, 2, (B, 18)).astype(np.float32))
    agent.memory.store([{k: torch.as_tensor(v).to(DEV) for k, v in bt.items()}])
    u_a, u_b = np.random.default_rng(1).random(agent.batch_size), np.random.default_rng(2).random(agent.batch_size)
    ua, ub = (torch.as_tensor(u, dtype=torch.float64, device=DEV) for u in (u_a, u_b))
    batch, weights, idx, _ = agent.memory.sample_device(agent.beta, agent.batch_size, ua, ub)
    agent.memory._sample_ctr -= 1
    agent._inject_per_u = (u_a, u_b)
    # the float64 oracle: oracle/muzero.py's learn at -gamma, keeping torch's Adam state
    p = {k: v.double().cpu().clone().requires_grad_(True) for k, v in agent.network.state_dict().items()}
    hp = dict(K=K, n=n, V=agent.V, R=agent.R, gamma=-agent.gamma, value_loss_coef=agent.value_loss_coef,
              alpha=agent.alpha, A=A)
    sample = {k: v.cpu().numpy() for k, v in batch.items()}
    z, _, _ = om.targets(sample["reward"], sample["done"], sample["root_value"], K, n, -agent.gamma)
    assert np.array_equal(z, ts.targets_two_player(sample["reward"], sample["done"], sample["root_value"], K, n,
                                                   agent.gamma)[0])
    total, st, prio = om.unroll_loss(p, sample, weights.cpu().numpy(), hp)
    total.backward()
    torch.nn.utils.clip_grad_norm_(list(p.values()), 5.0)
    opt = torch.optim.Adam(list(p.values()), lr=1e-3)
    opt.step()
    res = agent.learn()
    torch.cuda.synchronize()
    for k in ("loss", "value_loss", "reward_loss", "policy_loss"):
        assert abs(res[k] - st[k]) < 1e-4 * max(1.0, abs(st[k])), (k, res[k], st[k])
    state = agent.optimizer.state_dict()["state"]
    for i, (k, v) in enumerate(p.items()):
        np.testing.assert_allclose(agent.network.p[k].double().cpu().numpy(), v.detach().numpy(), rtol=1e-4, atol=2e-5,
                                   err_msg=k)
        for slot in ("exp_avg", "exp_avg_sq"):
            ref = opt.state[v][slot].numpy()
            np.testing.assert_allclose(state[i][slot].double().cpu().numpy().reshape(ref.shape), ref, rtol=1e-3,
                                       atol=1e-4 * float(np.abs(ref).max()) + 1e-12, err_msg=f"{k} {slot}")
    tree = agent.memory._tree.cpu().numpy()
    for i, j in {int(i): j for j, i in enumerate(idx.cpu().numpy())}.items():
        np.testing.assert_allclose(tree[i], prio[j].item(), rtol=1e-4, atol=1e-5)


def test_graph_act_is_bit_identical_to_eager_in_self_play():
    res = []
    for graph in (True, False):
        env = _env(32, "self", seed=8)
        env.reset_device()
        agent = _agent(use_cuda_graph=graph)
        agent.attach_legal(env.legal)
        steps = []
        for _ in range(8):
            a, v = agent.act_device(env.obs, training=True)
            steps.append((a.clone(), v.clone(), agent.step_inputs["policy"].clone(), env.legal.clone()))
            env.step_device(a)
        res.append(steps)
        if graph:
            assert (32, True) in agent._graphs
    for (a1, v1, p1, l1), (a2, v2, p2, l2) in zip(*res):
        assert torch.equal(a1, a2) and torch.equal(v1, v2) and torch.equal(p1, p2) and torch.equal(l1, l2)
        assert bool((l1.gather(1, a1.view(-1, 1)) == 1).all())


def test_two_player_changes_only_the_sign_of_the_discount():
    """The same seeded act with two_player=False and True at gamma 1 differs (the backup reads the sides), and the
    two_player=False agent passes +gamma as before."""
    env = _env(64, "random", seed=2)
    env.reset_device()
    outs = []
    for tp in (False, True):
        agent = _agent(two_player=tp, num_simulation=24, use_cuda_graph=False)
        assert agent._discount == (-1.0 if tp else 1.0)
        agent.attach_legal(env.legal)
        with torch.no_grad():
            agent.network.p["g.r.weight"].mul_(30.0)
        agent.act_device(env.obs, training=False)
        outs.append(agent._search_state(64)["n"].clone())
    assert not torch.equal(outs[0], outs[1])


def test_check_players():
    from jorldy_b200.core import Agent
    from jorldy_b200.run_mode import _check_players
    selfplay, rnd = _env(4, "self"), _env(4, "random")
    dqn = Agent("dqn", state_size=18, action_size=9, hidden_size=32, optim_config={"name": "adam"}, run_step=1000,
                device=DEV)
    with pytest.raises(ValueError):
        _check_players(selfplay, dqn)
    with pytest.raises(ValueError):
        _check_players(selfplay, _agent(two_player=False))
    with pytest.raises(ValueError):
        _check_players(rnd, _agent(two_player=True))
    _check_players(selfplay, _agent(two_player=True))
    _check_players(rnd, _agent(two_player=False))
    _check_players(_env(4, "perfect"), dqn)


# ------------------------------------------------------------------------------------------- 7. other collectors
def _cfg_agent(config_path, env, **override):
    from jorldy_b200 import config as builtin
    from jorldy_b200.core import Agent
    cfg = builtin.load(config_path)
    kw = dict(cfg.agent, state_size=env.state_size, action_size=env.action_size, optim_config=cfg.optim,
              run_step=1000, device=DEV)
    kw.update(override)
    return Agent(**kw)


def test_collectors_against_the_perfect_opponent():
    from jorldy_b200.core.collect import EpisodeCollector, ReplayCollector, RolloutCollector
    env = _env(8, "perfect", seed=1)
    ppo = _cfg_agent("config.ppo.cartpole", env, hidden_size=64, n_step=16, batch_size=32, n_epoch=1)
    res = ppo.learn_rollout(RolloutCollector(env, ppo, use_cuda_graph=False).collect())
    assert res and all(np.isfinite(v) for v in res.values())
    env = _env(8, "perfect", seed=2)
    dqn = _cfg_agent("config.dqn.cartpole", env, hidden_size=64, batch_size=32, buffer_size=1024, start_train_step=0)
    _, res = ReplayCollector(env, dqn, update_period=8).run_round(0)
    assert res and all(np.isfinite(v) for v in res.values())
    env = _env(8, "perfect", seed=3)
    rf = _cfg_agent("config.reinforce.cartpole", env, hidden_size=64)
    res = rf.learn_episodes(EpisodeCollector(env, rf, 16, use_cuda_graph=False).collect())
    assert res and all(np.isfinite(v) for v in res.values())


# ------------------------------------------------------------------------------------------- 8. drivers
@pytest.mark.parametrize("config,mode,extra,final", [
    ("config.muzero.tictactoe_selfplay", "--single", [], 300),
    ("config.muzero.tictactoe_selfplay", "--sync", ["--train.num_workers", "32", "--train.update_period", "4"], 800),
    ("config.muzero.tictactoe", "--sync", ["--env.opponent", "perfect", "--train.num_workers", "32"], 800),
])
def test_training_run_with_save_and_load(tmp_path, config, mode, extra, final):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base = [sys.executable, "-m", "jorldy_b200.main", mode, "--config", config, "--train.run_step", str(final),
            "--train.print_period", str(final // 2), "--train.save_period", str(final), "--agent.start_train_step",
            "200", "--agent.batch_size", "32", "--agent.num_simulation", "8", "--agent.hidden_size", "64",
            "--agent.latent_size", "32", *extra]
    r = subprocess.run(base, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith(f"{final} step |") for line in r.stdout.splitlines()), out[-4000:]
    assert any("policy_loss" in line for line in r.stdout.splitlines() if " step |" in line), out[-4000:]
    ckpts = [d for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    r2 = subprocess.run(base + ["--train.load_path", ckpts[0]], cwd=tmp_path / "logs", env=env, capture_output=True,
                        text=True, timeout=900)
    out2 = r2.stdout + r2.stderr
    assert "Traceback" not in out2 and "Load model from" in out2, out2[-4000:]


def test_driver_refuses_a_self_play_env_for_dqn(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "jorldy_b200.main", "--sync", "--config", "config.dqn.cartpole",
                        "--env.name", "tictactoe", "--env.opponent", "self", "--train.run_step", "10"], cwd=tmp_path,
                       env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "ValueError" in r.stderr and "two_player=True" in r.stderr, r.stderr[-2000:]
