"""MuZero on the GPU against the float64 oracle (oracle/muzero.py): the scaling and support kernels, the tree kernels
driven by a scripted model, the Dirichlet noise and action draws, the whole search with real networks, the unrolled loss,
one learn, reproducibility, the collector's windows, checkpoints, attach, and end-to-end runs of `jorldy_b200.main`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import muzero as om

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"


def _C():
    from jorldy_b200.core.dev import C
    return C


def ptr(t):
    return 0 if t is None else t.data_ptr()


def _agent(**kw):
    from jorldy_b200.core import Agent
    args = dict(state_size=4, action_size=2, hidden_size=32, latent_size=16, num_simulation=8, num_unroll=3, td_steps=4,
                value_support=5, reward_support=1, batch_size=16, buffer_size=256, start_train_step=0,
                optim_config={"name": "adam", "lr": 1e-3}, run_step=1000, lr_decay=False, device=DEV, seed=3)
    args.update(kw)
    return Agent("muzero", **args)


# ------------------------------------------------------------------------------------------- 1. scaling and supports
@pytest.mark.parametrize("M", [1, 7, 257])
@pytest.mark.parametrize("H", [64, 256])
def test_scale_fwd_bwd_vs_float64(M, H):
    C, g = _C(), torch.Generator().manual_seed(M * H)
    x = torch.randn(M, H, generator=g) * 3
    x[0] = 0.7                                   # a constant row: the range is clamped to 1e-5
    if M > 1:
        x[1] = x[1] * 1e-7                       # a row whose range is below 1e-5 without being constant
    dy = torch.randn(M, H, generator=g)
    xd, dyd = x.to(DEV), dy.to(DEV)
    y, y2, dx = torch.empty_like(xd), torch.zeros(M, H + 5, device=DEV), torch.empty_like(xd)
    C.jb_muzero_scale_fwd(ptr(xd), M, H, ptr(y), ptr(y2), H + 5, 0)
    C.jb_muzero_scale_bwd(ptr(xd), ptr(dyd), M, H, ptr(dx), 0)
    x64 = x.double().requires_grad_(True)
    ref = om.scale(x64)
    (ref * dy.double()).sum().backward()
    torch.cuda.synchronize()
    np.testing.assert_allclose(y.cpu().numpy(), ref.detach().numpy(), atol=2e-6)
    assert torch.equal(y2[:, :H], y)
    # per row: the clamped constant row's gradients are ~1e5 times the others'
    g_ref, g = x64.grad.numpy(), dx.cpu().numpy()
    for i in range(M):
        np.testing.assert_allclose(g[i], g_ref[i], rtol=1e-4, atol=1e-5 * float(np.abs(g_ref[i]).max()), err_msg=f"row {i}")
    assert np.abs(g_ref[0]).max() > 1e3


@pytest.mark.parametrize("V", [1, 20, 300])
@pytest.mark.parametrize("M", [1, 7, 257])
def test_support_kernels_vs_float64(V, M):
    C, g = _C(), torch.Generator().manual_seed(V + M)
    logits = torch.randn(M, 2 * V + 1, generator=g) * 2
    x = torch.randn(M, generator=g) * float(om.value_h_inv(torch.tensor(float(V), dtype=torch.float64))) * 0.7
    x[0] = 1e7                                   # beyond the support: clamped to the last atom
    if M > 1:
        x[1] = -1e7
    out, sup = torch.empty(M, device=DEV), torch.empty(M, 2 * V + 1, device=DEV)
    logits_d, x_d = logits.to(DEV), x.to(DEV)
    C.jb_muzero_support_to_scalar(ptr(logits_d), M, V, ptr(out), 0)
    C.jb_muzero_scalar_to_support(ptr(x_d), M, V, ptr(sup), 0)
    torch.cuda.synchronize()
    ref = om.support_to_scalar(logits.double(), V).numpy()
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(sup.cpu().numpy(), om.scalar_to_support(x.double(), V).numpy(), atol=1e-6)


# ------------------------------------------------------------------------------------------- 2-4. tree kernels
def _tree(N, A, S, Hs):
    f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)
    i = lambda *s: torch.zeros(*s, dtype=torch.int32, device=DEV)
    return {"n": i(N, S + 1, A), "w": f(N, S + 1, A), "p": f(N, S + 1, A), "r": f(N, S + 1, A),
            "child": i(N, S + 1, A), "latent": f(N, S + 1, Hs), "count": i(N), "bounds": f(N, 2), "path": i(N, S + 1),
            "path_len": i(N)}


def _scripted_search(N, A, S, gamma, seed, ties=False, training=False, gamma_in=None, u_in=None, temperature=1.0):
    """Runs the tree kernels with a scripted model (random logits per simulation) on the GPU and the oracle search per
    env with the same arrays; returns both."""
    C, Hs, V, R = _C(), 8, 5, 2
    g = torch.Generator().manual_seed(seed)
    scale = 0.0 if ties else 1.0
    root_pi = torch.randn(N, A, generator=g) * scale
    root_v = torch.randn(N, 2 * V + 1, generator=g)
    sims = {"pi": torch.randn(S, N, A, generator=g) * scale, "v": torch.randn(S, N, 2 * V + 1, generator=g),
            "r": torch.randn(S, N, 2 * R + 1, generator=g), "s": torch.rand(S, N, Hs, generator=g)}
    if ties:
        # all the mass on the centre atom: every value and reward is exactly 0 in any precision, so every pUCT
        # comparison between equal priors is an exact tie (a softmax expectation near 0 is not exact, and the min-max
        # normalisation would magnify its rounding)
        for k, W in (("v", V), ("r", R)):
            sims[k].fill_(-1e4)
            sims[k][..., W] = 0.0
    t = _tree(N, A, S, Hs)
    tree = [ptr(t[k]) for k in ("n", "w", "p", "r", "child", "latent", "count", "bounds", "path", "path_len")]
    dev = {k: v.to(DEV).contiguous() for k, v in sims.items()}
    leaf_n, leaf_a = torch.zeros(N, dtype=torch.int32, device=DEV), torch.zeros(N, dtype=torch.int32, device=DEV)
    dyn = torch.zeros(N, Hs + A, device=DEV)
    lat0 = torch.rand(N, Hs, generator=g).to(DEV)
    gin = None if gamma_in is None else torch.as_tensor(gamma_in, dtype=torch.float64, device=DEV)
    uin = None if u_in is None else torch.as_tensor(u_in, dtype=torch.float64, device=DEV)
    temp = torch.tensor([temperature], device=DEV)
    root_pi_d, root_v_d = root_pi.to(DEV), root_v.to(DEV)
    C.jb_mcts_root(ptr(root_pi_d), ptr(root_v_d), ptr(lat0), N, A, S, Hs, V, int(training), 0.25, 0.25, ptr(gin), 7, 0,
                   *tree, 0, 0)
    paths = []
    for j in range(S):
        C.jb_mcts_select(N, A, S, Hs, gamma, *tree, ptr(leaf_n), ptr(leaf_a), ptr(dyn), 0)
        paths.append((t["path"].clone(), t["path_len"].clone()))
        C.jb_mcts_expand_backup(ptr(dev["s"][j]), ptr(dev["pi"][j]), ptr(dev["v"][j]), ptr(dev["r"][j]), N, A, S, Hs, V,
                                R, gamma, ptr(leaf_n), ptr(leaf_a), *tree, 0)
    action = torch.zeros(N, dtype=torch.int64, device=DEV)
    pi, rv = torch.zeros(N, A, device=DEV), torch.zeros(N, device=DEV)
    C.jb_mcts_act(N, A, S, gamma, int(training), ptr(temp), ptr(uin), 11, 0, ptr(t["n"]), ptr(t["w"]), ptr(t["r"]),
                  ptr(action), ptr(pi), ptr(rv), 0)
    torch.cuda.synchronize()
    refs = []
    for e in range(N):
        model = lambda sim, lat, a, e=e: (sims["s"][sim, e].double(), sims["pi"][sim, e].double(),
                                          sims["v"][sim, e].double(), sims["r"][sim, e].double())
        refs.append(om.search(root_pi[e].double().numpy(), lat0[e].cpu(), model, A, S, gamma, V, R,
                              noise=None if gamma_in is None else np.asarray(gamma_in)[e], training=training,
                              temperature=temperature, u=None if u_in is None else float(np.asarray(u_in)[e])))
    return t, paths, action, pi, rv, refs


@pytest.mark.parametrize("N,A,S,gamma", [(1, 2, 1, 1.0), (7, 3, 2, 0.997), (256, 18, 50, 0.997), (7, 2, 50, 1.0),
                                         (256, 3, 50, 1.0)])
@pytest.mark.parametrize("ties", [False, True])
def test_tree_kernels_vs_oracle(N, A, S, gamma, ties):
    t, paths, action, pi, rv, refs = _scripted_search(N, A, S, gamma, seed=N * 31 + A * 7 + S, ties=ties)
    n, w, bounds = t["n"].cpu().numpy(), t["w"].cpu().numpy(), t["bounds"].cpu().numpy()
    for e, (tr, a, p, v) in enumerate(refs):
        np.testing.assert_array_equal(n[e], tr.n, err_msg=f"env {e}")
        np.testing.assert_allclose(w[e], tr.w, rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(bounds[e], [tr.qmin, tr.qmax], rtol=1e-5, atol=1e-5)
        assert int(action[e]) == a
        np.testing.assert_allclose(pi[e].cpu().numpy(), p, atol=1e-6)
        np.testing.assert_allclose(float(rv[e]), v, rtol=1e-5, atol=1e-5)
    # the last walk of every env equals the oracle's
    last, ln = paths[-1]
    for e, (tr, *_rest) in enumerate(refs):
        assert [(int(x) // A, int(x) % A) for x in last[e, :int(ln[e])].cpu()] == tr.path


def test_dirichlet_injected_gamma_draws_and_sampled_actions_vs_oracle():
    N, A, S = 64, 5, 16
    rng = np.random.default_rng(0)
    gam = rng.gamma(0.25, size=(N, A)) + 1e-3
    u = rng.random(N)
    t, _, action, pi, rv, refs = _scripted_search(N, A, S, 0.997, seed=5, training=True, gamma_in=gam, u_in=u,
                                                  temperature=0.5)
    for e, (tr, a, p, v) in enumerate(refs):
        np.testing.assert_allclose(t["p"][e, 0].cpu().numpy(), tr.p[0], rtol=1e-5, atol=1e-7)
        np.testing.assert_array_equal(t["n"][e].cpu().numpy(), tr.n)
        assert int(action[e]) == a


def test_dirichlet_philox_law_and_fresh_draws():
    """Mean alpha / (A alpha) and variance of each Dirichlet component; one marginal (Beta(alpha, (A - 1) alpha)) by a
    KS test at 10^5 rows; a second launch with the advanced counters draws new numbers."""
    from scipy import stats
    C, N, A, S, Hs, V = _C(), 100000, 4, 1, 4, 1
    t = _tree(N, A, S, Hs)
    tree = [ptr(t[k]) for k in ("n", "w", "p", "r", "child", "latent", "count", "bounds", "path", "path_len")]
    big = torch.zeros(N, A, device=DEV)                 # frac = 1: the priors are the noise alone
    zeros = torch.zeros(N, 2 * V + 1, device=DEV)
    ctr, lat = torch.zeros(N, dtype=torch.int64, device=DEV), torch.zeros(N, Hs, device=DEV)
    C.jb_mcts_root(ptr(big), ptr(zeros), ptr(lat), N, A, S, Hs, V, 1, 0.25, 1.0, 0, 9, ptr(ctr), *tree, 0, 0)
    p1 = t["p"][:, 0].double().cpu().numpy()
    C.jb_mcts_root(ptr(big), ptr(zeros), ptr(lat), N, A, S, Hs, V, 1, 0.25, 1.0, 0, 9, ptr(ctr), *tree, 0, 0)
    p2 = t["p"][:, 0].double().cpu().numpy()
    a = 0.25
    np.testing.assert_allclose(p1.mean(0), 1.0 / A, atol=5e-3)
    var = (a * (A - 1) * a) / ((A * a) ** 2 * (A * a + 1))
    np.testing.assert_allclose(p1.var(0), var, rtol=0.05)
    assert stats.kstest(p1[:, 0], stats.beta(a, (A - 1) * a).cdf).pvalue > 1e-3
    assert not np.array_equal(p1, p2) and int(ctr[0]) == 2


def test_greedy_and_sampled_action_law():
    """Greedy takes argmax N (lowest on ties); sampling follows N^(1/T): chi-square at 10^5 rows."""
    from scipy import stats
    C, N, A, S = _C(), 100000, 4, 8
    counts = torch.tensor([3, 0, 1, 4], dtype=torch.int32)
    n = torch.zeros(N, S + 1, A, dtype=torch.int32)
    n[:, 0] = counts
    n[0, 0] = torch.tensor([2, 2, 1, 0])
    n, w, r = n.to(DEV), torch.zeros(N, S + 1, A, device=DEV), torch.zeros(N, S + 1, A, device=DEV)
    act, pi, rv = torch.zeros(N, dtype=torch.int64, device=DEV), torch.zeros(N, A, device=DEV), torch.zeros(N, device=DEV)
    temp = torch.tensor([0.5], device=DEV)
    C.jb_mcts_act(N, A, S, 1.0, 0, ptr(temp), 0, 1, 0, ptr(n), ptr(w), ptr(r), ptr(act), ptr(pi), ptr(rv), 0)
    torch.cuda.synchronize()
    assert int(act[0]) == 0 and int(act[1]) == 3
    ctr = torch.zeros(N, dtype=torch.int64, device=DEV)
    C.jb_mcts_act(N, A, S, 1.0, 1, ptr(temp), 0, 1, ptr(ctr), ptr(n), ptr(w), ptr(r), ptr(act), ptr(pi), ptr(rv), 0)
    obs = np.bincount(act[1:].cpu().numpy(), minlength=A)
    p = counts.double().numpy() ** 2
    p /= p.sum()
    keep = p > 0
    assert obs[~keep].sum() == 0
    assert stats.chisquare(obs[keep], p[keep] * obs.sum()).pvalue > 1e-3


# ------------------------------------------------------------------------------------------- 5. whole search, real nets
def test_search_with_networks_vs_oracle():
    N = 64
    agent = _agent(num_simulation=12, action_size=3, use_cuda_graph=False)
    with torch.no_grad():                   # spread the priors and values: the policy head starts near uniform
        agent.network.p["f.pi.weight"].mul_(300.0)
        agent.network.p["f.v.weight"].mul_(30.0)
        agent.network.p["g.r.weight"].mul_(30.0)
    x = torch.randn(N, 4, generator=torch.Generator().manual_seed(1))
    action, _ = agent.act_device(x.to(DEV), training=False)
    n = agent._search_state(N)["n"].cpu().numpy()
    p = {k: v.double().cpu() for k, v in agent.network.state_dict().items()}
    model = om.network_model(p, 3)
    s0 = om.represent(p, x.double())
    pi0, _ = om.predict(p, s0)
    qualify = 0
    for e in range(N):
        margins = []
        tr, a, _, _ = om.search(pi0[e].numpy(), s0[e], model, 3, 12, agent.gamma, agent.V, agent.R, margins=margins)
        if min(margins) > 1e-3:
            qualify += 1
            np.testing.assert_array_equal(n[e], tr.n, err_msg=f"env {e}")
            assert int(action[e]) == a
    assert qualify >= 0.9 * N, qualify


# ------------------------------------------------------------------------------------------- 6. loss
def _windows(B, K, n, A, seed, done_at=None):
    rng = np.random.default_rng(seed)
    L = K + n + 1
    done = np.zeros((B, L), dtype=np.float32)
    if done_at == "first":
        done[:, 0] = 1
    elif done_at == "mid":
        done[::2, K // 2 + 1] = 1
    pol = rng.random((B, L, A)).astype(np.float32)
    return dict(reward=rng.normal(size=(B, L)).astype(np.float32), done=done,
                root_value=(rng.normal(size=(B, L)) * 5).astype(np.float32),
                policy=(pol / pol.sum(-1, keepdims=True)).astype(np.float32),
                action=rng.integers(0, A, (B, L)), state=rng.normal(size=(B, 4)).astype(np.float32))


@pytest.mark.parametrize("K,n", [(1, 1), (5, 10)])
@pytest.mark.parametrize("A", [2, 18])
@pytest.mark.parametrize("B", [1, 32, 257])
@pytest.mark.parametrize("done_at", [None, "first", "mid"])
@pytest.mark.parametrize("wkind", ["null", "ones", "random"])
def test_loss_kernel_vs_oracle(K, n, A, B, done_at, wkind):
    C, V, R = _C(), 20, 1
    bt = _windows(B, K, n, A, seed=K + n + A + B, done_at=done_at)
    g = torch.Generator().manual_seed(B)
    pi = torch.randn(K + 1, B, A, generator=g)
    v = torch.randn(K + 1, B, 2 * V + 1, generator=g)
    r = torch.randn(K, B, 2 * R + 1, generator=g)
    w = {"null": None, "ones": np.ones(B), "random": np.random.default_rng(B).random(B)}[wkind]
    d = {k: torch.as_tensor(bt[k]).to(DEV).contiguous() for k in ("reward", "done", "root_value", "policy")}
    dpi, dv, dr = (torch.empty(t.shape, device=DEV) for t in (pi, v, r))
    prio, stats = torch.empty(B, dtype=torch.float64, device=DEV), torch.empty(4, device=DEV)
    scratch = torch.empty(3 * B * (K + 1), dtype=torch.float64, device=DEV)
    wd = None if w is None else torch.as_tensor(w, dtype=torch.float64, device=DEV)
    pi_d, v_d, r_d = pi.to(DEV), v.to(DEV), r.to(DEV)
    C.jb_muzero_loss(ptr(pi_d), ptr(v_d), ptr(r_d), ptr(d["reward"]), ptr(d["done"]),
                     ptr(d["root_value"]), ptr(d["policy"]), ptr(wd), B, K, n, A, V, R, 0.997, 0.25, 1.0, ptr(dpi), ptr(dv),
                     ptr(dr), ptr(prio), ptr(stats), ptr(scratch), 0)
    hp = dict(K=K, n=n, V=V, R=R, gamma=0.997, value_loss_coef=0.25, alpha=1.0, A=A)
    pt, vt, rt = (t.double().requires_grad_(True) for t in (pi, v, r))
    total, st, pr = om.loss(pt, vt, rt, bt, w, hp)
    total.backward()
    torch.cuda.synchronize()
    np.testing.assert_allclose(stats.cpu().numpy(), [st["loss"], st["value_loss"], st["reward_loss"], st["policy_loss"]],
                               rtol=1e-5, atol=1e-6)
    for got, ref in ((dpi, pt.grad), (dv, vt.grad), (dr, rt.grad)):
        np.testing.assert_allclose(got.cpu().numpy(), ref.numpy(), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(prio.cpu().numpy(), pr.numpy(), rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------- 7-8. unroll and one learn
def _filled(agent, N=64, seed=0):
    bt = _windows(N, agent.K, agent.n_step, agent.action_size, seed, done_at="mid")
    agent.memory.store([{k: torch.as_tensor(v).to(DEV) for k, v in bt.items()}])
    return bt


def _oracle_learn(agent, lr=1e-3, clip=5.0):
    u_a = np.random.default_rng(1).random(agent.batch_size)
    u_b = np.random.default_rng(2).random(agent.batch_size)
    ua, ub = (torch.as_tensor(u, dtype=torch.float64, device=DEV) for u in (u_a, u_b))
    batch, weights, idx, _ = agent.memory.sample_device(agent.beta, agent.batch_size, ua, ub)
    agent.memory._sample_ctr -= 1
    agent._inject_per_u = (u_a, u_b)
    params = {k: v.double().cpu() for k, v in agent.network.state_dict().items()}
    hp = dict(K=agent.K, n=agent.n_step, V=agent.V, R=agent.R, gamma=agent.gamma, value_loss_coef=agent.value_loss_coef,
              alpha=agent.alpha, A=agent.action_size)
    bt = {k: v.cpu().numpy() for k, v in batch.items()}
    return om.learn(params, bt, weights.cpu().numpy(), hp, lr, clip), idx


def test_one_learn_vs_oracle():
    agent = _agent()
    _filled(agent)
    (new, st, prio, grads), idx = _oracle_learn(agent)
    res = agent.learn()
    torch.cuda.synchronize()
    assert set(res) == {"loss", "value_loss", "reward_loss", "policy_loss", "sampled_p", "mean_p", "num_learn"}
    for k in ("loss", "value_loss", "reward_loss", "policy_loss"):
        assert abs(res[k] - st[k]) < 1e-4 * max(1.0, abs(st[k])), (k, res[k], st[k])
    for k, g in grads.items():
        np.testing.assert_allclose(agent.network.g[k].double().cpu().numpy(), g.numpy(), rtol=1e-3,
                                   atol=1e-4 * float(g.abs().max()) + 1e-7, err_msg=k)
    for k, v in new.items():
        np.testing.assert_allclose(agent.network.p[k].double().cpu().numpy(), v.numpy(), rtol=1e-4, atol=2e-5, err_msg=k)
    tree = agent.memory._tree.cpu().numpy()
    last = {int(i): j for j, i in enumerate(idx.cpu().numpy())}
    for i, j in last.items():
        np.testing.assert_allclose(tree[i], prio[j].item(), rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------- 9. reproducibility
def test_learns_and_graph_act_are_bit_identical():
    outs = []
    for _ in range(2):
        agent = _agent()
        _filled(agent)
        agent._inject_per_u = (np.linspace(0.01, 0.99, 16), np.linspace(0.02, 0.98, 16))
        agent.learn()
        agent.learn()
        outs.append(agent.network.flat.clone())
    assert torch.equal(outs[0], outs[1])
    x = torch.randn(32, 4, generator=torch.Generator().manual_seed(4)).to(DEV)
    res = []
    for graph in (True, False):
        agent = _agent(use_cuda_graph=graph)
        steps = []
        for _ in range(3):
            a, v = agent.act_device(x, training=True)
            steps.append((a.clone(), v.clone(), agent.step_inputs["policy"].clone()))
        res.append(steps)
    for (a1, v1, p1), (a2, v2, p2) in zip(*res):
        assert torch.equal(a1, a2) and torch.equal(v1, v2) and torch.equal(p1, p2)


# ------------------------------------------------------------------------------------------- 10. collector windows
def test_collector_windows_match_a_step_record():
    """Every stored window equals the step-by-step record of what act returned and what env.step_device produced, and
    some of the checked windows run across an episode end."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    N, T = 16, 40
    env = Env("cartpole", num_envs=N, seed=0)
    agent = _agent(num_simulation=4, start_train_step=10 ** 9, buffer_size=1024, use_cuda_graph=False)
    col = ReplayCollector(env, agent, update_period=1)
    step_device, rec = env.step_device, []

    def recorded_step(action):
        out = step_device(action)
        rec[-1].update(reward=out[1].view(-1).clone(), done=out[2].view(-1).clone())
        return out
    env.step_device = recorded_step
    for _ in range(T):
        rec.append({"state": env.obs.clone()})
        col.run_round(0)
        rec[-1].update(action=agent._search_state(N)["action"].clone(),
                       root_value=agent.step_inputs["root_value"].clone(), policy=agent.step_inputs["policy"].clone())
    L = agent.L
    assert agent.memory.size == (T - L + 1) * N
    spans_episode_end = False
    for t0 in range(T - L + 1):
        w = agent.memory.gather_device(torch.arange(t0 * N, (t0 + 1) * N, device=DEV))
        assert torch.equal(w["state"], rec[t0]["state"]), t0
        for i in range(L):
            for k in ("action", "reward", "done", "root_value", "policy"):
                assert torch.equal(w[k][:, i], rec[t0 + i][k]), (t0, i, k)
        spans_episode_end |= bool((w["done"][:, :L - 1] != 0).any())
    assert spans_episode_end


def test_graph_replays_draw_fresh_root_noise():
    """Two replays of the training act graph on the same observations mix different Dirichlet noise into the root
    priors: the kernels advance the row counters on the device."""
    agent = _agent(use_cuda_graph=True)
    x = torch.randn(64, 4, generator=torch.Generator().manual_seed(2)).to(DEV)
    priors = []
    for _ in range(3):
        agent.act_device(x, training=True)
        priors.append(agent._search_state(64)["p"][:, 0].clone())
    assert (64, True) in agent._graphs
    assert not torch.equal(priors[0], priors[1]) and not torch.equal(priors[1], priors[2])
    assert int(agent._row_counter(64)[0]) == 2 * 3      # root noise and action draw, once per act


# ------------------------------------------------------------------------------------------- 11. checkpoint, attach
def test_checkpoint_round_trip(tmp_path):
    agent = _agent()
    _filled(agent)
    agent.learn()
    agent.save(str(tmp_path))
    ck = torch.load(os.path.join(tmp_path, "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "optimizer"} and list(ck["network"]) == list(agent.network.p)
    b = _agent(seed=9)
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, agent.network.flat)
    assert torch.equal(b.optimizer.exp_avg, agent.optimizer.exp_avg)


def test_attach_keeps_muzero_a_replica():
    from jorldy_b200.core import parallel
    agent = _agent()
    with pytest.warns(UserWarning, match="MuZero: replicas only \\(no data-parallel learner for MuZero\\)"):
        parallel.attach(agent, 2)
    assert agent.world_size == 1 and agent.allreduce is None


# ------------------------------------------------------------------------------------------- 12. end to end
@pytest.mark.parametrize("mode,extra,final", [
    ("--single", [], 400),
    ("--sync", ["--train.num_workers", "32", "--train.update_period", "4"], 800),
])
def test_training_run_with_save_and_load(tmp_path, mode, extra, final):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base = [sys.executable, "-m", "jorldy_b200.main", mode, "--config", "config.muzero.cartpole", "--train.run_step",
            str(final), "--train.print_period", str(final // 2), "--train.save_period", str(final),
            "--agent.start_train_step", "200", "--agent.batch_size", "32", "--agent.num_simulation", "8",
            "--agent.hidden_size", "64", "--agent.latent_size", "32", *extra]
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
