"""REINFORCE on the GPU: the episode kernels and the loss kernel against the float64 oracle, learn() and
learn_episodes() against oracle/reinforce.py, CUDA-graph against eager, the episode collector against a step-by-step
env run, checkpoints, attach, and end-to-end runs of `jorldy_b200.main`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from jorldy_b200._lib import JbError
from oracle import reinforce as orf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _C():
    from jorldy_b200.core.dev import C
    return C


def _agent(**kw):
    from jorldy_b200.core.agent.reinforce import REINFORCE
    args = dict(state_size=4, action_size=2, hidden_size=64, optim_config={"name": "adam", "lr": 1e-3}, lr_decay=False,
                use_standardization=True, device="cuda")
    args.update(kw)
    return REINFORCE(**args)


def _p(t):
    return 0 if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------- 1. episode kernels
def _done_pattern(case, rs, N, pos, elapsed, max_steps):
    if case == "length1":
        d = np.ones(N)
    elif case == "cross_rounds":
        d = np.zeros(N)
    elif case == "several_per_round":
        d = (rs.random_sample(N) < 0.6).astype(np.float64)
    elif case == "none_complete":
        d = (rs.random_sample(N) < 0.3).astype(np.float64)
        d[0] = 0.0
    else:
        d = (rs.random_sample(N) < 0.15).astype(np.float64)
    return np.where(elapsed + 1 >= max_steps, 1.0, d)


@pytest.mark.parametrize("standardize", [1, 0])
@pytest.mark.parametrize("case", ["random", "length1", "cross_rounds", "several_per_round", "none_complete", "wrap"])
@pytest.mark.parametrize("N", [1, 7, 4096])
def test_episode_kernels_match_oracle(N, case, standardize):
    C = _C()
    rs = np.random.RandomState(N + 31 * len(case))
    T, rounds, gamma = 8, 6 if case == "wrap" else 3, 0.97
    max_steps = 6 if case == "wrap" else 20 if case in ("cross_rounds", "none_complete") else 50
    L = max_steps - 1 + T
    Cr = 256
    n_rows = -(-N * L // Cr) * Cr
    reward, done = np.zeros((N, L), np.float32), np.zeros((N, L), np.float32)
    head = np.zeros(N, np.int64)
    elapsed = np.zeros(N, np.int64)
    dev = "cuda"
    g_head = torch.zeros(N, dtype=torch.int64, device=dev)
    g_pos = torch.zeros(1, dtype=torch.int64, device=dev)
    ret_ring = torch.zeros(N, L, device=dev)
    count = torch.zeros(N, dtype=torch.int32, device=dev)
    offsets = torch.zeros(N, dtype=torch.int32, device=dev)
    idx = torch.full((n_rows,), -7, dtype=torch.int32, device=dev)
    ret = torch.full((n_rows,), 9.0, device=dev)
    Mg = torch.zeros(1, dtype=torch.int32, device=dev)
    pos = 0
    for _ in range(rounds):
        for _ in range(T):
            d = _done_pattern(case, rs, N, pos, elapsed, max_steps)
            elapsed = np.where(d != 0, 0, elapsed + 1)
            reward[:, pos % L] = rs.standard_normal(N).astype(np.float32)
            done[:, pos % L] = d
            pos += 1
        g_pos.fill_(pos)
        r_dev, d_dev = torch.as_tensor(reward, device=dev), torch.as_tensor(done, device=dev)
        C.jb_episode_returns(_p(r_dev), _p(d_dev), N, L, _p(g_pos), _p(g_head), gamma, standardize, _p(ret_ring),
                             _p(count), 0)
        C.jb_episode_rows(_p(count), _p(g_head), _p(ret_ring), N, L, Cr, _p(offsets), _p(idx), _p(ret), _p(Mg), 0)
        torch.cuda.synchronize()
        e_idx, e_ret, e_count, e_head = orf.ring_rows(reward, done, pos, head, gamma, bool(standardize))
        M = int(Mg.item())
        assert M == len(e_idx)
        np.testing.assert_array_equal(count.cpu().numpy(), e_count)
        np.testing.assert_array_equal(g_head.cpu().numpy(), e_head)
        np.testing.assert_array_equal(idx[:M].cpu().numpy(), e_idx)
        np.testing.assert_allclose(ret[:M].cpu().numpy(), e_ret, rtol=1.2e-7, atol=1e-9)
        pad = -(-M // Cr) * Cr
        assert (idx[M:pad] == 0).all() and (ret[M:pad] == 0).all()
        head = e_head


def test_episode_rows_rejects_bad_arguments():
    C = _C()
    t = torch.zeros(16, dtype=torch.int64, device="cuda")
    with pytest.raises(JbError):
        C.jb_episode_rows(_p(t), _p(t), _p(t), 4, 4, 0, _p(t), _p(t), _p(t), _p(t), 0)
    with pytest.raises(JbError):
        C.jb_episode_rows(_p(t), _p(t), _p(t), 1 << 16, 1 << 16, 256, _p(t), _p(t), _p(t), _p(t), 0)
    with pytest.raises(JbError):
        C.jb_episode_returns(_p(t), _p(t), 0, 4, _p(t), _p(t), 0.99, 1, _p(t), _p(t), 0)


# ------------------------------------------------------------------------------------------- 2. loss kernel
def _loss_case(rs, Cr, M, k, A, continuous, rows_total):
    """Chunk k of a padded row list of M entries over a ring of rows_total rows."""
    n_pad = -(-M // Cr) * Cr
    idx = np.zeros(n_pad, np.int32)
    idx[:M] = rs.randint(0, rows_total, M)
    ret = np.zeros(n_pad, np.float32)
    ret[:M] = rs.standard_normal(M)
    nout = 2 * A if continuous else A
    out = (rs.standard_normal((Cr, nout)) * 2).astype(np.float32)
    if continuous:
        out[0, 0] = 5.0
        if Cr > 2:
            out[1, 0], out[2, 0] = -5.0, 6.5
        action = np.tanh(rs.standard_normal((rows_total, A))).astype(np.float32)
        action[0, 0] = 1.0
    else:
        action = rs.randint(0, A, rows_total).astype(np.int64)
    return idx, ret, out, action


def _run_loss(idx, ret, out, action, M, Cr, k, A, continuous):
    C = _C()
    dev = "cuda"
    g = lambda x: torch.as_tensor(x, device=dev)
    t_idx, t_ret, t_out, t_act = g(idx), g(ret), g(out), g(action)
    nout = out.shape[1]
    dout = torch.full((Cr, nout), 3.0, device=dev)
    partials = torch.zeros(C.jb_reinforce_loss_partials(Cr), device=dev)
    acc = torch.zeros(2, device=dev)
    cursor = torch.full((1,), k + 1, dtype=torch.int64, device=dev)
    Mg = torch.full((1,), M, dtype=torch.int32, device=dev)
    C.jb_reinforce_loss(int(continuous), _p(t_out), _p(t_idx), _p(t_ret), _p(cursor), _p(Mg), Cr, _p(t_act), A, nout,
                        _p(dout), _p(partials), _p(acc), 0)
    torch.cuda.synchronize()
    return dout.cpu(), acc.cpu()


@pytest.mark.parametrize("continuous, A", [(False, 2), (False, 18), (True, 1), (True, 3), (True, 8)])
@pytest.mark.parametrize("Cr", [1, 255, 256, 257, 8192])
@pytest.mark.parametrize("rel", ["below", "at", "above"])
def test_loss_kernel_matches_float64(continuous, A, Cr, rel):
    rs = np.random.RandomState(Cr + 7 * A)
    M = {"below": max(1, Cr - max(1, Cr // 3)), "at": Cr, "above": 2 * Cr + max(1, Cr // 2)}[rel]
    rows_total = 997
    idx, ret, out, action = _loss_case(rs, Cr, M, 0, A, continuous, rows_total)
    n_chunks = -(-M // Cr)
    total = 0.0
    for k in range(n_chunks):
        sl = slice(k * Cr, (k + 1) * Cr)
        dout, acc = _run_loss(idx, ret, out, action, M, Cr, k, A, continuous)
        dout2, acc2 = _run_loss(idx, ret, out, action, M, Cr, k, A, continuous)
        assert torch.equal(dout, dout2) and torch.equal(acc, acc2)           # bit-reproducible
        valid = min(Cr, M - k * Cr)
        a_rows = torch.as_tensor(action[idx[sl][:valid]])
        o = torch.as_tensor(out[:valid], dtype=torch.float64)
        r = torch.as_tensor(ret[sl][:valid], dtype=torch.float64)
        # the closed form over the chunk's rows with the batch size M of the whole learn
        exp = orf.closed_form(o, a_rows, r, A, continuous) * (valid / M)
        np.testing.assert_allclose(dout[:valid].numpy(), exp.numpy(), rtol=2e-4, atol=2e-6)
        assert (dout[valid:] == 0).all()                                    # padded rows: exactly 0
        chunk_loss = float(orf.loss(o, a_rows, r, A, continuous)) * valid / M
        np.testing.assert_allclose(float(acc[0]), chunk_loss, rtol=2e-4, atol=2e-5)
        assert float(acc[1]) == 1.0
        total += chunk_loss
    a_all = torch.as_tensor(action[idx[:M]])
    o_all = torch.as_tensor(np.concatenate([out] * n_chunks)[:M], dtype=torch.float64)
    np.testing.assert_allclose(total, float(orf.loss(o_all, a_all, torch.as_tensor(ret[:M], dtype=torch.float64), A,
                                                     continuous)), rtol=1e-6, atol=1e-9)


def test_loss_kernel_rejects_bad_arguments_and_ignores_empty_batches():
    C = _C()
    t = torch.zeros(4096, device="cuda")
    M0 = torch.zeros(1, dtype=torch.int32, device="cuda")
    call = lambda cont, Cr, A, nout, M=M0: C.jb_reinforce_loss(cont, _p(t), _p(t), _p(t), 0, _p(M), Cr, _p(t), A, nout,
                                                               _p(t), _p(t), _p(t), 0)
    for cont, Cr, A, nout in ((0, 8, 0, 0), (0, 8, 19, 19), (1, 8, 9, 18), (1, 8, 0, 0), (0, 0, 2, 2), (0, -4, 2, 2),
                              (0, 8, 2, 3), (1, 8, 2, 2)):
        with pytest.raises(JbError):
            call(cont, Cr, A, nout)
    with pytest.raises(JbError):
        call(0, 8, 2, 2, M=None)
    with pytest.raises(JbError):
        C.jb_reinforce_loss_partials(0)
    # a device M <= 0: every row is padding, the accumulator is untouched
    dout = torch.full((8, 2), 5.0, device="cuda")
    acc = torch.tensor([1.5, 2.0], device="cuda")
    out = torch.randn(8, 2, device="cuda")
    idx = torch.zeros(8, dtype=torch.int32, device="cuda")
    act = torch.zeros(8, dtype=torch.int64, device="cuda")
    ret = torch.ones(8, device="cuda")
    part = torch.zeros(1, device="cuda")
    C.jb_reinforce_loss(0, _p(out), _p(idx), _p(ret), 0, _p(M0), 8, _p(act), 2, 2, _p(dout), _p(part), _p(acc), 0)
    torch.cuda.synchronize()
    assert (dout == 0).all() and acc.tolist() == [1.5, 2.0]


# ------------------------------------------------------------------------------------------- 3. learn() (--single)
def _slots(opt, flat):
    return {k: v.detach().cpu() for k, v in zip(opt.network.p.keys(), opt._slot_views(flat))}


def _check_against_oracle(agent, res, ref, lr):
    assert abs(res["loss"] - ref["loss"]) <= 1e-4 * max(1.0, abs(ref["loss"])), (res["loss"], ref["loss"])
    for k, v in ref["params"].items():
        np.testing.assert_allclose(agent.network.p[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=0.05 * lr, err_msg=k)
    m, s = _slots(agent.optimizer, agent.optimizer.exp_avg), _slots(agent.optimizer, agent.optimizer.exp_avg_sq)
    for k in ref["params"]:
        gmax = float(ref["grads"][k].abs().max()) + 1e-12
        np.testing.assert_allclose(m[k].numpy(), ref["exp_avg"][k].numpy(), rtol=1e-3, atol=1e-4 * gmax, err_msg=k)
        np.testing.assert_allclose(s[k].numpy(), ref["exp_avg_sq"][k].numpy(), rtol=2e-3, atol=1e-4 * gmax ** 2, err_msg=k)


@pytest.mark.parametrize("continuous, D, A", [(False, 4, 2), (True, 3, 1), (True, 11, 3)])
def test_learn_single_episode_matches_oracle(continuous, D, A):
    rs = np.random.RandomState(D + A)
    lr = 1e-3
    agent = _agent(state_size=D, action_size=A, network="continuous_policy" if continuous else "discrete_policy",
                   lr_decay=True, run_step=1000)
    params = {k: v.cpu().clone() for k, v in agent.network.state_dict().items()}
    T = 37
    states = rs.standard_normal((T, 1, D)).astype(np.float32)
    actions = (np.tanh(rs.standard_normal((T, 1, A))) if continuous else rs.randint(0, A, (T, 1, 1))).astype(
        np.float32 if continuous else np.int64)
    rewards = rs.standard_normal(T)
    res = {}
    for t in range(T):
        tr = {"state": states[t], "action": actions[t], "reward": np.array([[rewards[t]]]),
              "next_state": states[t], "done": np.array([[t == T - 1]])}
        res = agent.process([tr], t + 1)
        assert (res == {}) == (t < T - 1)
    torch.cuda.synchronize()
    ret = orf.reference_returns(rewards.astype(np.float32), agent.gamma, True)
    a = torch.as_tensor(actions.reshape(T, -1) if continuous else actions.reshape(T))
    ref = orf.learn(params, torch.as_tensor(states.reshape(T, D)), a, torch.as_tensor(ret), A, continuous, lr)
    _check_against_oracle(agent, res, ref, lr)
    assert agent.last_M == T
    # lr_decay ran after the learn (cosine at step T of run_step 1000)
    assert agent.optimizer.param_groups[0]["lr"] == pytest.approx(lr * np.cos(np.pi / 2 * T / 1000))


# ------------------------------------------------------------------------------------------- 4. learn_episodes
def _random_ring(rs, N, L, D, A, continuous, pos, p_done=0.05):
    from jorldy_b200.core.buffer import EpisodeRing
    ring = EpisodeRing(N, L, D, A, "continuous" if continuous else "discrete", device="cuda")
    ring.state.copy_(torch.as_tensor(rs.standard_normal((N, L, D)), dtype=torch.float32))
    if continuous:
        ring.action.copy_(torch.as_tensor(np.tanh(rs.standard_normal((N, L, A))), dtype=torch.float32))
    else:
        ring.action.copy_(torch.as_tensor(rs.randint(0, A, (N, L))))
    ring.reward.copy_(torch.as_tensor(rs.standard_normal((N, L)), dtype=torch.float32))
    ring.done.copy_(torch.as_tensor((rs.random_sample((N, L)) < p_done).astype(np.float32)))
    ring.pos.fill_(pos)
    ring.head.copy_(torch.as_tensor(rs.randint(max(0, pos - L), max(0, pos - L) + 20, N)))
    return ring


@pytest.mark.parametrize("continuous, A", [(False, 3), (True, 2)])
def test_learn_episodes_several_chunks_matches_oracle_graph_and_eager(continuous, A):
    rs = np.random.RandomState(5 + A)
    N, L, D, lr = 64, 400, 5, 1e-3
    pos = 1000
    kw = dict(state_size=D, action_size=A, network="continuous_policy" if continuous else "discrete_policy")
    agents = [_agent(use_cuda_graph=g, **kw) for g in (True, False, True)]
    for a in agents[1:]:
        a.network.load_state_dict(agents[0].network.state_dict())
    params = {k: v.cpu().clone() for k, v in agents[0].network.state_dict().items()}
    rings = [_random_ring(np.random.RandomState(3), N, L, D, A, continuous, pos) for _ in agents]
    head0 = rings[0].head.cpu().numpy().copy()
    results = [a.learn_episodes(r) for a, r in zip(agents, rings)]
    torch.cuda.synchronize()
    M = agents[0].last_M
    Cr = agents[0]._work[next(iter(agents[0]._work))]["C"]
    assert M > 2 * Cr, (M, Cr)                          # several chunks
    for a, r in zip(agents[1:], results[1:]):           # graph == eager == a second graph run, bit for bit
        assert torch.equal(a.network.flat, agents[0].network.flat)
        assert torch.equal(a.optimizer.exp_avg, agents[0].optimizer.exp_avg)
        assert torch.equal(a.optimizer.exp_avg_sq, agents[0].optimizer.exp_avg_sq)
        assert r == results[0]
    ring = rings[0]
    reward, done = ring.reward.cpu().numpy(), ring.done.cpu().numpy()
    e_idx, e_ret, _, e_head = orf.ring_rows(reward, done, pos, head0, agents[0].gamma, True)
    assert len(e_idx) == M
    np.testing.assert_array_equal(ring.head.cpu().numpy(), e_head)
    st = ring.state.view(N * L, D).cpu()[torch.as_tensor(e_idx)]
    act = (ring.action.view(N * L, A) if continuous else ring.action.view(N * L)).cpu()[torch.as_tensor(e_idx)]
    ref = orf.learn(params, st, act, torch.as_tensor(e_ret), A, continuous, lr)
    _check_against_oracle(agents[0], results[0], ref, lr)


# ------------------------------------------------------------------------------------------- 5. EpisodeCollector
def test_episode_collector_matches_step_by_step_env():
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import EpisodeCollector
    N, T, rounds = 16, 150, 3
    agents = [_agent(seed=3) for _ in range(3)]
    for a in agents[1:]:
        a.network.load_state_dict(agents[0].network.state_dict())
    envs = [Env("cartpole", num_envs=N, seed=11) for _ in agents]
    graph = EpisodeCollector(envs[0], agents[0], T, use_cuda_graph=True)
    eager = EpisodeCollector(envs[1], agents[1], T, use_cuda_graph=False)
    L = graph.ring.L
    assert L == 500 - 1 + T
    envs[2].reset_device()
    seen = {"state": [], "action": [], "reward": [], "done": []}
    for _ in range(rounds):
        graph.collect()
        eager.collect()
        for _ in range(T):                              # the same agent and env, one step at a time
            seen["state"].append(envs[2].obs.clone())
            act = agents[2].act_device(envs[2].obs, training=True).clone()
            _, r, d = envs[2].step_device(act)
            seen["action"].append(act)
            seen["reward"].append(r.clone())
            seen["done"].append(d.clone())
    torch.cuda.synchronize()
    for k in ("state", "action", "reward", "done"):
        assert torch.equal(getattr(graph.ring, k), getattr(eager.ring, k)), k
        got = getattr(graph.ring, k)[:, :rounds * T]
        exp = torch.stack(seen[k], dim=1)
        assert torch.equal(got, exp.view(got.shape)), k
    assert int(graph.ring.pos) == rounds * T
    done = torch.stack(seen["done"], dim=1).cpu().numpy()
    assert done.sum() > 0
    ends = np.nonzero(done)
    assert any(0 < t % T < T - 1 for t in ends[1])      # episodes end inside rounds
    firsts = [ends[1][ends[0] == e] for e in range(N)]
    assert any(len(f) > 1 and (f[1:] // T > f[:-1] // T).any() for f in firsts)     # and run across rounds
    # the learn over the collected ring takes exactly the oracle's rows
    res = agents[0].learn_episodes(graph.ring)
    torch.cuda.synchronize()
    e_idx, _, _, e_head = orf.ring_rows(graph.ring.reward.cpu().numpy(), graph.ring.done.cpu().numpy(), rounds * T,
                                        np.zeros(N, np.int64), agents[0].gamma, True)
    assert res and agents[0].last_M == len(e_idx)
    np.testing.assert_array_equal(graph.ring.head.cpu().numpy(), e_head)


def test_round_without_a_completed_episode_changes_nothing():
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import EpisodeCollector
    agent = _agent(lr_decay=True, run_step=1000)
    col = EpisodeCollector(Env("cartpole", num_envs=8, seed=2), agent, 3, use_cuda_graph=True)
    before = [agent.network.flat.clone(), agent.optimizer.exp_avg.clone(), agent.optimizer.exp_avg_sq.clone(),
              agent.optimizer._step_dev.clone()]
    lr = agent.optimizer.param_groups[0]["lr"]
    for _ in range(2):                                  # CartPole's pole cannot fall within 6 steps
        assert agent.learn_episodes(col.collect()) == {}
    torch.cuda.synchronize()
    after = [agent.network.flat, agent.optimizer.exp_avg, agent.optimizer.exp_avg_sq, agent.optimizer._step_dev]
    assert all(torch.equal(x, y) for x, y in zip(before, after))
    assert agent.optimizer.param_groups[0]["lr"] == lr
    assert agent.last_M == 0 and int(col.ring.head.sum()) == 0


# ------------------------------------------------------------------------------------------- 6. checkpoint, attach
def test_checkpoint_round_trip(tmp_path):
    rs = np.random.RandomState(0)
    agent = _agent()
    agent.learn_episodes(_random_ring(rs, 8, 64, 4, 2, False, 100, p_done=0.3))
    agent.save(str(tmp_path))
    ck = torch.load(os.path.join(tmp_path, "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "optimizer"}
    b = _agent()
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, agent.network.flat)
    assert torch.equal(b.optimizer.exp_avg, agent.optimizer.exp_avg)
    assert torch.equal(b.optimizer.exp_avg_sq, agent.optimizer.exp_avg_sq)
    assert int(b.optimizer._step_dev) == int(agent.optimizer._step_dev) == 1


def test_attach_keeps_reinforce_a_replica():
    from jorldy_b200.core import parallel
    agent = _agent()
    with pytest.warns(UserWarning, match="REINFORCE: replicas only \\(no data-parallel learner for REINFORCE\\)"):
        parallel.attach(agent, 2)
    assert agent.world_size == 1


# ------------------------------------------------------------------------------------------- 7. end to end
@pytest.mark.parametrize("mode,config,extra,final", [
    ("--single", "config.reinforce.cartpole", ["--agent.hidden_size", "64"], 2048),
    ("--sync", "config.reinforce.cartpole", ["--train.num_workers", "64", "--agent.hidden_size", "64"], 2048),
    ("--sync", "config.reinforce.mujoco", ["--env.name", "hopper", "--train.num_workers", "16", "--train.update_period",
                                           "512", "--agent.hidden_size", "64"], 4096),
])
def test_training_run_with_save_and_load(tmp_path, mode, config, extra, final):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base = [sys.executable, "-m", "jorldy_b200.main", mode, "--config", config, "--train.run_step", str(final),
            "--train.print_period", str(final // 2), "--train.save_period", str(final), *extra]
    r = subprocess.run(base, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith(f"{final} step |") for line in r.stdout.splitlines()), out[-4000:]
    if config.endswith("cartpole"):
        assert any("loss" in line for line in r.stdout.splitlines() if " step |" in line), out[-4000:]
    ckpts = [d for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    saved = torch.load(os.path.join(ckpts[0], "ckpt"), map_location="cpu", weights_only=False)
    assert set(saved) == {"network", "optimizer"}
    r2 = subprocess.run(base + ["--train.load_path", ckpts[0]], cwd=tmp_path / "logs", env=env, capture_output=True,
                        text=True, timeout=900)
    out2 = r2.stdout + r2.stderr
    assert "Traceback" not in out2 and "Load model from" in out2, out2[-4000:]
