"""MPO on the GPU (pytest -m gpu): every csrc/mpo.cu kernel against the float64 oracle (oracle/mpo.py), the collected
windows against the env's own step records, eager learns against the oracle's at CartPole and Hopper dimensions, the
CUDA-graph path against eager, determinism, checkpoints, parallel.attach and end-to-end runs of main --sync.

Tolerances (fp32 kernels against float64):
  logp, sample z / tanh(z)      : rtol 1e-5, atol 1e-5 (a few transcendental round-offs per element)
  Qret, dq, critic stats        : rtol 1e-4, atol 1e-5 * (1 + max|Qret|) (n <= 32 fp32 recursion steps)
  dout                          : atol 2e-6 + 1e-4 * max|dout|
  dmult, policy stats           : rtol 1e-4, atol 1e-5 (d eta at eta = min_eta: atol 1e-3, Q'/eta ~ 1e8)
  parameters after a learn      : atol 0.1 * lr (Adam normalises the update to ~lr)
  Adam moments                  : atol 1e-3 * max|moment| + 1e-9, rtol 5e-3
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mpo as om

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
EPS = (0.01, 0.01, 5e-5)
MINS = (1e-8, 1e-8, 1e-8)


def _C():
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    return C, ptr, stream_ptr


_LIVE = []          # device copies handed to a kernel by pointer stay referenced until the test ends


@pytest.fixture(autouse=True)
def _release_inputs():
    yield
    _LIVE.clear()


def _g(x, dtype=torch.float32):
    t = torch.as_tensor(np.asarray(x)).to(dtype).to(DEV).contiguous()
    _LIVE.append(t)
    return t


def _d(x):
    return torch.as_tensor(x).detach().cpu().to(torch.float64)


# ------------------------------------------------------------------------------------------------------ 1. kernels
@pytest.mark.parametrize("cont,A", [(False, 2), (False, 18), (True, 3), (True, 8)])
def test_logp_kernel(cont, A):
    C, ptr, sp = _C()
    rs = np.random.RandomState(A)
    M = 300
    nout = 2 * A if cont else A + 1                     # a wider row stride than the head, as with a value column
    out = rs.standard_normal((M, nout)).astype(np.float32)
    act = np.tanh(rs.standard_normal((M, A))).astype(np.float32) if cont else rs.randint(0, A, M)
    ga = _g(act) if cont else _g(act, torch.int64)
    lp = torch.empty(M, device=DEV)
    C.jb_mpo_logp(int(cont), ptr(_g(out)), nout, ptr(ga), M, A, ptr(lp), sp())
    ref = om.logp(torch.tensor(out, dtype=torch.float64)[:, :2 * A if cont else A], torch.tensor(act), A, cont)
    np.testing.assert_allclose(lp.cpu().numpy(), ref.numpy(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("A", [3, 8])
def test_sample_kernel(A):
    C, ptr, sp = _C()
    rs = np.random.RandomState(A)
    B, n, K, D = 5, 8, 30, 11
    R = B * (n + 1)
    raw = rs.standard_normal((R, 2 * A)).astype(np.float32)
    raw[::7, 0] = 7.0
    eps = rs.standard_normal((R, K, A)).astype(np.float32)
    x = rs.standard_normal((R, D)).astype(np.float32)
    taken = np.tanh(rs.standard_normal((B * n, A))).astype(np.float32)
    z, xs, xa = (torch.empty(s, device=DEV) for s in ((R, K, A), (R * (K + 1), D), (R * (K + 1), A)))
    C.jb_mpo_sample(ptr(_g(raw)), ptr(_g(eps)), R, K, A, ptr(_g(x)), D, ptr(_g(taken)), n, ptr(z), ptr(xs), ptr(xa), sp())
    zr, ar = om.sample(torch.tensor(raw, dtype=torch.float64), torch.tensor(eps, dtype=torch.float64), A)
    np.testing.assert_allclose(z.cpu().numpy(), zr.numpy(), rtol=1e-5, atol=1e-5)
    xa = xa.cpu().numpy().reshape(R, K + 1, A)
    np.testing.assert_allclose(xa[:, :K], ar.numpy(), rtol=1e-5, atol=1e-5)
    t_rows = np.zeros((B, n + 1, A), np.float32)
    t_rows[:, :n] = taken.reshape(B, n, A)
    assert np.array_equal(xa[:, K], t_rows.reshape(R, A))
    assert np.array_equal(xs.cpu().numpy().reshape(R, K + 1, D), np.repeat(x[:, None], K + 1, 1))


def _target_inputs(rs, B, n, A, K, cont):
    R = B * (n + 1)
    nout = 2 * A if cont else A
    tout = rs.standard_normal((R, nout)).astype(np.float32)
    tq = rs.standard_normal((R, K + 1) if cont else (R, A)).astype(np.float32)
    if cont:
        act = np.tanh(rs.standard_normal((B * n, A))).astype(np.float32)
        q = rs.standard_normal(B * n).astype(np.float32)
    else:
        act = rs.randint(0, A, B * n)
        q = rs.standard_normal((B * n, A)).astype(np.float32)
    lp = om.logp(torch.tensor(tout, dtype=torch.float64).view(B, n + 1, nout)[:, :n],
                 torch.tensor(act).view(B, n, -1).squeeze(-1) if not cont else torch.tensor(act, dtype=torch.float64).view(B, n, A),
                 A, cont).reshape(-1).numpy()
    log_mu = (lp + rs.uniform(-1, 1, B * n)).astype(np.float32)         # ratios on both sides of 1
    reward = rs.standard_normal(B * n).astype(np.float32)
    done = (rs.uniform(size=B * n) < 0.15).astype(np.float32)
    return dict(tout=tout, tq=tq, act=act, q=q, log_mu=log_mu, reward=reward, done=done)


@pytest.mark.parametrize("retrace", [1, 0])
@pytest.mark.parametrize("n", [8, 32])
@pytest.mark.parametrize("cont,A", [(False, 2), (False, 18), (True, 3), (True, 8)])
def test_critic_target_kernel(cont, A, n, retrace):
    C, ptr, sp = _C()
    rs = np.random.RandomState(A + n)
    B, K, gamma = 37, 30, 0.99
    x = _target_inputs(rs, B, n, A, K, cont)
    S = B * n
    dq = torch.empty((S,) if cont else (S, A), device=DEV)
    qret, stats = torch.empty(S, device=DEV), torch.zeros(16, device=DEV)
    ga = _g(x["act"]) if cont else _g(x["act"], torch.int64)
    C.jb_mpo_critic_target(int(cont), ptr(_g(x["tq"])), ptr(_g(x["tout"])), ptr(_g(x["q"])), ptr(ga), ptr(_g(x["log_mu"])),
                           ptr(_g(x["reward"])), ptr(_g(x["done"])), B, n, A, K, gamma, retrace, ptr(dq), ptr(qret),
                           ptr(stats), sp())
    f = lambda k, *s: torch.tensor(x[k], dtype=torch.float64).view(*s)
    act = f("act", B, n, A) if cont else torch.tensor(x["act"]).view(B, n)
    ref = om.critic_target(f("tout", B, n + 1, -1), f("tq", B, n + 1, -1), act, f("log_mu", B, n), f("reward", B, n),
                           f("done", B, n), gamma, A, cont, bool(retrace)).reshape(-1)
    tol = 1e-5 * (1 + float(ref.abs().max()))
    np.testing.assert_allclose(qret.cpu().numpy(), ref.numpy(), rtol=1e-4, atol=tol)
    qt = torch.tensor(x["q"], dtype=torch.float64)
    if not cont:
        qt = qt.gather(1, torch.tensor(x["act"]).view(-1, 1)).squeeze(1)
    diff = qt - ref
    dref = 2 * diff / S
    if cont:
        np.testing.assert_allclose(dq.cpu().numpy(), dref.numpy(), rtol=1e-4, atol=tol / S)
    else:
        full = torch.zeros(S, A, dtype=torch.float64).scatter_(1, torch.tensor(x["act"]).view(-1, 1), dref.view(-1, 1))
        np.testing.assert_allclose(dq.cpu().numpy(), full.numpy(), rtol=1e-4, atol=tol / S)
    np.testing.assert_allclose(stats[:2].cpu().numpy(), [float((diff ** 2).mean()), float(ref.mean())], rtol=1e-4, atol=tol)


def _policy_call(rs, B, n, A, K, cont, eta=0.7):
    C, ptr, sp = _C()
    S, R = B * n, B * (n + 1)
    nout = 2 * A if cont else A
    tout = rs.standard_normal((R, nout)).astype(np.float32)
    rows = (np.arange(S) // n) * (n + 1) + np.arange(S) % n
    out = (tout[rows] + 0.3 * rs.standard_normal((S, nout))).astype(np.float32)
    if cont:
        out[::5, 0] = 6.0
        tq = rs.standard_normal((R, K + 1)).astype(np.float32)
        z = rs.standard_normal((R, K, A)).astype(np.float32)
    else:
        tq, z = rs.standard_normal((R, A)).astype(np.float32), None
    mult = np.array([eta, 1.3, 0.4], np.float32)
    dout, dmult, stats = torch.empty(S, nout, device=DEV), torch.empty(3, device=DEV), torch.zeros(8, device=DEV)
    part = torch.empty(C.jb_mpo_policy_partials(S), device=DEV)
    C.jb_mpo_policy_loss(int(cont), ptr(_g(out)), ptr(_g(tout)), ptr(_g(tq)), ptr(_g(z) if cont else None), B, n, A, K,
                         ptr(_g(mult)), *EPS, ptr(dout), ptr(dmult), ptr(part), ptr(stats), sp())
    d64 = lambda a: torch.tensor(a, dtype=torch.float64)
    args = (d64(out), d64(tout[rows]), d64(tq[rows][:, :K] if cont else tq[rows]), d64(z[rows]) if cont else None)
    m64 = [torch.tensor(float(v), dtype=torch.float64) for v in mult]
    loss, aux = om.policy_loss(*args, *m64, EPS, A, cont)
    g, dm = om.policy_closed(*args, *m64, EPS, A, cont)
    return dout, dmult, stats, g, dm, aux


@pytest.mark.parametrize("n", [8, 32])
@pytest.mark.parametrize("cont,A", [(False, 2), (False, 18), (True, 3), (True, 8)])
def test_policy_loss_kernel(cont, A, n):
    rs = np.random.RandomState(A * n)
    dout, dmult, stats, g, dm, aux = _policy_call(rs, 21, n, A, 30, cont)
    gmax = float(g.abs().max())
    np.testing.assert_allclose(dout.cpu().numpy(), g.numpy(), rtol=0, atol=2e-6 + 1e-4 * gmax)
    np.testing.assert_allclose(dmult.cpu().numpy(), dm.numpy(), rtol=1e-4, atol=1e-5)
    ref = [aux[k] for k in ("actor_loss", "eta_loss", "alpha_loss", "kl_mu", "kl_sigma")]
    np.testing.assert_allclose(stats[:5].cpu().numpy(), [float(v) for v in ref], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("cont", [False, True])
def test_policy_loss_kernel_at_min_eta(cont):
    rs = np.random.RandomState(11)
    dout, dmult, stats, g, dm, aux = _policy_call(rs, 8, 8, 3, 30, cont, eta=1e-8)
    assert torch.isfinite(dout).all() and torch.isfinite(dmult).all() and torch.isfinite(stats).all()
    np.testing.assert_allclose(dout.cpu().numpy(), g.numpy(), rtol=0, atol=2e-6 + 1e-4 * float(g.abs().max()))
    np.testing.assert_allclose(dmult.cpu().numpy(), dm.numpy(), rtol=1e-4, atol=1e-3)


def test_kernels_reject_bad_arguments():
    from jorldy_b200._lib import JbError
    C, ptr, sp = _C()
    t = torch.zeros(4096, device=DEV)
    p = ptr(t)
    with pytest.raises(JbError):          # n > 32
        C.jb_mpo_critic_target(0, p, p, p, p, p, p, p, 2, 33, 2, 1, 0.99, 1, p, p, p, sp())
    with pytest.raises(JbError):          # continuous A > 8
        C.jb_mpo_policy_loss(1, p, p, p, p, 2, 4, 9, 4, p, *EPS, p, p, p, p, sp())
    with pytest.raises(JbError):          # K > 64
        C.jb_mpo_sample(p, p, 9, 65, 2, p, 4, None, 8, p, p, p, sp())
    with pytest.raises(JbError):          # discrete A > 18
        C.jb_mpo_logp(0, p, 19, p, 4, 19, p, sp())


# ------------------------------------------------------------------------------------------------ 2. collected windows
def _mpo(**kw):
    from jorldy_b200.core.agent.mpo import MPO
    args = dict(hidden_size=64, batch_size=16, n_step=4, buffer_size=4096, start_train_step=0, run_step=10000,
                lr_decay=False, device=DEV, seed=3, optim_config={"name": "adam", "lr": 1e-3})
    args.update(kw)
    return MPO(**args)


@pytest.mark.parametrize("envname", ["cartpole", "hopper"])
def test_collected_windows_match_the_env_steps(envname):
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import NStepAssembler, ReplayCollector
    if envname == "cartpole":
        env = Env("cartpole", action_type="discrete", num_envs=16, seed=1)
        agent = _mpo(state_size=4, action_size=2)
    else:
        env = Env("hopper", num_envs=16, seed=1, p_done=0.05)
        agent = _mpo(state_size=11, action_size=3, actor="continuous_policy", critic="continuous_q_network")
    n, T = agent.n_step, 40
    rec, batches = [], []
    step_device = env.step_device

    def recording_step(action):
        obs = env.obs.clone()
        nxt, r, d = step_device(action)
        rec.append(dict(state=obs, next_state=nxt.clone(), action=action.clone(), reward=r.view(-1).clone(), done=d.view(-1).clone()))
        return nxt, r, d

    env.step_device = recording_step
    col = ReplayCollector(env, agent, update_period=T)
    agent.process = lambda b, step: batches.extend(b) or {}
    col.run_round(0)
    assert len(batches) == T - n + 1
    assert sum(float(r["done"].sum()) for r in rec) > 0, "no episode ended: the done masks go untested"
    plain = NStepAssembler(n)
    for j, r in enumerate(rec):
        ref = plain.push({k: (v.view(v.shape[0], -1) if k == "action" else v) for k, v in r.items()})
        if j < n - 1:
            continue
        w = batches[j - n + 1]
        steps = rec[j - n + 1:j + 1]
        assert w["state"].shape[1] == n + 1 and w["reward"].shape[1] == n
        for t, s in enumerate(steps):
            assert torch.equal(w["state"][:, t], s["state"])
            assert torch.equal(w["action"][:, t].reshape(-1), s["action"].reshape(-1))
            assert torch.equal(w["reward"][:, t], s["reward"]) and torch.equal(w["done"][:, t], s["done"])
            keep = s["done"] == 0
            assert torch.equal(w["state"][:, t + 1][keep], s["next_state"][keep])      # s_{t+1} = next_state_t
        assert torch.equal(w["state"][:, n], steps[-1]["next_state"])
        # the plain n-step window of the same steps is unchanged
        assert torch.equal(ref["state"], w["state"][:, 0]) and torch.equal(ref["next_state"], w["state"][:, n])
        assert torch.equal(ref["reward"].squeeze(-1), w["reward"]) and torch.equal(ref["done"].squeeze(-1), w["done"])
    # log mu is the acting policy's log-probability of the stored action (the weights did not change while collecting)
    p = {k: v.cpu().to(torch.float64) for k, v in agent.actor.state_dict().items()}
    w = batches[0]
    cont = agent.continuous
    out = om.actor_out(p, _d(w["state"][:, :n]), cont)
    act = _d(w["action"]) if cont else w["action"].view(16, n).cpu()
    np.testing.assert_allclose(w["log_mu"].cpu().numpy(), om.logp(out, act, agent.action_size, cont).numpy(),
                               rtol=1e-4, atol=1e-4)


# --------------------------------------------------------------------------------------------------- 3. whole learns
CASES = {
    "cartpole": dict(D=4, A=2, cont=False),
    "hopper": dict(D=11, A=3, cont=True),
}


def _windows(rs, N, n, D, A, cont):
    st = rs.standard_normal((N, n + 1, D)).astype(np.float32)
    if cont:
        act = np.tanh(rs.standard_normal((N, n, A))).astype(np.float32)
    else:
        act = rs.randint(0, A, (N, n, 1)).astype(np.int64)
    return dict(state=st, action=act, reward=rs.standard_normal((N, n)).astype(np.float32),
                done=(rs.uniform(size=(N, n)) < 0.1).astype(np.float32),
                log_mu=(rs.uniform(-2.5, 0.5, (N, n)) * (A if cont else 1)).astype(np.float32))


def _filled(case, N=48, **kw):
    c = CASES[case]
    kw = dict(dict(state_size=c["D"], action_size=c["A"], n_step=8, batch_size=16, num_sample=30, target_update_period=2), **kw)
    if c["cont"]:
        kw.update(actor="continuous_policy", critic="continuous_q_network")
    torch.manual_seed(kw.pop("init_seed", 0))            # the networks' initial weights
    agent = _mpo(**kw)
    data = _windows(np.random.RandomState(7), N, agent.n_step, c["D"], c["A"], c["cont"])
    agent.memory.store([{k: torch.as_tensor(v).to(DEV) for k, v in data.items()}])
    return agent, data


def _oracle_batch(data, idx, cont):
    b = {k: torch.as_tensor(v[idx]) for k, v in data.items()}
    if not cont:
        b["action"] = b["action"][..., 0]
    return b


def _compare_nets(net, ref, lr):
    for k, v in ref.items():
        np.testing.assert_allclose(net.p[k].cpu().numpy(), v.detach().numpy(), rtol=0, atol=0.1 * lr, err_msg=k)


def _compare_moments(opt, ref_opt, params):
    for i, (m, v) in enumerate(zip(opt._slot_views(opt.exp_avg), opt._slot_views(opt.exp_avg_sq))):
        st = ref_opt.state[params[i]]
        for got, want in ((m, st["exp_avg"]), (v, st["exp_avg_sq"])):
            want = want.detach().numpy()
            np.testing.assert_allclose(got.cpu().numpy(), want, rtol=5e-3, atol=1e-3 * np.abs(want).max() + 1e-9)


@pytest.mark.parametrize("case", list(CASES))
def test_eager_learns_match_the_float64_oracle(case):
    """Three learns with target_update_period 2: the second ends with the hard target copy, the third reads it."""
    lr = 1e-3
    agent, data = _filled(case)
    c = CASES[case]
    hp = dict(continuous=c["cont"], A=c["A"], gamma=agent.gamma, lr=lr, clip_grad_norm=1.0, target_update_period=2,
              critic_loss_type="retrace", eps=EPS, mins=MINS)
    cpu = lambda net: {k: v.cpu() for k, v in net.state_dict().items()}
    ref = om.Learner(cpu(agent.actor), cpu(agent.critic), [1.0, 1.0, 1.0], hp)
    rs = np.random.RandomState(0)
    for it in range(3):
        idx = rs.randint(0, 48, 16)
        R = 16 * (agent.n_step + 1)
        eps = rs.standard_normal((R, 30, c["A"])).astype(np.float32)
        agent._inject_idx = idx
        agent._inject_noise = {"sample": _g(eps)} if c["cont"] else {}
        res = agent.learn()
        want, qret = ref.learn(_oracle_batch(data, idx, c["cont"]), torch.tensor(eps, dtype=torch.float64).view(16, agent.n_step + 1, 30, c["A"]))
        for k in ("critic_loss", "actor_loss", "eta_loss", "alpha_loss", "mean_Q", "eta", "alpha_mu", "alpha_sigma"):
            assert abs(res[k] - want[k]) <= 1e-3 * (1 + abs(want[k])), (it, k, res[k], want[k])
        np.testing.assert_allclose(agent._qret.cpu().numpy(), qret.reshape(-1).numpy(), rtol=1e-3, atol=1e-3)
        _compare_nets(agent.actor, ref.actor, lr)
        _compare_nets(agent.critic, ref.critic, lr)
        _compare_nets(agent.target_actor, ref.t_actor, lr)
        _compare_nets(agent.target_critic, ref.t_critic, lr)
        np.testing.assert_allclose(agent.mult.flat[:3].cpu().numpy(), [float(m) for m in ref.mult], rtol=1e-4, atol=1e-6)
    _compare_moments(agent.actor_optimizer, ref.actor_opt, list(ref.actor.values()))
    _compare_moments(agent.critic_optimizers[0], ref.critic_opt, list(ref.critic.values()))
    assert not torch.equal(agent.target_actor.flat, agent.actor.flat)        # copied after learn 2, stale after learn 3


@pytest.mark.parametrize("case", list(CASES))
def test_graph_learn_is_bit_identical_to_eager_and_reproducible(case):
    idx = [np.random.RandomState(i).randint(0, 48, 16) for i in range(5)]

    def run(graph):
        agent, _ = _filled(case, use_cuda_graph=graph)
        out = []
        for i in idx:
            agent._inject_idx = i
            out.append(agent.learn())
        torch.cuda.synchronize()
        return agent, out

    g1, r1 = run(True)
    g2, r2 = run(True)
    e, re = run(False)
    assert len(g1._graphs) == 2                            # with and without the target copy
    for a in (g2, e):
        for x, y in ((g1.actor, a.actor), (g1.critic, a.critic), (g1.target_actor, a.target_actor), (g1.mult, a.mult)):
            assert torch.equal(x.flat, y.flat)
        assert torch.equal(g1.actor_optimizer.exp_avg, a.actor_optimizer.exp_avg)
    assert r1 == r2 == re


# ------------------------------------------------------------------------------------------ 4. checkpoint, attach
def test_checkpoint_round_trip_and_layout(tmp_path):
    agent, _ = _filled("hopper")
    for i in range(3):
        agent._inject_idx = np.arange(16) + i
        agent.learn()
    agent.save(str(tmp_path))
    ck = torch.load(str(tmp_path / "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"actor", "critic", "actor_optimizer", "critic_optimizer", "eta", "alpha_mu", "alpha_sigma"}
    P = len(agent.actor.p)
    assert sorted(ck["actor_optimizer"]["state"]) == list(range(P + 3))
    assert ck["actor_optimizer"]["param_groups"][0]["params"] == list(range(P + 3))
    assert sorted(ck["critic_optimizer"]["state"]) == list(range(len(agent.critic.p)))
    assert float(ck["eta"]) == float(agent.mult.flat[0])
    b, _ = _filled("hopper", seed=9, init_seed=9)
    b.load(str(tmp_path))
    for x, y in ((agent.actor, b.actor), (agent.critic, b.critic)):
        assert torch.equal(x.flat, y.flat)
    assert torch.equal(agent.mult.flat[:3], b.mult.flat[:3])
    assert torch.equal(b.target_actor.flat, b.actor.flat) and torch.equal(b.target_critic.flat, b.critic.flat)
    for o1, o2 in ((agent.actor_optimizer, b.actor_optimizer), (agent.critic_optimizers[0], b.critic_optimizers[0]),
                   (agent.mult_optimizer, b.mult_optimizer)):
        assert torch.equal(o1.exp_avg, o2.exp_avg) and torch.equal(o1.exp_avg_sq, o2.exp_avg_sq)
        assert int(o1._step_dev) == int(o2._step_dev)


def test_attach_keeps_mpo_a_replica():
    from jorldy_b200.core import parallel
    agent = _mpo(state_size=4, action_size=2)
    with pytest.warns(UserWarning, match="MPO: replicas only \\(no data-parallel learner for MPO\\)"):
        parallel.attach(agent, 2)
    assert agent.world_size == 1


# -------------------------------------------------------------------------------------------------- 5. end to end
@pytest.mark.parametrize("config,extra", [
    ("config.mpo.cartpole", ["--train.num_workers", "8", "--agent.start_train_step", "256", "--agent.hidden_size", "64"]),
    ("config.mpo.mujoco", ["--env.name", "hopper", "--train.num_workers", "16", "--train.update_period", "32",
                           "--agent.start_train_step", "512", "--agent.hidden_size", "64"]),
])
def test_sync_training_run_with_save_and_load(tmp_path, config, extra):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base = [sys.executable, "-m", "jorldy_b200.main", "--sync", "--config", config, "--train.run_step", "2048",
            "--train.print_period", "1024", "--train.save_period", "2048", *extra]
    r = subprocess.run(base, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith("2048 step |") and "critic_loss" in line for line in r.stdout.splitlines()), out[-4000:]
    ckpts = [d for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    saved = torch.load(os.path.join(ckpts[0], "ckpt"), map_location="cpu", weights_only=False)
    assert {"actor", "critic", "actor_optimizer", "critic_optimizer", "eta", "alpha_mu", "alpha_sigma"} <= set(saved)
    assert all(np.isfinite(float(saved[k])) for k in ("eta", "alpha_mu", "alpha_sigma"))
    r2 = subprocess.run(base + ["--train.load_path", ckpts[0]], cwd=tmp_path / "logs", env=env, capture_output=True,
                        text=True, timeout=900)
    out2 = r2.stdout + r2.stderr
    assert "Traceback" not in out2 and "Load model from" in out2, out2[-4000:]
