"""V-MPO on the GPU (pytest -m gpu): jb_vmpo_loss against the float64 oracle (oracle/vmpo.py), eager learns against
the oracle's learn on CartPole, Hopper and Atari-frame shapes, the CUDA-graph path against eager, determinism, the
persistent PPO kernel staying off, checkpoints, parallel.attach and end-to-end runs of main --sync.

Tolerances (fp32 kernels against float64):
  dout                          : atol 2e-6 + 1e-4 * max|dout|   (per row a few exp / log / divide round-offs)
  dmult, losses, stats          : rtol 1e-4, atol 1e-5 (d eta at eta = min_eta: atol 1e-3, z = adv / eta ~ 1e8)
  parameters after a learn      : atol 0.1 * lr (Adam normalises the update to ~lr), CNN: normwise 2e-2 of the update
  Adam moments                  : atol 1e-3 * max|moment| + tiny, rtol 5e-3
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import vmpo as ov

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
EPS = (0.01, 0.01, 5e-5)


def _C():
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    return C, ptr, stream_ptr


# ------------------------------------------------------------------------------------------------ 1. the loss kernel
def _inputs(rs, B, A, continuous, kind):
    NT = B + 5
    nout = 2 * A + 1 if continuous else A + 1
    out_old = rs.standard_normal((NT, nout)).astype(np.float32)
    idx = rs.permutation(NT)[:B].astype(np.int32)
    out = out_old[idx] + 0.3 * rs.standard_normal((B, nout)).astype(np.float32)
    if continuous:
        action = rs.uniform(-0.999, 0.999, (NT, A)).astype(np.float32)
        out[:, 0] = np.where(rs.uniform(size=B) < 0.2, 6.0, out[:, 0])      # clamped mu rows
    else:
        action = rs.randint(0, A, NT).astype(np.int32)
    adv = rs.standard_normal(NT).astype(np.float32)
    ret = rs.standard_normal(NT).astype(np.float32)
    mult = np.array([0.7, 1.3, 0.4], np.float32)
    if kind == "ties":              # a third of the rows equal the median value
        adv[idx[rs.uniform(size=B) < 0.34]] = 0.125
    elif kind == "all_equal":
        adv[:] = -0.5
    elif kind == "min_eta":
        mult[0] = 1e-8
    elif kind == "zero_kl":
        out = out_old[idx].copy()
    elif kind == "tiny_p_old":      # old probabilities of 1e-13 (below fp32 eps) for action 0
        if not continuous:
            out_old[:, 0] = -30.0
    return dict(out=out, out_old=out_old, idx=idx, action=action, adv=adv, ret=ret, mult=mult, A=A, cont=continuous)


def _run_kernel(c):
    C, ptr, sp = _C()
    t = {k: torch.from_numpy(np.ascontiguousarray(c[k])).to(DEV) for k in ("out", "out_old", "idx", "action", "adv", "ret", "mult")}
    B, nout = c["out"].shape
    dout = torch.full((B, nout), float("nan"), device=DEV)
    dmult = torch.empty(3, device=DEV)
    stats = torch.empty(16 + 4 * ((B + 255) // 256), device=DEV)
    acc = torch.zeros(8, device=DEV)
    C.jb_vmpo_loss(int(c["cont"]), ptr(t["out"]), ptr(t["out_old"]), ptr(t["idx"]), ptr(t["action"]), ptr(t["adv"]),
                   ptr(t["ret"]), B, c["A"], nout, ptr(t["mult"]), *EPS, ptr(dout), ptr(dmult), ptr(stats), ptr(acc), sp())
    torch.cuda.synchronize()
    return dout.cpu().numpy(), dmult.cpu().numpy(), stats.cpu().numpy(), acc.cpu().numpy()


def _oracle(c):
    d = lambda a: torch.from_numpy(np.asarray(a)).double()
    idx = c["idx"].astype(np.int64)
    args = (d(c["out"]), d(c["out_old"][idx]), d(c["action"][idx]), d(c["adv"][idx]), d(c["ret"][idx]))
    mult = [torch.tensor(float(v), dtype=torch.float64) for v in c["mult"]]
    g, dm = ov.closed_form(*args, *mult, EPS, c["A"], c["cont"])
    _, aux = ov.minibatch_loss(*args, *mult, EPS, c["A"], c["cont"])
    return g.numpy(), dm.numpy(), aux


@pytest.mark.parametrize("kind", ["random", "ties", "all_equal", "min_eta", "zero_kl", "tiny_p_old"])
@pytest.mark.parametrize("B", [1, 2, 31, 256, 257, 2048])
@pytest.mark.parametrize("cont,A", [(False, 2), (False, 4), (False, 18), (True, 1), (True, 3), (True, 8)])
def test_loss_kernel_matches_the_float64_oracle(cont, A, B, kind):
    rs = np.random.RandomState(B * 7 + A + (100 if cont else 0))
    c = _inputs(rs, B, A, cont, kind)
    dout, dmult, stats, acc = _run_kernel(c)
    g, dm, aux = _oracle(c)
    assert np.all(np.isfinite(dout)) and np.all(np.isfinite(dmult)) and np.all(np.isfinite(stats[:8]))
    np.testing.assert_allclose(dout, g, rtol=0, atol=2e-6 + 1e-4 * np.abs(g).max(), err_msg="dout")
    np.testing.assert_allclose(dmult[1:], dm[1:], rtol=1e-4, atol=1e-5, err_msg="dmult")
    np.testing.assert_allclose(dmult[0], dm[0], rtol=1e-4, atol=1e-3 if kind == "min_eta" else 1e-5, err_msg="d eta")
    assert stats[6] == aux["n"] and stats[7] == np.float32(float(aux["median"]))
    for i, k in enumerate(("actor_loss", "critic_loss", "eta_loss", "alpha_loss", "kl_mu", "kl_sigma")):
        np.testing.assert_allclose(stats[i], float(aux[k]), rtol=1e-4, atol=1e-5, err_msg=k)
    np.testing.assert_array_equal(acc[:4], stats[:4])
    assert acc[4] == 1.0
    if kind == "all_equal":
        assert aux["n"] == 0 and dmult[0] == 0.0 and stats[0] == 0.0 and stats[2] == 0.0
    if kind == "zero_kl":
        assert abs(stats[4]) < 1e-6 and abs(stats[5]) < 1e-6
    if not cont:
        assert dmult[2] == 0.0


def test_loss_kernel_is_bit_reproducible():
    c = _inputs(np.random.RandomState(0), 2048, 18, False, "ties")
    r1, r2 = _run_kernel(c), _run_kernel(c)
    for a, b in zip(r1, r2):
        assert np.array_equal(a, b)


def test_loss_kernel_rejects_bad_arguments():
    from jorldy_b200._lib import JbError
    C, ptr, sp = _C()
    ins, outs = torch.ones(4096, device=DEV), [torch.zeros(4096, device=DEV) for _ in range(3)]
    ib = torch.zeros(64, dtype=torch.int32, device=DEV)
    p = ptr(ins)
    dout, dmult, stats = (ptr(t) for t in outs)

    def call(cont=0, B=8, A=2, nout=3, out=p, act=ptr(ib), mult=p):
        C.jb_vmpo_loss(cont, out, p, ptr(ib), act, p, p, B, A, nout, mult, *EPS, dout, dmult, stats, 0, sp())
    call()
    torch.cuda.synchronize()
    for kw in (dict(B=0), dict(B=-3), dict(A=0), dict(A=19, nout=20), dict(cont=1, A=9, nout=19), dict(nout=4),
               dict(cont=1, A=2, nout=3), dict(out=0), dict(act=0), dict(mult=0)):
        with pytest.raises(JbError):
            call(**kw)


# ------------------------------------------------------------------------------------------------- 2. learn
CASES = {
    "cartpole_h64": dict(seed=31, N=4, T=32, D=4, A=2, H=64, continuous=False, batch_size=32, n_epoch=2, lr=2.5e-4),
    "cartpole_h512": dict(seed=32, N=8, T=64, D=4, A=2, H=512, continuous=False, batch_size=256, n_epoch=2, lr=2.5e-4),
    "hopper": dict(seed=33, N=4, T=64, D=11, A=3, H=256, continuous=True, batch_size=64, n_epoch=2, lr=3e-4),
}
MULT0 = (1.0, 5.0, 1.0)
MINS = (1e-8, 1e-8, 1e-8)


def _agent(case, **kw):
    from jorldy_b200.core import Agent
    net = "continuous_policy_value" if case["continuous"] else "discrete_policy_value"
    return Agent("vmpo", state_size=case["D"], action_size=case["A"], hidden_size=case["H"], network=net,
                 optim_config={"name": "adam", "lr": case["lr"]}, gamma=0.99, use_standardization=True, run_step=1000,
                 lr_decay=False, device=DEV, batch_size=case["batch_size"], n_step=case["T"], n_epoch=case["n_epoch"],
                 _lambda=0.95, clip_grad_norm=1.0, eta=MULT0[0], alpha_mu=MULT0[1], alpha_sigma=MULT0[2],
                 eps_eta=EPS[0], eps_alpha_mu=EPS[1], eps_alpha_sigma=EPS[2], **kw)


def _batch(case):
    rs = np.random.RandomState(case["seed"])
    NT, D, A = case["N"] * case["T"], case["D"], case["A"]
    state = rs.standard_normal((NT, D)).astype(np.float32)
    next_state = rs.standard_normal((NT, D)).astype(np.float32)
    action = (rs.uniform(-0.95, 0.95, (NT, A)) if case["continuous"] else rs.randint(0, A, (NT, 1))).astype(np.float32)
    reward = rs.standard_normal((NT, 1)).astype(np.float32)
    done = (rs.uniform(size=(NT, 1)) < 0.05).astype(np.float32)
    perms = [rs.permutation(NT) for _ in range(case["n_epoch"])]
    return {k: torch.from_numpy(v) for k, v in dict(state=state, next_state=next_state, action=action, reward=reward,
                                                     done=done).items()}, perms


def _learn(agent, case, batch, perms):
    agent._inject_perms = perms
    action = batch["action"].to(DEV)
    action = action if case["continuous"] else action.reshape(-1).to(torch.int32)
    res = agent._learn_tensors(batch["state"].to(DEV), action, batch["reward"].reshape(-1).to(DEV),
                               batch["done"].reshape(-1).to(DEV), next_state=batch["next_state"].to(DEV))
    torch.cuda.synchronize()
    return res


def _hp(case):
    return {"continuous": case["continuous"], "A": case["A"], "n_step": case["T"], "gamma": 0.99, "lambda": 0.95,
            "standardize": True, "batch_size": case["batch_size"], "n_epoch": case["n_epoch"], "clip_grad_norm": 1.0}


def _check_moments(agent, ref, names, scale_tol=1e-3):
    st = ref["opt_state"]["state"]
    m, v = agent.optimizer._slot_views(agent.optimizer.exp_avg), agent.optimizer._slot_views(agent.optimizer.exp_avg_sq)
    for i, k in enumerate(names):
        for got, key in ((m[i], "exp_avg"), (v[i], "exp_avg_sq")):
            r = st[i][key].numpy()
            np.testing.assert_allclose(got.cpu().numpy(), r, rtol=5e-3, atol=scale_tol * np.abs(r).max() + 1e-12,
                                       err_msg=f"{key} {k}")
    P = len(names)
    for j in range(3):
        for key, buf in (("exp_avg", agent.mult_optimizer.exp_avg), ("exp_avg_sq", agent.mult_optimizer.exp_avg_sq)):
            r = float(st[P + j][key])
            np.testing.assert_allclose(float(buf[j]), r, rtol=5e-3, atol=1e-6 * max(1.0, abs(r)), err_msg=f"{key} mult {j}")


@pytest.mark.parametrize("name", list(CASES))
def test_eager_learn_matches_the_float64_oracle(name):
    case = CASES[name]
    agent = _agent(case, use_cuda_graph=False)
    batch, perms = _batch(case)
    params = {k: v.detach().cpu().clone() for k, v in agent.network.p.items()}
    res = _learn(agent, case, batch, perms)
    ref = ov.learn(params, batch, _hp(case), perms, case["lr"], MULT0, MINS, EPS)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(agent.network.p[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)
    for k, v in ref["result"].items():
        np.testing.assert_allclose(res[k], v, rtol=2e-4, atol=2e-4, err_msg=k)
    np.testing.assert_allclose(agent.mult.flat[:3].cpu().numpy(), ref["mult"], rtol=1e-4, atol=1e-6)
    _check_moments(agent, ref, list(params))
    if not case["continuous"]:
        assert res["alpha_sigma"] == np.float32(MULT0[2])


def test_eager_learn_on_atari_frames_with_the_cnn_head_matches_the_float64_oracle():
    """A = 18, the CNN head on uint8 frame stacks; 2 Adam steps.  A ReLU input within fp32 round-off of 0 can take the
    other side in float64, so parameters are compared normwise against the update."""
    from jorldy_b200.core import Agent
    N, T, B, A, lr = 4, 8, 16, 18, 2.5e-4
    case = dict(continuous=False, A=A, T=T, batch_size=B, n_epoch=1)
    agent = Agent("vmpo", state_size=[4, 84, 84], action_size=A, hidden_size=64, network="discrete_policy_value",
                  head="cnn", optim_config={"name": "adam", "lr": lr}, run_step=1000, lr_decay=False, device=DEV,
                  batch_size=B, n_step=T, n_epoch=1, use_cuda_graph=False, eta=MULT0[0], alpha_mu=MULT0[1],
                  alpha_sigma=MULT0[2], eps_eta=EPS[0], eps_alpha_mu=EPS[1], eps_alpha_sigma=EPS[2])
    rs = np.random.RandomState(8)
    state = torch.from_numpy(rs.randint(0, 256, (N * T, 4, 84, 84)).astype(np.uint8))
    nxt = torch.from_numpy(rs.randint(0, 256, (N * T, 4, 84, 84)).astype(np.uint8))
    action = torch.from_numpy(rs.randint(0, A, (N * T, 1)).astype(np.float32))
    reward = torch.from_numpy(rs.standard_normal((N * T, 1)).astype(np.float32))
    done = torch.from_numpy((rs.uniform(size=(N * T, 1)) < 0.1).astype(np.float32))
    perms = [rs.permutation(N * T)]
    params = {k: v.detach().cpu().clone() for k, v in agent.network.p.items()}
    agent._inject_perms = perms
    res = agent._learn_tensors(state.to(DEV), action.reshape(-1).to(torch.int32).to(DEV), reward.reshape(-1).to(DEV),
                               done.reshape(-1).to(DEV), next_state=nxt.to(DEV))
    torch.cuda.synchronize()
    batch = dict(state=state.double(), next_state=nxt.double(), action=action, reward=reward, done=done)
    ref = ov.learn(params, batch, dict(_hp(case), clip_grad_norm=agent.clip_grad_norm), perms, lr, MULT0, MINS, EPS)
    for k, v in ref["params"].items():
        upd = (v - params[k].double()).norm().item()
        err = (agent.network.p[k].cpu().double() - v).norm().item()
        assert err <= 2e-2 * upd + 1e-9, (k, err, upd)
    for k, v in ref["result"].items():
        np.testing.assert_allclose(res[k], v, rtol=1e-3, atol=1e-3, err_msg=k)
    np.testing.assert_allclose(agent.mult.flat[:3].cpu().numpy(), ref["mult"], rtol=1e-4, atol=1e-6)


def test_graph_learn_is_bit_identical_to_eager_and_reproducible(monkeypatch):
    import jorldy_b200.core.agent.ppo as ppo_mod
    monkeypatch.setattr(ppo_mod, "GRAPH_CHUNK", 2)
    case = dict(CASES["cartpole_h64"], N=8, T=40, batch_size=24)          # 13 full minibatches + a tail of 8
    batch, perms = _batch(case)
    agents = [_agent(case, use_cuda_graph=g) for g in (True, False, True)]
    for a in agents[1:]:
        a.network.load_state_dict(agents[0].network.state_dict())
    results = [[_learn(a, case, batch, perms) for _ in range(2)] for a in agents]
    assert agents[0]._graphs and not agents[1]._graphs
    for a, r in zip(agents[1:], results[1:]):
        assert r == results[0]
        assert torch.equal(a.network.flat, agents[0].network.flat) and torch.equal(a.mult.flat, agents[0].mult.flat)
        state = lambda g: [*g.optimizer.state_tensors(), *g.mult_optimizer.state_tensors(), g._acc]
        for x, y in zip(state(a), state(agents[0])):
            assert torch.equal(x, y)


def test_the_persistent_ppo_kernel_is_never_used():
    case = CASES["cartpole_h64"]                  # MLP head, B % 32 == 0, H <= 512: a PPO agent would take ppo_fused
    from jorldy_b200.core.agent import ppo_fused
    agent = _agent(case, use_fused=True)
    assert agent.use_fused is False and ppo_fused.supported(agent, case["batch_size"])
    batch, perms = _batch(case)
    _learn(agent, case, batch, perms)
    assert agent._fused == {}
    assert agent.n_launches == agent.LAUNCHES_PER_MINIBATCH * case["n_epoch"] * (case["N"] * case["T"] // case["batch_size"])


# ------------------------------------------------------------------------------------------ 3. checkpoint, attach
def test_checkpoint_round_trip_and_layout(tmp_path):
    case = CASES["hopper"]
    a = _agent(case, use_cuda_graph=False)
    batch, perms = _batch(case)
    _learn(a, case, batch, perms)
    a.save(str(tmp_path))
    ck = torch.load(str(tmp_path / "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "optimizer", "eta", "alpha_mu", "alpha_sigma"}
    P = len(a.network.p)
    assert ck["optimizer"]["param_groups"][0]["params"] == list(range(P + 3))
    assert sorted(ck["optimizer"]["state"]) == list(range(P + 3)) and ck["optimizer"]["state"][P]["exp_avg"].shape == ()
    assert float(ck["eta"]) == float(a.mult.flat[0])
    b = _agent(case, seed=9)
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, a.network.flat) and torch.equal(b.mult.flat, a.mult.flat)
    for x, y in zip(b.optimizer.state_tensors() + b.mult_optimizer.state_tensors(),
                    a.optimizer.state_tensors() + a.mult_optimizer.state_tensors()):
        assert torch.equal(x, y)
    for k in ("eta", "alpha_mu", "alpha_sigma"):
        del ck[k]
    torch.save(ck, str(tmp_path / "ckpt"))
    c = _agent(case)
    c.load(str(tmp_path))
    assert c.mult.flat[:3].tolist() == [np.float32(v) for v in MULT0]


def test_attach_keeps_vmpo_a_replica():
    from jorldy_b200.core import parallel
    a = _agent(CASES["cartpole_h64"])
    with pytest.warns(UserWarning, match="replicas only"):
        parallel.attach(a, 2)
    assert a.world_size == 1 and a.allreduce is None


# -------------------------------------------------------------------------------------------------- 4. end to end
@pytest.mark.parametrize("config,extra", [
    ("config.vmpo.cartpole", ["--train.num_workers", "8", "--agent.n_step", "32"]),
    ("config.vmpo.mujoco", ["--env.name", "hopper", "--train.num_workers", "16", "--agent.n_step", "32",
                            "--agent.batch_size", "64", "--agent.hidden_size", "64", "--train.update_period", "32",
                            "--train.distributed_batch_size", "64"]),
    ("config.vmpo.atari", ["--env.name", "seaquest", "--train.num_workers", "16", "--agent.n_step", "32",
                           "--agent.hidden_size", "64"]),
])
def test_sync_training_run(tmp_path, config, extra):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable, "-m", "jorldy_b200.main", "--sync", "--config", config, "--train.run_step", "1024",
           "--train.print_period", "512", "--train.save_period", "1024", *extra]
    r = subprocess.run(cmd, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith("1024 step |") for line in r.stdout.splitlines()), out[-4000:]
    ckpts = [d for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    saved = torch.load(os.path.join(ckpts[0], "ckpt"), map_location="cpu", weights_only=False)
    assert {"eta", "alpha_mu", "alpha_sigma"} <= set(saved) and all(np.isfinite(float(saved[k])) for k in ("eta", "alpha_mu"))
    P = len(saved["network"])
    assert sorted(saved["optimizer"]["state"]) == list(range(P + 3))      # at least one learn stepped all parameters
