"""ICM-PPO on the GPU (pytest -m gpu): jb_icm_loss against the float64 oracle (oracle/icm_ppo.py), the BatchNorm + ELU
kernels against float64 autograd, the running statistics against numpy, the rollout's next_state column at done steps,
eager learns against the oracle's learn, the CUDA-graph path against eager, the persistent PPO kernel staying off,
checkpoints, parallel.attach and end-to-end runs of main --sync.

Tolerances (fp32 kernels against float64):
  ICM loss gradients            : atol 1e-7 + 1e-5 * max|grad|;  r_i, losses: rtol 1e-5, atol 1e-6
  BatchNorm + ELU               : y / dx atol 1e-5 * scale, dgamma / dbeta and running buffers rtol 1e-4
  parameters after a learn      : atol 0.1 * lr (Adam normalises the update to ~lr)
  Adam moments                  : atol 1e-3 * max|moment| + tiny, rtol 5e-3
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import icm_ppo as oi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
FW = 256


def _C():
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    return C, ptr, stream_ptr


# ------------------------------------------------------------------------------------------------ 1. the loss kernel
def _loss_inputs(rs, B, A, cont):
    NT = B + 3
    f = rs.standard_normal((B, FW)).astype(np.float32)
    pp = rs.standard_normal((B, 2 * FW)).astype(np.float32)          # phi(s') is the second half, ld 2F
    g = (3 * rs.standard_normal((B, A))).astype(np.float32)
    idx = rs.permutation(NT)[:B].astype(np.int32)
    action = rs.uniform(-1, 1, (NT, A)).astype(np.float32) if cont else rs.randint(0, A, NT).astype(np.int32)
    return dict(f=f, pp=pp, g=g, idx=idx, action=action)


def _run_loss(c, A, cont, eta, beta, reward_only=False):
    C, ptr, sp = _C()
    t = {k: torch.from_numpy(v).to(DEV) for k, v in c.items()}
    B = c["f"].shape[0]
    ri = torch.full((B,), float("nan"), device=DEV)
    df = torch.full((B, FW), float("nan"), device=DEV)
    dg = torch.full((B, A), float("nan"), device=DEV)
    stats = torch.full((4 + 3 * ((B + 7) // 8),), float("nan"), device=DEV)
    acc = torch.zeros(4, device=DEV)
    if reward_only:
        C.jb_icm_loss(int(cont), ptr(t["f"]), ptr(t["pp"][:, FW:]), 2 * FW, 0, 0, 0, B, A, FW, eta, beta, ptr(ri), 0, 0,
                      0, 0, sp())
    else:
        C.jb_icm_loss(int(cont), ptr(t["f"]), ptr(t["pp"][:, FW:]), 2 * FW, ptr(t["g"]), ptr(t["idx"]), ptr(t["action"]),
                      B, A, FW, eta, beta, ptr(ri), ptr(df), ptr(dg), ptr(stats), ptr(acc), sp())
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (ri, df, dg, stats, acc)]


@pytest.mark.parametrize("beta", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("eta", [0.0, 0.01])
@pytest.mark.parametrize("B", [1, 7, 256, 257, 2048])
@pytest.mark.parametrize("cont,A", [(False, 2), (False, 4), (False, 18), (True, 1), (True, 3), (True, 8)])
def test_loss_kernel_matches_the_float64_oracle(cont, A, B, eta, beta):
    rs = np.random.RandomState(B * 31 + A + (100 if cont else 0))
    c = _loss_inputs(rs, B, A, cont)
    ri, df, dg, stats, acc = _run_loss(c, A, cont, eta, beta)
    d = lambda a: torch.from_numpy(np.asarray(a)).double()
    act = d(c["action"][c["idx"]])
    f, phi_n, g = d(c["f"]), d(c["pp"][:, FW:]), d(c["g"])
    r_ref, l_f, l_i, l_tot = oi.icm_loss(f, phi_n, g, act, A, cont, eta, beta)
    df_ref, dg_ref = oi.closed_form(f, phi_n, g, act, A, cont, beta)
    np.testing.assert_allclose(ri, r_ref.numpy(), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(df, df_ref.numpy(), rtol=0, atol=1e-7 * beta + 1e-5 * np.abs(df_ref.numpy()).max())
    np.testing.assert_allclose(dg, dg_ref.numpy(), rtol=0, atol=1e-7 + 1e-5 * np.abs(dg_ref.numpy()).max())
    for i, v in enumerate((r_ref.mean(), l_f, l_i, l_tot)):
        np.testing.assert_allclose(stats[i], float(v), rtol=1e-5, atol=1e-6, err_msg=str(i))
    np.testing.assert_array_equal(acc[:3], stats[:3])
    assert acc[3] == 1.0
    # the reward-only pre-pass writes the same r_i and nothing else
    ri2, df2, dg2, stats2, _ = _run_loss(c, A, cont, eta, beta, reward_only=True)
    np.testing.assert_array_equal(ri2, ri)
    assert np.isnan(df2).all() and np.isnan(dg2).all() and np.isnan(stats2).all()


def test_loss_kernel_is_bit_reproducible():
    c = _loss_inputs(np.random.RandomState(0), 2048, 18, False)
    r1, r2 = _run_loss(c, 18, False, 0.01, 0.2), _run_loss(c, 18, False, 0.01, 0.2)
    for a, b in zip(r1, r2):
        assert np.array_equal(a, b, equal_nan=True)


def test_loss_kernel_rejects_bad_arguments():
    from jorldy_b200._lib import JbError
    C, ptr, sp = _C()
    buf = torch.zeros(1 << 16, device=DEV)
    ib = torch.zeros(64, dtype=torch.int32, device=DEV)
    p = ptr(buf)

    def call(cont=0, B=8, A=2, F=FW, f=p, ld=2 * FW, g=p, act=ptr(ib), ri=p, df=p, dg=p, stats=p):
        C.jb_icm_loss(cont, f, p, ld, g, 0, act, B, A, F, 0.01, 0.2, ri, df, dg, stats, 0, sp())
    call()
    call(df=0, dg=0, g=0, act=0, stats=0)
    torch.cuda.synchronize()
    for kw in (dict(B=0), dict(A=0), dict(A=19), dict(cont=1, A=9), dict(F=128), dict(F=512, ld=1024), dict(ld=100),
               dict(f=0), dict(g=0), dict(act=0), dict(stats=0), dict(df=0), dict(dg=0), dict(df=0, dg=0, ri=0)):
        with pytest.raises(JbError):
            call(**kw)


# ----------------------------------------------------------------------------------------- 2. BatchNorm + ELU
@pytest.mark.parametrize("bn", [True, False])
@pytest.mark.parametrize("M", [2, 255, 256, 257, 65537])
def test_bn_elu_forward_and_backward_match_float64_autograd(M, bn):
    C, ptr, sp = _C()
    N = 256
    rs = np.random.RandomState(M + bn)
    x = (rs.standard_normal((M, N)) * 2 + 0.5).astype(np.float32)
    gamma = rs.uniform(0.5, 1.5, N).astype(np.float32)
    beta = (0.3 * rs.standard_normal(N)).astype(np.float32)
    dy = rs.standard_normal((M, N)).astype(np.float32)
    rm0, rv0 = (0.1 * rs.standard_normal(N)).astype(np.float32), rs.uniform(0.5, 2, N).astype(np.float32)
    tx, tg, tb, tdy = (torch.from_numpy(a).to(DEV) for a in (x, gamma, beta, dy))
    rm, rv = torch.from_numpy(rm0).to(DEV), torch.from_numpy(rv0).to(DEV)
    nbt = torch.zeros((), dtype=torch.int64, device=DEV)
    mean, invstd = torch.empty(N, device=DEV), torch.empty(N, device=DEV)
    part = torch.empty(C.jb_col_partials_doubles(M, N), dtype=torch.float64, device=DEV)
    y = torch.empty(M, N, device=DEV)
    dx, xhat = torch.empty(M, N, device=DEV), torch.empty(M, N, device=DEV)
    dgam, dbet = torch.empty(N, device=DEV), torch.empty(N, device=DEV)
    if bn:
        C.jb_bn_elu_fwd(ptr(tx), M, N, ptr(tg), ptr(tb), ptr(rm), ptr(rv), ptr(nbt), 0.1, 1e-5, ptr(mean), ptr(invstd),
                        ptr(part), ptr(y), N, 0, 0, sp())
        C.jb_bn_elu_bwd(ptr(tdy), N, ptr(y), N, ptr(tx), M, N, ptr(tg), ptr(mean), ptr(invstd), ptr(xhat), ptr(part),
                        ptr(dx), ptr(dgam), ptr(dbet), sp())
    else:
        C.jb_bn_elu_fwd(ptr(tx), M, N, 0, 0, 0, 0, 0, 0.0, 0.0, 0, 0, 0, ptr(y), N, 0, 0, sp())
        C.jb_bn_elu_bwd(ptr(tdy), N, ptr(y), N, 0, M, N, 0, 0, 0, 0, 0, ptr(dx), 0, 0, sp())
    torch.cuda.synchronize()
    X = torch.from_numpy(x).double().requires_grad_(True)
    G = torch.from_numpy(gamma).double().requires_grad_(True)
    Bt = torch.from_numpy(beta).double().requires_grad_(True)
    rm_ref, rv_ref = torch.from_numpy(rm0).double(), torch.from_numpy(rv0).double()
    u = F.batch_norm(X, rm_ref, rv_ref, G, Bt, training=True, momentum=0.1, eps=1e-5) if bn else X
    Y = F.elu(u)
    Y.backward(torch.from_numpy(dy).double())
    np.testing.assert_allclose(y.cpu().numpy(), Y.detach().numpy(), rtol=0, atol=1e-5 * (1 + float(Y.abs().max())))
    np.testing.assert_allclose(dx.cpu().numpy(), X.grad.numpy(), rtol=0, atol=2e-5 * (1 + float(X.grad.abs().max())))
    if bn:
        np.testing.assert_allclose(dgam.cpu().numpy(), G.grad.numpy(), rtol=1e-4, atol=1e-4 * np.sqrt(M))
        np.testing.assert_allclose(dbet.cpu().numpy(), Bt.grad.numpy(), rtol=1e-4, atol=1e-4 * np.sqrt(M))
        np.testing.assert_allclose(rm.cpu().numpy(), rm_ref.numpy(), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(rv.cpu().numpy(), rv_ref.numpy(), rtol=1e-5, atol=1e-6)
        assert int(nbt) == 1


def test_bn_with_one_row_is_rejected():
    from jorldy_b200._lib import JbError
    C, ptr, sp = _C()
    t = torch.zeros(1 << 12, device=DEV)
    nbt = torch.zeros((), dtype=torch.int64, device=DEV)
    part = torch.zeros(4096, dtype=torch.float64, device=DEV)
    p = ptr(t)
    with pytest.raises(JbError):
        C.jb_bn_elu_fwd(p, 1, 256, p, p, p, p, ptr(nbt), 0.1, 1e-5, p, p, ptr(part), p, 256, 0, 0, sp())
    with pytest.raises(JbError):
        C.jb_bn_elu_bwd(p, 256, p, 256, p, 1, 256, p, p, p, p, ptr(part), p, p, p, sp())
    C.jb_bn_elu_fwd(p, 1, 256, 0, 0, 0, 0, 0, 0.0, 0.0, 0, 0, 0, p, 256, 0, 0, sp())        # ELU alone takes one row
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------- 3. running statistics
def test_statistics_kernels_match_numpy_over_two_learns():
    C, ptr, sp = _C()
    from jorldy_b200.core.agent.icm_ppo import _RunningMeanStd
    rs = np.random.RandomState(5)
    N, T, D = 16, 33, 11
    obs = _RunningMeanStd((D,), DEV)
    ri_rms = _RunningMeanStd((1,), DEV)
    rewems = torch.zeros(N, device=DEV)
    ref_obs, ref_ri, ref_e = oi.RunningMeanStd((D,)), oi.RunningMeanStd(()), np.zeros(N)
    for learn in range(2):
        x = (rs.standard_normal((N * T, D)) * 3 + learn).astype(np.float32)
        tx = torch.from_numpy(x).to(DEV)
        part = torch.empty(C.jb_col_partials_doubles(N * T, D), dtype=torch.float64, device=DEV)
        C.jb_rms_update(ptr(tx), N * T, D, *(ptr(t) for t in obs.tensors()), ptr(part), sp())
        ref_obs.update(x)
        idx = rs.permutation(N * T)[:100].astype(np.int32)
        tidx = torch.from_numpy(idx).to(DEV)
        y = torch.empty(100, D, device=DEV)
        C.jb_rms_normalize(ptr(tx), ptr(tidx), 100, D, ptr(obs.mean), ptr(obs.var), 5.0, ptr(y), sp())
        ri = rs.uniform(0, 0.1, N * T).astype(np.float32)
        r = rs.standard_normal(N * T).astype(np.float32)
        tr, tri = torch.from_numpy(r).to(DEV), torch.from_numpy(ri).to(DEV)
        out = torch.empty(N * T, device=DEV)
        filt = torch.empty(N * T, device=DEV)
        part1 = torch.empty(C.jb_col_partials_doubles(N * T, 1), dtype=torch.float64, device=DEV)
        C.jb_icm_reward(ptr(tr), ptr(tri), N, T, 0.99, 1, ptr(rewems),
                        *(ptr(t) for t in ri_rms.tensors()), ptr(part1), ptr(filt), 0.5, 2.0, ptr(out), sp())
        torch.cuda.synchronize()
        f_ref, ref_e = oi.reward_filter(ref_e, ri.astype(np.float64).reshape(N, T), 0.99)
        ref_ri.update(f_ref.reshape(-1))
        np.testing.assert_allclose(obs.mean.cpu().numpy(), ref_obs.mean, rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(obs.var.cpu().numpy(), ref_obs.var, rtol=1e-10)
        assert float(obs.count) == pytest.approx(ref_obs.count, rel=1e-15)
        yref = np.clip((x[idx] - ref_obs.mean) / np.sqrt(ref_obs.var), -5, 5)
        np.testing.assert_allclose(y.cpu().numpy(), yref, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(filt.cpu().numpy(), f_ref.reshape(-1), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(rewems.cpu().numpy(), ref_e, rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(float(ri_rms.mean), float(ref_ri.mean), rtol=1e-5)
        np.testing.assert_allclose(float(ri_rms.var), float(ref_ri.var), rtol=1e-4)
        mix = 0.5 * r + 2.0 * ri / (np.sqrt(ref_ri.var) + 1e-7)
        np.testing.assert_allclose(out.cpu().numpy(), mix, rtol=1e-4, atol=1e-6)


# ------------------------------------------------------------------------------------------ 4. rollout next_state
def test_rollout_next_state_holds_the_terminal_observation_at_done_steps():
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import RolloutCollector
    env = Env("cartpole", num_envs=64, seed=3)
    agent = Agent("icm_ppo", state_size=4, action_size=2, hidden_size=64, batch_size=64, n_step=64, n_epoch=1,
                  device=DEV, run_step=1000)
    col = RolloutCollector(env, agent, use_cuda_graph=False)
    seen = []
    step = env.step_device

    def recording_step(action):
        out = step(action)
        seen.append(out[0].clone())
        return out
    env.step_device = recording_step
    ro = col.collect()
    torch.cuda.synchronize()
    done = ro.done.bool()
    assert done.any()
    for t in range(ro.T):
        assert torch.equal(ro.next_state[:, t], seen[t])
        if t + 1 < ro.T:
            keep = ~done[:, t]
            assert torch.equal(ro.next_state[keep, t], ro.state[keep, t + 1])
    assert torch.equal(ro.last_next_state, seen[-1])
    ppo = Agent("ppo", state_size=4, action_size=2, hidden_size=64, batch_size=64, n_step=16, device=DEV, run_step=1000)
    assert RolloutCollector(Env("cartpole", num_envs=8, seed=0), ppo, use_cuda_graph=False).rollout.next_state is None


def test_frame_rollout_next_ref_names_the_terminal_stack_at_done_steps():
    """Atari frames (256 lanes, T = 8, seed 0 ends episodes inside the rollout): every step's next_ref gathers back to the
    env's next observation bit for bit, the terminal stack at done steps included, and PPO's frame rollout keeps none."""
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import RolloutCollector
    N, T = 256, 8
    env = Env("breakout", num_envs=N, seed=0, device=DEV)
    agent = Agent("icm_ppo", state_size=[4, 84, 84], action_size=env.action_size, hidden_size=64, head="cnn",
                  icm_network="icm_cnn", obs_normalize=False, batch_size=64, n_step=T, n_epoch=1, device=DEV, run_step=1000)
    col = RolloutCollector(env, agent, use_cuda_graph=False)
    seen = []
    step = env.step_device

    def recording_step(action):
        out = step(action)
        seen.append(out[0].clone())
        return out
    env.step_device = recording_step
    ro = col.collect()
    refs = ro.next_ref.reshape(-1)
    got, _ = ro.frames.gather(refs, refs)
    ro.frames.check()
    assert ro.done.bool().any()
    assert torch.equal(got.view(N, T, 4, 84, 84), torch.stack(seen, 1))
    assert torch.equal(ro.next_ref[:, -1], ro.last_next_state)
    ppo = Agent("ppo", state_size=[4, 84, 84], action_size=env.action_size, hidden_size=64, head="cnn", n_step=T,
                batch_size=64, device=DEV, run_step=1000)
    assert RolloutCollector(Env("breakout", num_envs=8, seed=0, device=DEV), ppo, use_cuda_graph=False).rollout.next_ref is None


# ------------------------------------------------------------------------------------------------- 5. learn
CASES = {
    "cartpole_h64": dict(seed=31, N=4, T=32, D=4, A=2, H=64, continuous=False, batch_size=32, n_epoch=2, lr=2.5e-4),
    "cartpole_h512": dict(seed=32, N=8, T=64, D=4, A=2, H=512, continuous=False, batch_size=256, n_epoch=2, lr=2.5e-4),
    "hopper": dict(seed=33, N=4, T=64, D=11, A=3, H=256, continuous=True, batch_size=64, n_epoch=2, lr=3e-4),
}
ICM_KW = dict(beta=0.2, lamb=0.5, eta=0.01, extrinsic_coeff=1.0, intrinsic_coeff=1.0, obs_normalize=True,
              ri_normalize=True, batch_norm=True)


def _agent(case, **kw):
    from jorldy_b200.core import Agent
    net = "continuous_policy_value" if case["continuous"] else "discrete_policy_value"
    args = dict(ICM_KW, **kw)
    return Agent("icm_ppo", state_size=case["D"], action_size=case["A"], hidden_size=case["H"], network=net,
                 optim_config={"name": "adam", "lr": case["lr"]}, gamma=0.99, use_standardization=True, run_step=1000,
                 lr_decay=False, device=DEV, batch_size=case["batch_size"], n_step=case["T"], n_epoch=case["n_epoch"],
                 _lambda=0.95, clip_grad_norm=1.0, epsilon_clip=0.1, vf_coef=1.0, ent_coef=0.01, **args)


def _batch(case, learn=0):
    rs = np.random.RandomState(case["seed"] + 1000 * learn)
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
            "standardize": True, "batch_size": case["batch_size"], "n_epoch": case["n_epoch"], "clip_grad_norm": 1.0,
            "eps_clip": 0.1, "vf_coef": 1.0, "ent_coef": 0.01}


@pytest.mark.parametrize("name", list(CASES))
def test_two_eager_learns_match_the_float64_oracle(name):
    case = CASES[name]
    agent = _agent(case, use_cuda_graph=False)
    params = {k: v.detach().cpu().clone() for k, v in agent.network.p.items()}
    icm = {k: v.detach().cpu().clone() for k, v in agent.icm.p.items()}
    bufs = {k: v.detach().cpu().clone() for k, v in agent.icm.buffers.items()}
    ss = oi.new_state(case["D"], case["N"])
    opt_state = None
    for learn in range(2):
        batch, perms = _batch(case, learn)
        res = _learn(agent, case, batch, perms)
        ref = oi.learn(params, icm, bufs, batch, _hp(case), ICM_KW, perms, case["lr"], ss, opt_state=opt_state)
        params, icm, bufs, opt_state = ref["params"], ref["icm"], ref["buffers"], ref["opt_state"]
        for k, v in ref["params"].items():
            np.testing.assert_allclose(agent.network.p[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)
        # BatchNorm cancels fc1's bias: its float64 gradient is 0 and the fp32 one is round-off, which Adam turns into steps
        # of up to ~lr.  fc1.bias, and the running means that carry it, are held to that bound: lr per step taken so far.
        drift = case["lr"] * (learn + 1) * case["n_epoch"] * -(-case["N"] * case["T"] // case["batch_size"])
        for k, v in ref["icm"].items():
            atol = drift if k == "fc1.bias" else 0.1 * case["lr"]
            np.testing.assert_allclose(agent.icm.p[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=atol, err_msg=k)
        for k, v in ref["buffers"].items():
            got = agent.icm.buffers[k].cpu()
            if v.dtype == torch.int64:
                assert int(got) == int(v), k
            else:
                atol = drift if k.endswith("running_mean") else 1e-5
                np.testing.assert_allclose(got.numpy(), v.numpy(), rtol=1e-4, atol=atol, err_msg=k)
        for k, v in ref["result"].items():
            np.testing.assert_allclose(res[k], v, rtol=2e-4, atol=2e-4, err_msg=k)
        np.testing.assert_allclose(agent.rms_obs.mean.cpu().numpy(), ss["rms_obs"].mean, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(agent.rms_obs.var.cpu().numpy(), ss["rms_obs"].var, rtol=1e-9)
        np.testing.assert_allclose(float(agent.rms_ri.var), float(ss["rms_ri"].var), rtol=1e-3)
        np.testing.assert_allclose(agent.rewems.cpu().numpy(), ss["rewems"], rtol=1e-3, atol=1e-7)
        st = opt_state["state"]
        P = len(agent.network.p)
        for opt, names, off in ((agent.optimizer, list(agent.network.p), 0), (agent.icm_optimizer, list(agent.icm.p), P)):
            m, v = opt._slot_views(opt.exp_avg), opt._slot_views(opt.exp_avg_sq)
            for i, k in enumerate(names):
                if k == "fc1.bias" and opt is agent.icm_optimizer:
                    continue        # BatchNorm cancels fc1's bias: its gradient is 0 in float64 and fp32 round-off here
                for got, key in ((m[i], "exp_avg"), (v[i], "exp_avg_sq")):
                    r = st[off + i][key].numpy()
                    np.testing.assert_allclose(got.cpu().numpy(), r, rtol=5e-3, atol=1e-3 * np.abs(r).max() + 1e-12,
                                               err_msg=f"{key} {k}")


def test_eager_learn_on_atari_frames_with_the_cnn_icm_matches_the_float64_oracle():
    """A = 18, the CNN head and the CNN ICM on uint8 frame stacks, one epoch of 2 Adam steps.  A ReLU input within fp32
    round-off of 0 can take the other side in float64, so parameters are compared normwise against the update."""
    from jorldy_b200.core import Agent
    N, T, B, A, lr = 4, 8, 16, 18, 2.5e-4
    case = dict(continuous=False, A=A, T=T, batch_size=B, n_epoch=1)
    ikw = dict(ICM_KW, obs_normalize=False)
    agent = Agent("icm_ppo", state_size=[4, 84, 84], action_size=A, hidden_size=64, network="discrete_policy_value",
                  head="cnn", icm_network="icm_cnn", optim_config={"name": "adam", "lr": lr}, run_step=1000,
                  lr_decay=False, device=DEV, batch_size=B, n_step=T, n_epoch=1, use_cuda_graph=False, **ikw)
    rs = np.random.RandomState(8)
    state = torch.from_numpy(rs.randint(0, 256, (N * T, 4, 84, 84)).astype(np.uint8))
    nxt = torch.from_numpy(rs.randint(0, 256, (N * T, 4, 84, 84)).astype(np.uint8))
    action = torch.from_numpy(rs.randint(0, A, (N * T, 1)).astype(np.float32))
    reward = torch.from_numpy(rs.standard_normal((N * T, 1)).astype(np.float32))
    done = torch.from_numpy((rs.uniform(size=(N * T, 1)) < 0.1).astype(np.float32))
    perms = [rs.permutation(N * T)]
    params = {k: v.detach().cpu().clone() for k, v in agent.network.p.items()}
    icm = {k: v.detach().cpu().clone() for k, v in agent.icm.p.items()}
    bufs = {k: v.detach().cpu().clone() for k, v in agent.icm.buffers.items()}
    agent._inject_perms = perms
    res = agent._learn_tensors(state.to(DEV), action.reshape(-1).to(torch.int32).to(DEV), reward.reshape(-1).to(DEV),
                               done.reshape(-1).to(DEV), next_state=nxt.to(DEV))
    torch.cuda.synchronize()
    batch = dict(state=state.double(), next_state=nxt.double(), action=action, reward=reward, done=done)
    ref = oi.learn(params, icm, bufs, batch, _hp(case), ikw, perms, lr, oi.new_state(1, N))
    # Below the ICM's BatchNorm the gradient reaching fc1's input sums to 0 over each half's rows, so the trunk's bias
    # gradients are what the ReLU masks leave of a cancelling sum, and fc1's bias gets only round-off (see the MLP learns):
    # those are held to 5e-2 of their update, fc1.bias is skipped, everything else to 2e-2.
    for which, start, got_p, ref_p in (("network", params, agent.network.p, ref["params"]),
                                       ("icm", icm, agent.icm.p, ref["icm"])):
        for k, v in ref_p.items():
            if which == "icm" and k == "fc1.bias":
                continue
            tol = 5e-2 if which == "icm" and k.startswith("head.") and k.endswith(".bias") else 2e-2
            upd = (v - start[k].double()).norm().item()
            err = (got_p[k].cpu().double() - v).norm().item()
            assert err <= tol * upd + 1e-9, (which, k, err, upd)
    for k, v in ref["buffers"].items():
        got = agent.icm.buffers[k].cpu()
        if v.dtype == torch.int64:
            assert int(got) == int(v), k
        elif k.endswith("running_var"):
            np.testing.assert_allclose(got.numpy(), v.numpy(), rtol=1e-3, atol=1e-5, err_msg=k)
    for k, v in ref["result"].items():
        np.testing.assert_allclose(res[k], v, rtol=1e-3, atol=1e-3, err_msg=k)


def test_graph_learn_is_bit_identical_to_eager_and_reproducible(monkeypatch):
    import jorldy_b200.core.agent.ppo as ppo_mod
    monkeypatch.setattr(ppo_mod, "GRAPH_CHUNK", 2)
    case = dict(CASES["cartpole_h64"], N=8, T=40, batch_size=24)          # 13 full minibatches + a tail of 8
    agents = [_agent(case, use_cuda_graph=g) for g in (True, False, True)]
    for a in agents[1:]:
        a.network.load_state_dict(agents[0].network.state_dict())
        a.icm.load_state_dict(agents[0].icm.state_dict())
    results = []
    for a in agents:
        r = []
        for learn in range(2):
            batch, perms = _batch(case, learn)
            r.append(_learn(a, case, batch, perms))
        results.append(r)
    assert agents[0]._graphs and not agents[1]._graphs
    state = lambda g: [g.network.flat, g.icm.flat, *g.icm.buffer_tensors(), *g.optimizer.state_tensors(),
                       *g.icm_optimizer.state_tensors(), g._acc, g._icm_acc, *g.rms_obs.tensors(), *g.rms_ri.tensors(),
                       g.rewems]
    for a, r in zip(agents[1:], results[1:]):
        assert r == results[0]
        for x, y in zip(state(a), state(agents[0])):
            assert torch.equal(x, y)


def test_the_persistent_ppo_kernel_is_never_used():
    case = CASES["cartpole_h64"]
    from jorldy_b200.core.agent import ppo_fused
    agent = _agent(case, use_fused=True)
    assert agent.use_fused is False and ppo_fused.supported(agent, case["batch_size"])
    batch, perms = _batch(case)
    _learn(agent, case, batch, perms)
    assert agent._fused == {}


def test_learn_with_lamb_one_and_no_normalisation_or_batch_norm():
    case = CASES["cartpole_h64"]
    kw = dict(lamb=1.0, obs_normalize=False, ri_normalize=False, batch_norm=False)
    agent = _agent(case, use_cuda_graph=False, **kw)
    assert not agent.icm.buffers and "bn1.weight" not in agent.icm.p
    params = {k: v.detach().cpu().clone() for k, v in agent.network.p.items()}
    icm = {k: v.detach().cpu().clone() for k, v in agent.icm.p.items()}
    batch, perms = _batch(case)
    res = _learn(agent, case, batch, perms)
    ref = oi.learn(params, icm, {}, batch, _hp(case), dict(ICM_KW, **kw), perms, case["lr"], oi.new_state(4, case["N"]))
    for k, v in list(ref["params"].items()) + [("icm." + k, v) for k, v in ref["icm"].items()]:
        got = agent.icm.p[k[4:]] if k.startswith("icm.") else agent.network.p[k]
        np.testing.assert_allclose(got.cpu().numpy(), v.numpy(), rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)
    for k, v in ref["result"].items():
        np.testing.assert_allclose(res[k], v, rtol=2e-4, atol=2e-4, err_msg=k)


# ------------------------------------------------------------------------------------------ 6. checkpoint, attach
def test_checkpoint_round_trip_and_layout(tmp_path):
    case = CASES["hopper"]
    a = _agent(case, use_cuda_graph=False)
    batch, perms = _batch(case)
    _learn(a, case, batch, perms)
    a.save(str(tmp_path))
    ck = torch.load(str(tmp_path / "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "icm", "optimizer"}
    P, Q = len(a.network.p), len(a.icm.p)
    assert ck["optimizer"]["param_groups"][0]["params"] == list(range(P + Q))
    assert sorted(ck["optimizer"]["state"]) == list(range(P + Q))
    assert "bn1.running_var" in ck["icm"] and "bn1_next.num_batches_tracked" in ck["icm"]
    b = _agent(case, seed=9)
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, a.network.flat) and torch.equal(b.icm.flat, a.icm.flat)
    for x, y in zip(b.icm.buffer_tensors() + b.optimizer.state_tensors() + b.icm_optimizer.state_tensors(),
                    a.icm.buffer_tensors() + a.optimizer.state_tensors() + a.icm_optimizer.state_tensors()):
        assert torch.equal(x, y)


def test_attach_keeps_icm_ppo_a_replica():
    from jorldy_b200.core import parallel
    a = _agent(CASES["cartpole_h64"])
    with pytest.warns(UserWarning, match="replicas only .*ICM-PPO"):
        parallel.attach(a, 2)
    assert a.world_size == 1 and a.allreduce is None


# -------------------------------------------------------------------------------------------------- 7. end to end
@pytest.mark.parametrize("config,extra", [
    ("config.icm_ppo.cartpole", ["--train.num_workers", "8", "--agent.n_step", "32"]),
    ("config.icm_ppo.mujoco", ["--env.name", "hopper", "--train.num_workers", "16", "--agent.n_step", "32",
                               "--agent.batch_size", "64", "--agent.hidden_size", "64", "--train.update_period", "32",
                               "--train.distributed_batch_size", "64"]),
    ("config.icm_ppo.atari", ["--env.name", "seaquest", "--train.num_workers", "16", "--agent.n_step", "32",
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
    assert {"network", "icm", "optimizer"} == set(saved)
