"""CUDA-vs-oracle parity for the PPO path (run on the GPU: pytest -m gpu).

Tolerances (fp32, stated per output; the CUDA kernels accumulate in fp32 FFMA with a different
summation order from torch-CPU):
  value / log_prob_old / adv / ret : rtol 1e-4, atol 2e-5      (forward + scan)
  unstandardised adv / ret given identical value inputs (test_gae_*) : BIT-EXACT
  first-minibatch gradients        : rtol 2e-3, atol 2e-6
  parameters after the whole learn(): atol 0.1*lr (Adam normalises the update to ~lr, so a
                                      relative gradient error e moves a parameter by ~lr*e)
  result dict (losses, ratios)     : rtol/atol 2e-4
"""
import numpy as np
import pytest
import torch

import gen_inputs as G
from helpers import check_against_golden, load_golden, ppo_oracle_inputs
from oracle import ppo as oppo

pytestmark = pytest.mark.gpu


def _make_agent(case, **kw):
    from jorldy_b200.core import Agent
    net = "continuous_policy_value" if case["continuous"] else "discrete_policy_value"
    agent = Agent("ppo", state_size=case["D"], action_size=case["A"], hidden_size=case["H"], network=net,
                  optim_config={"name": "adam", "lr": case["lr"]}, gamma=case["gamma"],
                  use_standardization=case["standardize"], run_step=1000, lr_decay=False, device="cuda",
                  batch_size=case["batch_size"], n_step=case["T"], n_epoch=case["n_epoch"], _lambda=case["lam"],
                  epsilon_clip=case["eps_clip"], vf_coef=case["vf_coef"], ent_coef=case["ent_coef"],
                  clip_grad_norm=case["clip_grad_norm"], **kw)
    return agent


def _run_cuda(case, use_graph, use_fused=False):
    params, batch, hp, perms = ppo_oracle_inputs(case)
    agent = _make_agent(case, use_cuda_graph=use_graph, use_fused=use_fused)
    agent.network.load_state_dict(params)
    agent._inject_perms = perms
    dev = "cuda"
    action = batch["action"].to(dev)
    action = action if case["continuous"] else action.reshape(-1).to(torch.int32)
    res = agent._learn_tensors(batch["state"].to(dev), action, batch["reward"].reshape(-1).to(dev),
                               batch["done"].reshape(-1).to(dev), next_state=batch["next_state"].to(dev))
    torch.cuda.synchronize()
    return agent, res, (params, batch, hp, perms)


@pytest.mark.parametrize("name", list(G.PPO_CASES.keys()))
@pytest.mark.parametrize("use_graph", [False, True])
def test_ppo_learn_matches_reference_golden(name, use_graph, monkeypatch):
    if use_graph:
        import jorldy_b200.core.agent.ppo as ppo_mod
        monkeypatch.setattr(ppo_mod, "GRAPH_CHUNK", 2)
    case = G.PPO_CASES[name]
    agent, res, _ = _run_cuda(case, use_graph)
    gold = load_golden(name)
    st = agent._st
    pre = {"value": st["value"].cpu().numpy(), "adv": st["adv"].cpu().numpy(), "ret": st["ret"].cpu().numpy(),
           "log_prob_old": st["logp_old"].cpu().numpy(), "next_value": st["next_value"].cpu().numpy()}
    params_after = {k: v.cpu().numpy() for k, v in agent.network.state_dict().items()}
    check_against_golden(gold, params_after, res, pre, rtol=1e-4, atol=0.1 * case["lr"], stat_tol=2e-4)


# "tcgen05" is the tensor-core engine's long-standing test id, kept so that test ids stay stable; the engine it selects is
# the wgmma instantiation
@pytest.fixture(params=["ffma", "wgmma"], ids=["ffma", "tcgen05"])
def tile_engine(request, monkeypatch):
    """Both instantiations of the persistent kernel: fp32 FFMA tiles (default) and the 3xTF32 wgmma tiles (JB_FUSED_TC=1,
    taken when B % 128 == 0 and H % 128 == 0, else the launcher keeps the FFMA tiles)."""
    monkeypatch.setenv("JB_FUSED_TC", "1" if request.param == "wgmma" else "0")
    return request.param


@pytest.mark.parametrize("name", list(G.PPO_CASES.keys()))
def test_ppo_fused_kernel_matches_reference_golden(name, tile_engine):
    """Persistent cooperative minibatch-loop kernel (csrc/ppo_fused.cu) against the same goldens."""
    case = G.PPO_CASES[name]
    if case["batch_size"] % 32:
        pytest.skip("fused kernel needs B % 32 == 0 (host falls back to the multi-launch path)")
    if tile_engine == "wgmma" and (case["batch_size"] % 128 or case["H"] % 128):
        pytest.skip("tensor-core tiles need B % 128 == 0 and H % 128 == 0")
    agent, res, _ = _run_cuda(case, False, use_fused=True)
    assert agent._fused, "fused path was not taken"
    gold = load_golden(name)
    params_after = {k: v.cpu().numpy() for k, v in agent.network.state_dict().items()}
    check_against_golden(gold, params_after, res, None, rtol=1e-4, atol=0.1 * case["lr"], stat_tol=2e-4)


def test_ppo_fused_equals_multilaunch_path(tile_engine):
    """Same inputs through the fused kernel and the 13-launch path: parameters agree to fp32 round-off
    (the two paths share the row math and the Adam formula; only summation orders differ)."""
    case = G.PPO_CASES["ppo_discrete_h512"]
    a1, r1, _ = _run_cuda(case, False, use_fused=True)
    a2, r2, _ = _run_cuda(case, False, use_fused=False)
    for k in a1.network.p:
        np.testing.assert_allclose(a1.network.p[k].cpu().numpy(), a2.network.p[k].cpu().numpy(), rtol=1e-4,
                                   atol=0.02 * case["lr"], err_msg=k)
    for k in r1:
        np.testing.assert_allclose(r1[k], r2[k], rtol=1e-4, atol=1e-5, err_msg=k)


# shapes that exercise the generic paths of the persistent kernel the golden cases do not reach
_FUSED_SHAPES = {
    # B > 256: panels in 256-row chunks, JA pairs not shared; 256 forward tiles > 132 CTAs: several tiles per CTA
    "b512_h512": dict(seed=21, N=16, T=128, D=4, A=2, H=512, continuous=False, batch_size=512, n_epoch=1),
    # odd number of column tiles (H/32 = 3): the last dW2 pair has one member; tiny grid of jobs
    "b64_h96_cont": dict(seed=22, N=4, T=64, D=3, A=1, H=96, continuous=True, batch_size=64, n_epoch=2),
    # D = 16 (widest input the kernel takes), A = 7 (nout = 8: both head-output quads)
    "b128_h256_d16_a7": dict(seed=23, N=8, T=64, D=16, A=7, H=256, continuous=False, batch_size=128, n_epoch=1),
    # ragged tail: 1000 rows = 3 x 256 + 232 -> the tail minibatch takes the multi-launch path after the fused launch
    "b256_tail": dict(seed=24, N=8, T=125, D=4, A=2, H=128, continuous=False, batch_size=256, n_epoch=2),
}


@pytest.mark.parametrize("name", list(_FUSED_SHAPES.keys()))
def test_ppo_fused_generic_shapes_equal_multilaunch(name, tile_engine):
    case = dict(lr=2.5e-4, gamma=0.99, lam=0.95, eps_clip=0.1, vf_coef=1.0, ent_coef=0.01, clip_grad_norm=1.0,
                standardize=True, **_FUSED_SHAPES[name])
    a1, r1, _ = _run_cuda(case, False, use_fused=True)
    assert a1._fused, "fused path was not taken"
    a2, r2, _ = _run_cuda(case, False, use_fused=False)
    assert not a2._fused
    for k in a1.network.p:
        np.testing.assert_allclose(a1.network.p[k].cpu().numpy(), a2.network.p[k].cpu().numpy(), rtol=1e-4,
                                   atol=0.02 * case["lr"], err_msg=k)
    for k in r1:
        np.testing.assert_allclose(r1[k], r2[k], rtol=2e-4, atol=2e-5, err_msg=k)


def test_rebind_grad_keeps_both_paths_working():
    """parallel.attach() moves the flat gradient into a peer-mapped buffer (network.rebind_grad): every backward kernel
    must follow the rebuilt views (no cached pointers)."""
    case = G.PPO_CASES["ppo_discrete_h512"]
    outs = []
    for fused in (True, False):
        params, batch, hp, perms = ppo_oracle_inputs(case)
        agent = _make_agent(case, use_cuda_graph=False, use_fused=fused)
        agent.network.load_state_dict(params)
        new = torch.full((agent.network.num_flat + 256,), 7.0, device="cuda")
        old_ptr = agent.network.grad.data_ptr()
        agent.network.rebind_grad(new)
        assert agent.network.grad.data_ptr() == new.data_ptr() != old_ptr
        agent._inject_perms = perms
        res = agent._learn_tensors(batch["state"].cuda(), batch["action"].reshape(-1).to(torch.int32).cuda(),
                                   batch["reward"].reshape(-1).cuda(), batch["done"].reshape(-1).cuda(),
                                   next_state=batch["next_state"].cuda())
        torch.cuda.synchronize()
        assert torch.all(new[agent.network.num_flat:] == 7.0), "wrote past the gradient region"
        assert float(new[:agent.network.num_flat].abs().sum()) > 0, "gradients did not land in the new buffer"
        gold = load_golden("ppo_discrete_h512")
        params_after = {k: v.cpu().numpy() for k, v in agent.network.state_dict().items()}
        check_against_golden(gold, params_after, res, None, rtol=1e-4, atol=0.1 * case["lr"], stat_tol=2e-4)


def test_ppo_fused_is_bit_reproducible(tile_engine):
    """Static job maps + fixed-order reductions: two runs give identical bits."""
    case = G.PPO_CASES["ppo_discrete_h512"]
    a1, _, _ = _run_cuda(case, False, use_fused=True)
    a2, _, _ = _run_cuda(case, False, use_fused=True)
    assert torch.equal(a1.network.flat, a2.network.flat)


@pytest.mark.parametrize("name", ["ppo_discrete_small", "ppo_continuous_small", "ppo_discrete_h512"])
def test_ppo_first_minibatch_grads_match_oracle(name):
    case = dict(G.PPO_CASES[name])
    params, batch, hp, perms = ppo_oracle_inputs(case)
    ref = oppo.learn(params, batch, hp, perms, lr=case["lr"], max_minibatches=1)
    case1 = dict(case, n_epoch=1)
    agent = _make_agent(case1, use_cuda_graph=False)
    agent.network.load_state_dict(params)
    # run the pre-pass + exactly one minibatch step by giving a 1-minibatch permutation
    B = case["batch_size"]
    dev = "cuda"
    action = batch["action"].to(dev)
    action = action if case["continuous"] else action.reshape(-1).to(torch.int32)
    agent.batch_size = B
    NT = batch["state"].shape[0]
    # shrink the epoch to one minibatch: perm = first B indices of the oracle's permutation, rest dropped
    agent._inject_perms = [np.concatenate([perms[0][:B], perms[0][:B]])[:NT] if NT <= 2 * B else perms[0]]
    # do the pre-pass by hand and a single step
    agent.n_epoch = 0
    agent._learn_tensors(batch["state"].to(dev), action, batch["reward"].reshape(-1).to(dev),
                         batch["done"].reshape(-1).to(dev), next_state=batch["next_state"].to(dev))
    idx = torch.as_tensor(np.asarray(perms[0][:B]), dtype=torch.int32, device=dev)
    agent._minibatch_step(agent._st, idx, B)
    torch.cuda.synchronize()
    for k, g in ref["first_grads"].items():
        got = agent.network.g[k].cpu().numpy()
        np.testing.assert_allclose(got, g.numpy(), rtol=2e-3, atol=2e-6, err_msg=k)


def test_gae_bit_exact():
    """Given identical value inputs the TD residual / scan / returns are bit-exact vs torch-CPU."""
    from jorldy_b200._lib import C
    rs = np.random.RandomState(3)
    for (N, T) in [(5, 7), (33, 128), (64, 200)]:
        reward = torch.from_numpy(rs.standard_normal((N * T, 1)).astype(np.float32))
        done = torch.from_numpy((rs.uniform(size=(N * T, 1)) < 0.1).astype(np.float32))
        value = torch.from_numpy(rs.standard_normal((N * T, 1)).astype(np.float32))
        next_value = torch.from_numpy(rs.standard_normal((N * T, 1)).astype(np.float32))
        adv_ref, ret_ref = oppo.gae(reward, done, value, next_value, T, 0.99, 0.95, False)
        adv_s, _ = oppo.gae(reward, done, value, next_value, T, 0.99, 0.95, True)
        d = lambda t: t.reshape(-1).cuda()
        adv = torch.empty(N * T, device="cuda"); ret = torch.empty(N * T, device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        r_, dn_, v_, nv_ = d(reward), d(done), d(value), d(next_value)
        C.jb_gae(r_.data_ptr(), dn_.data_ptr(), v_.data_ptr(), nv_.data_ptr(), 0, N, T,
                 0.99, 0.95, 0, adv.data_ptr(), ret.data_ptr(), s)
        torch.cuda.synchronize()
        assert np.array_equal(adv.cpu().numpy(), adv_ref.reshape(-1).numpy())
        assert np.array_equal(ret.cpu().numpy(), ret_ref.reshape(-1).numpy())
        C.jb_gae(r_.data_ptr(), dn_.data_ptr(), v_.data_ptr(), nv_.data_ptr(), 0, N, T, 0.99, 0.95, 1,
                 adv.data_ptr(), ret.data_ptr(), s)
        torch.cuda.synchronize()
        np.testing.assert_allclose(adv.cpu().numpy(), adv_s.reshape(-1).numpy(), rtol=2e-6, atol=2e-6)
        assert np.array_equal(ret.cpu().numpy(), ret_ref.reshape(-1).numpy())


def test_gae_value_shift_equals_next_value_path():
    """next_value=NULL + last_value reproduces the explicit next_value path whenever
    next_state[t] == state[t+1] on non-terminal steps (the resident rollout layout)."""
    from jorldy_b200._lib import C
    rs = np.random.RandomState(5)
    N, T = 40, 96
    value = rs.standard_normal((N, T)).astype(np.float32)
    last = rs.standard_normal(N).astype(np.float32)
    done = (rs.uniform(size=(N, T)) < 0.1).astype(np.float32)
    reward = rs.standard_normal((N, T)).astype(np.float32)
    nv = np.concatenate([value[:, 1:], last[:, None]], axis=1)
    nv = np.where(done > 0, rs.standard_normal((N, T)).astype(np.float32), nv)   # garbage where done
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    r, d, v, n, l = t(reward), t(done), t(value), t(nv), t(last)
    a1 = torch.empty(N * T, device="cuda"); r1 = torch.empty_like(a1); a2 = torch.empty_like(a1); r2 = torch.empty_like(a1)
    s = torch.cuda.current_stream().cuda_stream
    C.jb_gae(r.data_ptr(), d.data_ptr(), v.data_ptr(), n.data_ptr(), 0, N, T, 0.99, 0.95, 1, a1.data_ptr(), r1.data_ptr(), s)
    C.jb_gae(r.data_ptr(), d.data_ptr(), v.data_ptr(), 0, l.data_ptr(), N, T, 0.99, 0.95, 1, a2.data_ptr(), r2.data_ptr(), s)
    torch.cuda.synchronize()
    assert torch.equal(a1, a2) and torch.equal(r1, r2)
