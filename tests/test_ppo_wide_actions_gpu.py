"""PPO with 9 to 18 discrete actions (pytest -m gpu): the NA = 18 instantiation of the act, pre-pass and loss kernels
(csrc/ppo.cu, csrc/ppo_rowmath.cuh) that the 9- and 18-action Atari games need.

Tolerances follow test_ppo_gpu.py: value / log_prob_old rtol 1e-4 atol 2e-5; loss gradients and statistics rtol 1e-4
against float64 with an absolute floor of 1e-5 max|ref| (one fp32 row of at most 19 outputs, no long sums); after a
whole learn(), parameters atol 0.1 lr and the Adam moments normwise 1e-2 (gradients agree to ~2e-3, test_ppo_gpu.py).
A sampled action may differ from the float32 CPU oracle only where the uniform lands within rounding of a CDF step."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ppo_oracle_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _agent(A, D=8, H=64, **kw):
    from jorldy_b200.core import Agent
    return Agent("ppo", state_size=D, action_size=A, hidden_size=H, run_step=1000, lr_decay=False, device=DEV, **kw)


def _check_samples(got, ref, pi, u):
    """got == ref except where u * sum(pi) is within 1e-5 of the CDF step between them (fp32 rounding of pi)."""
    got, ref = np.asarray(got).reshape(-1), np.asarray(ref).reshape(-1)
    for m in np.nonzero(got != ref)[0]:
        cdf = np.cumsum(pi[m].astype(np.float64))
        step = cdf[min(got[m], ref[m])]
        assert abs(u[m] * cdf[-1] - step) < 1e-5, f"row {m}: kernel {got[m]}, oracle {ref[m]}"


# ------------------------------------------------------------------------------------------------------------- 1. act
@pytest.mark.parametrize("A", [9, 12, 18])
@pytest.mark.parametrize("M", [1, 1000])
def test_act_with_injected_uniforms_equals_oracle(A, M):
    from oracle import collect as ocol
    from oracle import nets as onets
    agent = _agent(A, seed=A)
    rs = np.random.RandomState(M + A)
    state = (2.0 * rs.standard_normal((M, 8))).astype(np.float32)
    u = rs.uniform(size=M).astype(np.float32)
    got = agent.act_device(torch.as_tensor(state, device=DEV), True, noise=torch.as_tensor(u, device=DEV)).cpu().numpy()
    params = {k: v.cpu() for k, v in agent.network.state_dict().items()}
    ref = ocol.act_ppo(params, state, False, training=True, u=u)
    with torch.no_grad():
        pi = onets.discrete_policy_value(params, torch.as_tensor(state))[0].numpy()
    assert got.min() >= 0 and got.max() < A
    _check_samples(got, ref, pi, u)
    greedy = agent.act_device(torch.as_tensor(state, device=DEV), False).cpu().numpy()
    rows = np.arange(M)
    assert np.all(pi[rows, greedy] >= pi[rows, pi.argmax(1)] * (1 - 1e-5))     # argmax up to fp32 near-ties


@pytest.mark.parametrize("A", [9, 12, 18])
@pytest.mark.parametrize("M", [1, 1000])
def test_greedy_is_argmax_lowest_index_on_ties(A, M):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(A * M)
    out = rs.standard_normal((M, A + 1)).astype(np.float32)
    for m in range(M):                                   # a tie for the maximum between two random actions
        i, j = sorted(rs.choice(A, 2, replace=False))
        out[m, i] = out[m, j] = out[m, :A].max() + 1.0
    out_d, act = torch.as_tensor(out, device=DEV), torch.empty(M, dtype=torch.int64, device=DEV)
    C.jb_ppo_act_discrete(ptr(out_d), M, A, A + 1, 0, 0, 0, 0, 0, 1, ptr(act), stream_ptr())
    assert np.array_equal(act.cpu().numpy(), out[:, :A].argmax(1))


def test_philox_law_chi_square():
    """10^5 draws from one fixed 18-logit row (one row per draw, distinct Philox streams) against softmax in float64."""
    from scipy.stats import chisquare
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    A, M = 18, 100000
    logits = np.linspace(-2.0, 1.5, A).astype(np.float32)
    out = torch.as_tensor(np.tile(np.append(logits, 0.0), (M, 1)).astype(np.float32), device=DEV)
    act = torch.empty(M, dtype=torch.int64, device=DEV)
    C.jb_ppo_act_discrete(ptr(out), M, A, A + 1, 0, 7, 0, 0, 0, 0, ptr(act), stream_ptr())
    counts = np.bincount(act.cpu().numpy(), minlength=A)
    p = np.exp(logits.astype(np.float64) - logits.max())
    p /= p.sum()
    assert chisquare(counts, M * p).pvalue > 1e-3, counts


def test_captured_graph_draws_fresh_actions_every_replay():
    agent = _agent(18, seed=3)
    M = 1000
    state = torch.randn(M, 8, device=DEV, generator=torch.Generator(DEV).manual_seed(0))
    agent.act_device(state)                              # allocates the buffers and the row counters
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        action = agent.act_device(state)
    draws = []
    for _ in range(3):
        g.replay()
        draws.append(action.clone())
    torch.cuda.synchronize()
    assert int(agent._row_ctr[M].min().item()) == int(agent._row_ctr[M].max().item()) == 4
    assert not torch.equal(draws[0], draws[1]) and not torch.equal(draws[1], draws[2])
    assert int(draws[0].max().item()) > 8


# -------------------------------------------------------------------------------------------------------- 2. pre-pass
@pytest.mark.parametrize("A", [9, 18])
def test_prepass_vs_float64(A):
    from oracle import ppo as oppo
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    agent = _agent(A, seed=A)
    net = agent.network
    M = 777
    rs = np.random.RandomState(A)
    state = torch.as_tensor((2.0 * rs.standard_normal((M, 8))).astype(np.float32))
    action = torch.as_tensor(rs.randint(0, A, M).astype(np.int32))
    out = torch.empty(M, net.nout, device=DEV)
    net.forward_rows(state.to(DEV), out)
    value, logp = torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    C.jb_ppo_prepass_discrete(ptr(out), ptr(action.to(DEV)), M, A, net.nout, ptr(value), ptr(logp), stream_ptr())
    p64 = {k: v.cpu().double() for k, v in net.state_dict().items()}
    rv, _, rl = oppo.prepass(p64, state.double(), action.view(-1, 1).double(), state.double(), False)
    np.testing.assert_allclose(value.cpu().numpy(), rv.view(-1).numpy(), rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(logp.cpu().numpy(), rl.view(-1).numpy(), rtol=1e-4, atol=2e-5)


# ------------------------------------------------------------------------------------------------------------ 3. loss
def _loss_case(A, B, seed):
    """Head outputs of B minibatch rows and full-rollout arrays of NT = B + 37 rows gathered through a shuffled idx.
    Row 0 has one dominant logit (the other 17 probabilities sit below float32 eps, so the clamp's mask is active);
    log_prob_old spreads the ratios over both sides of the clip; the value deltas fall inside and outside eps_clip.
    B = 1 makes the two critic means tie exactly (v = v_old on its only row, so v_clip = v)."""
    rs = np.random.RandomState(seed)
    NT = B + 37
    out = rs.standard_normal((B, A + 1)).astype(np.float32)
    out[0, :A] = -4.0
    out[0, 0] = 30.0
    idx = rs.permutation(NT)[:B].astype(np.int32)
    action = rs.randint(0, A, NT).astype(np.int32)
    action[idx[0]] = 0
    logits = torch.as_tensor(out[:, :A]).double()
    lp = torch.log_softmax(logits, -1).gather(1, torch.as_tensor(action[idx]).long().view(-1, 1)).view(-1).numpy()
    logp_old = rs.standard_normal(NT).astype(np.float32)
    logp_old[idx] = (lp + rs.uniform(-0.4, 0.4, B)).astype(np.float32)
    adv = rs.standard_normal(NT).astype(np.float32)
    ret = rs.standard_normal(NT).astype(np.float32)
    vold = rs.standard_normal(NT).astype(np.float32)
    vold[idx] = out[:, A] + rs.uniform(-0.3, 0.3, B).astype(np.float32)
    if B == 1:
        vold[idx] = out[:, A]
    return out, idx, action, adv, ret, vold, logp_old


@pytest.mark.parametrize("A", [9, 18])
@pytest.mark.parametrize("B", [1, 255, 256, 257])
def test_loss_vs_float64_autograd(A, B, monkeypatch):
    from oracle import nets as onets
    from oracle import ppo as oppo
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    eps_clip, vf_coef, ent_coef = 0.1, 1.0, 0.01
    out, idx, action, adv, ret, vold, logp_old = _loss_case(A, B, 100 * A + B)
    dev = [torch.as_tensor(a, device=DEV) for a in (out, idx, action, adv, ret, vold, logp_old)]   # alive until synced
    dout = torch.empty(B, A + 1, device=DEV)
    stats = torch.zeros(8 + 4 * ((B + 255) // 256), device=DEV)
    C.jb_ppo_loss(0, *(ptr(t) for t in dev), B, A, A + 1, eps_clip, vf_coef, ent_coef, ptr(dout), ptr(stats), 0,
                  stream_ptr())
    torch.cuda.synchronize()

    # float64: the "state" is the head output itself, so d loss / d state is d loss / d out
    monkeypatch.setattr(onets, "discrete_policy_value", lambda p, x: (torch.softmax(x[:, :A], -1), x[:, A:]))
    x = torch.as_tensor(out).double().requires_grad_(True)
    col = lambda a: torch.as_tensor(a[idx]).double().view(-1, 1)
    loss, aux = oppo.minibatch_loss({}, x, col(action), col(vold), col(ret), col(adv), col(logp_old), False,
                                    eps_clip, vf_coef, ent_coef)
    loss.backward()
    ratio = torch.exp(torch.log_softmax(x[:, :A], -1).gather(1, col(action).long()) - col(logp_old)).detach()
    if B > 1:
        assert bool(((ratio < 1 - eps_clip) | (ratio > 1 + eps_clip)).any()) and bool(((ratio - 1).abs() < eps_clip).any())
    ref = x.grad.numpy()
    np.testing.assert_allclose(dout.cpu().numpy(), ref, rtol=1e-4, atol=1e-5 * np.abs(ref).max())
    got = stats[:5].cpu().numpy()
    want = np.array([aux[k].item() for k in ("actor_loss", "critic_loss", "entropy_loss", "max_ratio", "min_prob")])
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------- 4. bounds
def test_nineteen_actions_are_rejected():
    from jorldy_b200._lib import JbError
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    A, M = 19, 4
    out = torch.zeros(M, A + 1, device=DEV)
    act = torch.empty(M, dtype=torch.int64, device=DEV)
    a32 = torch.zeros(M, dtype=torch.int32, device=DEV)
    v = torch.empty(M, device=DEV)
    with pytest.raises(JbError):
        C.jb_ppo_act_discrete(ptr(out), M, A, A + 1, 0, 0, 0, 0, 0, 0, ptr(act), stream_ptr())
    with pytest.raises(JbError):
        C.jb_ppo_prepass_discrete(ptr(out), ptr(a32), M, A, A + 1, ptr(v), ptr(v), stream_ptr())
    with pytest.raises(JbError):
        C.jb_ppo_loss(0, ptr(out), 0, ptr(a32), ptr(v), ptr(v), ptr(v), ptr(v), M, A, A + 1, 0.1, 1.0, 0.01, ptr(out),
                      ptr(torch.zeros(16, device=DEV)), 0, stream_ptr())
    with pytest.raises(ValueError, match="18"):
        _agent(19)
    with pytest.raises(ValueError, match="8"):
        _agent(9, network="continuous_policy_value")


# ---------------------------------------------------------------------------------------------- 5. learn, MLP network
CASE18 = dict(seed=31, N=8, T=32, D=8, A=18, H=128, continuous=False, batch_size=16, n_epoch=2, lr=2.5e-4, gamma=0.99,
              lam=0.95, eps_clip=0.1, vf_coef=1.0, ent_coef=0.01, clip_grad_norm=1.0, standardize=True)


def _learn18(use_graph):
    c = CASE18
    params, batch, hp, perms = ppo_oracle_inputs(c)
    agent = _agent(c["A"], D=c["D"], H=c["H"], optim_config={"name": "adam", "lr": c["lr"]}, batch_size=c["batch_size"],
                   n_step=c["T"], n_epoch=c["n_epoch"], use_cuda_graph=use_graph)
    agent.network.load_state_dict(params)
    agent._inject_perms = perms
    res = agent._learn_tensors(batch["state"].to(DEV), batch["action"].reshape(-1).to(torch.int32).to(DEV),
                               batch["reward"].reshape(-1).to(DEV), batch["done"].reshape(-1).to(DEV),
                               next_state=batch["next_state"].to(DEV))
    torch.cuda.synchronize()
    return agent, res


def test_learn_18_actions_vs_float64_and_graph_equals_eager():
    """16 full minibatches per epoch: the graph path replays one captured chunk of 16 steps per epoch."""
    from oracle import ppo as oppo
    c = CASE18
    eager, res = _learn18(False)
    graph, res_g = _learn18(True)
    assert not eager._fused and not graph._fused and graph._graphs
    assert res == res_g
    assert torch.equal(eager.network.flat, graph.network.flat)
    assert all(torch.equal(x, y) for x, y in zip(eager.optimizer.state_tensors(), graph.optimizer.state_tensors()))

    params, batch, hp, perms = ppo_oracle_inputs(c)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        ref = oppo.learn({k: v.double() for k, v in params.items()}, {k: v.double() for k, v in batch.items()}, hp,
                         perms, lr=c["lr"])
    finally:
        torch.set_default_dtype(prev)
    for k, v in ref["result"].items():
        assert abs(res[k] - v) <= 2e-4 * max(1.0, abs(v)), (k, res[k], v)
    names = list(params)
    state = eager.optimizer.state_dict()["state"]
    for j, k in enumerate(eager.network.p):
        np.testing.assert_allclose(eager.network.p[k].cpu().numpy(), ref["params"][k].numpy(), rtol=1e-4,
                                   atol=0.1 * c["lr"], err_msg=k)
        r = ref["opt_state"]["state"][names.index(k)]
        for m in ("exp_avg", "exp_avg_sq"):
            err = (state[j][m].cpu().double() - r[m]).abs().max().item()
            assert err <= 1e-2 * r[m].abs().max().item(), (k, m, err)


# ---------------------------------------------------------------------------------------------- 6. learn, CNN network
def test_cnn_learn_on_seaquest_vs_float64(monkeypatch):
    """test_ppo_frames_gpu.py::test_learn_vs_float64 (one collect + learn_rollout against float64, every minibatch's
    gradients, the result dict, parameters and Adam state) with the agent and env of the 18-action `seaquest`."""
    import jorldy_b200.core as core
    import test_ppo_frames_gpu as tpf
    env_cls = core.Env
    monkeypatch.setattr(tpf, "_ppo", lambda T, B, H=64, n_epoch=3, seed=0, **kw: core.Agent(
        "ppo", state_size=[4, 84, 84], action_size=18, hidden_size=H, head="cnn", n_step=T, batch_size=B,
        n_epoch=n_epoch, optim_config={"name": "adam", "lr": 2.5e-4}, run_step=1000, lr_decay=False, device=DEV,
        seed=seed, **kw))
    monkeypatch.setattr(core, "Env", lambda name, **kw: env_cls("seaquest", **kw))
    with pytest.MonkeyPatch.context() as inner:
        tpf.test_learn_vs_float64(inner)


# ------------------------------------------------------------------------------------------------------ 7. end to end
def test_sync_training_run_on_seaquest(tmp_path):
    """`main --sync --config config.ppo.atari --env.name seaquest`: 16 envs, 512 steps, then the checkpoint loads into a
    fresh 18-action agent with an identical state_dict."""
    from jorldy_b200.core import Agent
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable, "-m", "jorldy_b200.main", "--sync", "--config", "config.ppo.atari", "--env.name", "seaquest",
           "--train.num_workers", "16", "--train.run_step", "512", "--train.print_period", "256",
           "--train.save_period", "512"]
    r = subprocess.run(cmd, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith("512 step |") for line in r.stdout.splitlines()), out[-4000:]
    ckpts = [os.path.join(d, "ckpt") for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    saved = torch.load(ckpts[0], map_location="cpu", weights_only=False)["network"]
    assert saved["pi.weight"].shape[0] == 18
    fresh = Agent("ppo", state_size=[4, 84, 84], action_size=18, network="discrete_policy_value", head="cnn", device=DEV,
                  run_step=512)
    fresh.load(os.path.dirname(ckpts[0]))
    got = fresh.network.state_dict()
    assert sorted(got) == sorted(saved)
    for k, v in saved.items():
        assert torch.equal(got[k].cpu(), v), k
