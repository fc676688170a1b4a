"""QR-DQN and IQN on the GPU (csrc/quantile.cu, core/network/iqn.py, core/agent/quantile.py) against the float64
oracle (oracle/quantile.py), float64 autograd, the stacked replay layout and the run loop (pytest -m gpu).

Tolerances.  u = 2^-24 is fp32's unit roundoff.
- Loss kernel (1).  A per-sample loss is a sum of N * N' <= 40000 non-negative terms, accumulated as N' sequential
  fp32 adds per predicted quantile and a fixed-order tree over the N quantiles: relative error <= (N' + 13) u ~ 1.3e-5.
  The targets y_j = r + ((1 - d) gamma) theta'_j carry 3 roundings (|dy| <= 3 u |y|), which moves each u_ij by the same
  amount and each rho_ij by at most |dy| (h is 1-Lipschitz, weights <= 1).  With |theta| <= 8 that is ~2e-6 per term,
  far below R = 1e-4 of the loss scale.  Each gradient element is -(1/(B N')) sum_j w clamp(u), |w clamp| <= 1, so its
  error is at most (N' u + 3 u |y|) / B: checked normwise at R = 1e-4 against the scale 1/B.  max_Q and a* come from
  means of <= 200 values (error <= 200 u * max|theta| ~ 1e-4 absolute at |theta| <= 8): max_Q is checked at 1e-5
  relative to max|theta|, and a* must equal the float64 argmax unless the two best means lie within 1e-4 of each other.
  A mutated kernel (tau and 1 - tau swapped, the target without (1 - d), a sum instead of a mean over N') moves the
  loss or gradient by O(0.1..1) of its scale.
- Embedding (2).  phi's pre-activation contracts 64 cosines (error <= 64 u sum|terms|), z = psi * phi and dpsi sums
  N <= 64 products: all at R = 1e-4 normwise.  dpre is compared where the float64 pre-activation is farther than 1e-5
  from 0 (nearer, fp32 may take the other ReLU branch; such elements are counted and must be rare), and dW_e / db_e
  against the float64 contraction of the kernel's OWN dpre over B*N <= 2048 rows, at 2e-4 normwise (B N u = 1.2e-4).
- One learn (3): the contractions run over <= 12800 terms (conv1's weight gradient at B = 32); normwise error grows
  like K u = 7.6e-4 at worst.  Gradients are checked normwise per tensor: 1e-3 (MLP), 2e-3 (CNN, outside the trunk),
  2e-2 for the conv trunk and, in IQN, sample_embed: both sum over ~10^5..10^6 ReLU pre-activations per pass, of which
  a few lie within fp32 rounding of 0 and take the other branch in float64 (one such term is ~1/sqrt(rows) of a
  typical element).  loss and max_Q at rtol 5e-4.  Post-step parameters are checked against a float64 Adam step on the
  kernel's OWN gradients (first step: p - lr g / (|g| + eps)), bound 1e-3 lr + 2 u |p|, because near |g| ~ eps a first
  Adam step turns rounding-level gradient differences into O(lr) parameter differences.
- Repeated learns (4), frames vs stacks (6) and checkpoints (7) are bit-exact.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import quantile as oq

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def _close(got, ref, R, what, scale=None):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = max(float(np.abs(ref).max()), 1e-30) if scale is None else scale
    err = float(np.abs(got - ref).max())
    assert err <= R * scale, f"{what}: max |err| {err:.3e} > {R} * {scale:.3e}"


def _dv(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


# ----------------------------------------------------------------------------------------- 1. loss kernel vs oracle
def _run_loss(layout, B, A, N, Np, d, seed):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(seed)
    th = (2.0 * rs.standard_normal((B, A, N))).clip(-8, 8).astype(np.float32)        # [B, A, N] logical
    tn = (2.0 * rs.standard_normal((B, A, Np))).clip(-8, 8).astype(np.float32)
    if layout == "qr":
        tau = oq.qr_tau(N).to(torch.float32).numpy()
        tau_g, tau_stride = _dv(tau), 0
        pred, nxt, sa, sq, tsa, tsq = th, tn, N, 1, Np, 1
        tau64 = torch.from_numpy(tau).to(torch.float64)
    else:
        tau = rs.uniform(size=(B, N)).astype(np.float32)
        tau_g, tau_stride = _dv(tau), N
        pred, nxt, sa, sq, tsa, tsq = th.transpose(0, 2, 1), tn.transpose(0, 2, 1), 1, A, 1, A
        tau64 = torch.from_numpy(tau).to(torch.float64)
    action = rs.randint(A, size=B).astype(np.int64)
    reward = rs.standard_normal(B).astype(np.float32)
    done = np.full(B, float(d), np.float32)
    g_pred, g_nxt = _dv(pred), _dv(nxt)
    dpred = torch.full(g_pred.shape, float("nan"), device=DEV)
    loss = torch.empty(B, device=DEV)
    a_star = torch.empty(B, dtype=torch.int32, device=DEV)
    stats = torch.full((4,), float("nan"), device=DEV)
    scratch = torch.empty(2 * B, device=DEV)
    g_a, g_r, g_d = _dv(action), _dv(reward), _dv(done)
    C.jb_quantile_loss(ptr(g_pred), sa, sq, ptr(g_nxt), tsa, tsq, ptr(tau_g), tau_stride, ptr(g_a), 0, ptr(g_r), ptr(g_d),
                       B, A, N, Np, 0.99, ptr(dpred), ptr(loss), ptr(a_star), ptr(stats), ptr(scratch), stream_ptr())
    torch.cuda.synchronize()
    dp = dpred.cpu().numpy()
    if layout == "iqn":
        dp = dp.transpose(0, 2, 1)
    return dict(th=th, tn=tn, tau64=tau64, action=action, reward=reward, done=done, dtheta=dp, loss=loss.cpu().numpy(),
                a_star=a_star.cpu().numpy(), stats=stats.cpu().numpy())


@pytest.mark.parametrize("layout", ["qr", "iqn"])
@pytest.mark.parametrize("N,Np", [(1, 1), (32, 32), (64, 8), (200, 200)])
@pytest.mark.parametrize("A", [2, 18])
@pytest.mark.parametrize("B", [1, 32, 257])
@pytest.mark.parametrize("d", [0, 1])
def test_loss_kernel_matches_the_oracle(layout, N, Np, A, B, d):
    o = _run_loss(layout, B, A, N, Np, d, seed=N * 7 + Np * 3 + A * 11 + B + d)
    h = lambda x: torch.from_numpy(np.asarray(x)).to(torch.float64)
    tn = h(o["tn"])
    means = tn.mean(2)
    ref_a = means.argmax(1).numpy()
    top2 = torch.topk(means, min(2, A), dim=1).values
    gap = (top2[:, 0] - top2[:, -1]).numpy() if A > 1 else np.full(B, np.inf)
    bad = (o["a_star"] != ref_a) & (gap > 1e-4)
    assert not bad.any(), f"a* differs at {np.nonzero(bad)[0][:8]}"
    # the loss and gradient given the kernel's a* (a near-tie above cannot cascade)
    sel = tn[torch.arange(B), torch.from_numpy(o["a_star"].astype(np.int64))]
    gamma = float(np.float32(0.99))
    y = h(o["reward"]).view(B, 1) + (1 - h(o["done"]).view(B, 1)) * gamma * sel
    a = torch.from_numpy(o["action"])
    theta = h(o["th"])[torch.arange(B), a]
    tau = o["tau64"]
    per = oq.per_sample_loss(theta, y, tau)
    _close(o["loss"], per.numpy(), 1e-4, "per-sample loss")
    _close(o["stats"][0], per.mean().item(), 1e-4, "loss", float(per.abs().max()))
    _close(o["stats"][1], h(o["th"]).mean(2).max().item(), 1e-5, "max_Q", float(np.abs(o["th"]).max()))
    want = torch.zeros(B, A, N, dtype=torch.float64)
    want[torch.arange(B), a] = oq.grad_closed(theta, y, tau)
    _close(o["dtheta"], want.numpy(), 1e-4, "dtheta", 1.0 / B)
    mask = np.ones((B, A), bool)
    mask[np.arange(B), o["action"]] = False
    assert np.all(o["dtheta"][mask] == 0.0)


def test_loss_kernel_rejects_out_of_range_shapes():
    from jorldy_b200._lib import JbError
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    B = 2
    for A, N, Np in ((2, 257, 8), (2, 8, 257), (19, 8, 8)):
        x = torch.zeros(B * A * max(N, Np), device=DEV)
        tau = torch.zeros(max(N, Np), device=DEV)
        a = torch.zeros(B, dtype=torch.int64, device=DEV)
        out = torch.zeros(B * A * max(N, Np), device=DEV)
        small = torch.zeros(8, device=DEV)
        with pytest.raises(JbError):
            C.jb_quantile_loss(ptr(x), N, 1, ptr(x), Np, 1, ptr(tau), 0, ptr(a), 0, ptr(small), ptr(small), B, A, N, Np, 0.99,
                               ptr(out), ptr(small), None, ptr(small), ptr(small), stream_ptr())


def test_quantile_mean_both_layouts():
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(0)
    M, A, N = 300, 18, 64
    x = rs.standard_normal((M, A, N)).astype(np.float32)
    q1, q2 = torch.empty(M, A, device=DEV), torch.empty(M, A, device=DEV)
    x1, x2 = _dv(x), _dv(x.transpose(0, 2, 1))
    C.jb_quantile_mean(ptr(x1), N, 1, M, A, N, ptr(q1), stream_ptr())
    C.jb_quantile_mean(ptr(x2), 1, A, M, A, N, ptr(q2), stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(q1, q2)
    _close(q1.cpu().numpy(), x.astype(np.float64).mean(2), 1e-5, "mean", float(np.abs(x).max()))


# ----------------------------------------------------------------------------------------------- 2. IQN embedding
@pytest.mark.parametrize("Dh", [64, 512, 3136])
@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("B", [1, 32])
def test_embedding_forward_and_backward_match_autograd(Dh, N, B):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    from jorldy_b200.core.network import layers as L
    rs = np.random.RandomState(Dh + N + B)
    E = 64
    tau = rs.uniform(size=(B, N)).astype(np.float32)
    W = (rs.standard_normal((Dh, E)) / 8).astype(np.float32)
    bias = (0.1 * rs.standard_normal(Dh)).astype(np.float32)
    psi_pre = rs.standard_normal((B, Dh)).astype(np.float32)
    psi = np.maximum(psi_pre, 0)
    dz = rs.standard_normal((B, N, Dh)).astype(np.float32)
    s = stream_ptr()
    g_tau, g_W, g_b, g_psi, g_dz = (_dv(v) for v in (tau, W, bias, psi, dz))
    c = torch.empty(B * N, E, device=DEV)
    phi = torch.empty(B * N, Dh, device=DEV)
    z = torch.empty(B * N, Dh, device=DEV)
    C.jb_iqn_cos(ptr(g_tau), B * N, E, ptr(c), s)
    L.linear_fwd(c, g_W, g_b, phi, relu=True)
    C.jb_iqn_mul_fwd(ptr(g_psi), ptr(phi), B, N, Dh, ptr(z), s)
    dpsi, dpre = torch.empty(B, Dh, device=DEV), torch.empty(B * N, Dh, device=DEV)
    C.jb_iqn_mul_bwd(ptr(g_dz), ptr(g_psi), ptr(phi), B, N, Dh, ptr(dpsi), ptr(dpre), s)
    dW, db = torch.empty(Dh, E, device=DEV), torch.empty(Dh, device=DEV)
    L.linear_bwd_dw(dpre, c, dW, db)
    torch.cuda.synchronize()
    h = lambda x: torch.from_numpy(np.asarray(x)).to(torch.float64)
    pp, W64, b64 = h(psi_pre).requires_grad_(True), h(W).requires_grad_(True), h(bias).requires_grad_(True)
    i = torch.arange(E, dtype=torch.float64)
    c64 = torch.cos(np.pi * i * h(tau).unsqueeze(-1))
    pre = torch.nn.functional.linear(c64, W64, b64)
    z64 = torch.relu(pp).unsqueeze(1) * torch.relu(pre)
    (z64 * h(dz)).sum().backward()
    _close(c.cpu().numpy(), c64.reshape(B * N, E).numpy(), 1e-5, "cos features", 1.0)
    _close(z.cpu().numpy(), z64.detach().reshape(B * N, Dh).numpy(), 1e-4, "z")
    _close(dpsi.cpu().numpy(), pp.grad.numpy(), 1e-4, "dpsi")
    dpre_ref = (h(dz) * torch.relu(pp).detach().unsqueeze(1) * (pre.detach() > 0)).reshape(B * N, Dh).numpy()
    near = np.abs(pre.detach().reshape(B * N, Dh).numpy()) < 1e-5
    assert near.sum() <= max(4, near.size // 10 ** 4)
    _close(np.where(near, 0, dpre.cpu().numpy()), np.where(near, 0, dpre_ref), 1e-4, "dpre")
    dpre64 = h(dpre.cpu().numpy())
    _close(dW.cpu().numpy(), (dpre64.T @ c64.reshape(B * N, E)).numpy(), 2e-4, "dW_e")
    _close(db.cpu().numpy(), dpre64.sum(0).numpy(), 2e-4, "db_e")
    if not near.any():                              # then the kernel's mask equals float64's: the full chain
        _close(dW.cpu().numpy(), W64.grad.numpy(), 2e-4, "dW_e (autograd)")
        _close(db.cpu().numpy(), b64.grad.numpy(), 2e-4, "db_e (autograd)")


def test_tau_draws_follow_the_philox_law():
    from scipy.stats import kstest
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    from oracle import philox
    rows, N = 1563, 64                                          # 100 032 draws
    ctr = torch.zeros(1, dtype=torch.int64, device=DEV)
    a, b = torch.empty(rows, N, device=DEV), torch.empty(rows, N, device=DEV)
    C.jb_iqn_tau(ptr(a), rows, N, 0.0, 1.0, 11, 5, ptr(ctr), stream_ptr())
    C.jb_iqn_tau(ptr(b), rows, N, 0.0, 1.0, 11, 5, ptr(ctr), stream_ptr())
    torch.cuda.synchronize()
    n = rows * N
    assert ctr.item() == 2 * ((n + 3) // 4)
    x = a.cpu().numpy().reshape(-1)
    assert x.min() >= 0.0 and x.max() < 1.0
    assert kstest(x, "uniform").pvalue > 1e-3
    assert not torch.equal(a, b) and (a == b).float().mean().item() < 1e-3      # fresh draws per call
    # bit-exact against the numpy Philox: element e is word e % 4 of Philox(seed, stream, ctr + e / 4)
    words = np.stack(philox.philox4x32(11, 5, np.arange((n + 3) // 4, dtype=np.uint64)), 1).reshape(-1)[:n]
    assert np.array_equal(x, philox.u01_float(words))
    lo, hi = 0.25, 0.75
    C.jb_iqn_tau(ptr(a), rows, N, lo, hi, 11, 5, ptr(ctr), stream_ptr())
    torch.cuda.synchronize()
    y = a.cpu().numpy().reshape(-1)
    assert y.min() >= lo and y.max() < hi
    assert kstest(y, "uniform", args=(lo, hi - lo)).pvalue > 1e-3


# ----------------------------------------------------------------------------------- 3. one eager learn vs oracle
CAP = 64
LR = 1e-3
LEARN_CASES = {
    "qrdqn_mlp_h64": dict(agent="qrdqn", head="mlp", D=4, A=2, H=64, B=16, K=32),
    "qrdqn_mlp_h512": dict(agent="qrdqn", head="mlp", D=4, A=2, H=512, B=32, K=200),
    "qrdqn_cnn": dict(agent="qrdqn", head="cnn", D=[4, 84, 84], A=18, H=512, B=32, K=200),
    "iqn_mlp": dict(agent="iqn", head="mlp", D=4, A=2, H=64, B=16, N=16),
    "iqn_cnn": dict(agent="iqn", head="cnn", D=[4, 84, 84], A=18, H=512, B=32, N=64),
}


def _agent(case, seed=0, buffer_size=CAP, **extra):
    from jorldy_b200.core import Agent
    torch.manual_seed(seed)
    kw = dict(state_size=case["D"], action_size=case["A"], hidden_size=case["H"], head=case["head"],
              optim_config={"name": "adam", "lr": LR}, gamma=0.99, buffer_size=buffer_size, batch_size=case["B"],
              run_step=1000, lr_decay=False, device=DEV, seed=seed)
    kw.update(dict(num_support=case["K"]) if case["agent"] == "qrdqn" else dict(num_sample=case["N"]))
    kw.update(extra)
    return Agent(case["agent"], **kw)


def _replay(case, rs, n=CAP):
    if case["head"] == "cnn":
        s = rs.randint(0, 256, size=(n, 4, 84, 84)).astype(np.uint8)
        ns = rs.randint(0, 256, size=(n, 4, 84, 84)).astype(np.uint8)
    else:
        s = rs.standard_normal((n, case["D"])).astype(np.float32)
        ns = rs.standard_normal((n, case["D"])).astype(np.float32)
    return {"state": s, "next_state": ns, "action": rs.randint(case["A"], size=(n, 1)).astype(np.int64),
            "reward": rs.standard_normal((n, 1)), "done": rs.uniform(size=(n, 1)) < 0.25}


def _params(net):
    return {k: v.detach().cpu().to(torch.float64) for k, v in net.p.items()}


def _perturb_target(agent, rs):
    """A target net that differs from the online one, so that a* and y depend on which net produced them."""
    with torch.no_grad():
        for k, v in agent.target_network.p.items():
            v.add_(torch.from_numpy(rs.standard_normal(tuple(v.shape)).astype(np.float32)).to(DEV) * 0.05)


@pytest.mark.parametrize("name", list(LEARN_CASES))
def test_eager_learn_matches_the_float64_oracle(name):
    case = LEARN_CASES[name]
    rs = np.random.RandomState(5)
    agent = _agent(case)
    _perturb_target(agent, rs)
    tr = _replay(case, rs)
    agent.memory.store([tr])
    idx = rs.randint(CAP, size=case["B"])
    batch = {"state": torch.from_numpy(tr["state"][idx]), "next_state": torch.from_numpy(tr["next_state"][idx]),
             "action": torch.from_numpy(tr["action"][idx, 0]),
             "reward": torch.from_numpy(tr["reward"][idx, 0].astype(np.float32)),
             "done": torch.from_numpy(tr["done"][idx, 0].astype(np.float32))}
    pre, tgt = _params(agent.network), _params(agent.target_network)
    if case["agent"] == "qrdqn":
        ref = oq.qrdqn_learn(pre, tgt, batch, dict(A=case["A"], K=case["K"], gamma=0.99, lr=LR))
    else:
        tau = rs.uniform(size=(case["B"], case["N"])).astype(np.float32)
        tau_n = rs.uniform(size=(case["B"], case["N"])).astype(np.float32)
        agent._inject_tau = [tau, tau_n, None]
        ref = oq.iqn_learn(pre, tgt, batch, torch.from_numpy(tau), torch.from_numpy(tau_n),
                           dict(D_em=64, gamma=0.99, lr=LR))
    agent._inject_idx = idx
    res = agent.learn()
    torch.cuda.synchronize()
    assert set(res) == {"loss", "epsilon", "max_Q"}
    for k, v in ref["result"].items():
        assert abs(res[k] - v) <= 5e-4 * max(abs(v), 1.0), (name, k, res[k], v)
    cnn = case["head"] == "cnn"
    for k, g in ref["grads"].items():
        loose = k.startswith("head.conv") or (cnn and k.startswith("sample_embed."))
        R = 2e-2 if loose else (2e-3 if cnn else 1e-3)
        _close(agent.network.g[k].cpu().numpy(), g.numpy(), R, f"grad {k}", float(g.abs().max()) + 1e-12)
    for k, p0 in pre.items():
        g = agent.network.g[k].cpu().to(torch.float64)
        want = p0 - LR * g / (g.abs() + 1e-8)
        got = agent.network.p[k].cpu().to(torch.float64)
        assert (got - want).abs().max().item() <= 1e-3 * LR + 2 * U * p0.abs().max().item(), k


# ------------------------------------------------------------------------------------------ 4. bit-reproducible
@pytest.mark.parametrize("agent_name", ["qrdqn", "iqn"])
def test_two_learns_from_the_same_state_are_bit_identical(agent_name):
    case = dict(LEARN_CASES["qrdqn_mlp_h64" if agent_name == "qrdqn" else "iqn_mlp"])
    rs = np.random.RandomState(9)
    a, b = _agent(case), _agent(case)
    b.network.flat.copy_(a.network.flat)
    b.target_network.flat.copy_(a.target_network.flat)
    tr = _replay(case, rs)
    a.memory.store([tr]); b.memory.store([tr])
    for _ in range(3):
        a._inject_idx = b._inject_idx = rs.randint(CAP, size=case["B"])
        ra, rb = a.learn(), b.learn()                  # IQN: the same seed and counter give the same tau draws
        assert ra == rb
    torch.cuda.synchronize()
    assert torch.equal(a.network.flat, b.network.flat)
    if agent_name == "iqn":
        assert a._tau_ctr.item() == b._tau_ctr.item() > 0


# ------------------------------------------------------------------------------------------------------- 5. act
@pytest.mark.parametrize("agent_name", ["qrdqn", "iqn"])
def test_act_greedy_and_epsilon_paths(agent_name):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    case = dict(LEARN_CASES["qrdqn_mlp_h64" if agent_name == "qrdqn" else "iqn_mlp"], A=18)
    agent = _agent(case)
    rs = np.random.RandomState(3)
    M = 2048
    s = torch.from_numpy(rs.standard_normal((M, 4)).astype(np.float32)).to(DEV)
    params = _params(agent.network)
    if agent_name == "iqn":
        tau = rs.uniform(size=(M, case["N"])).astype(np.float32)
        agent._inject_tau = [None, None, tau]
        ref = oq.iqn_q(params, s.cpu(), torch.from_numpy(tau), 64)
    else:
        ref = oq.qrdqn_q(params, s.cpu(), case["A"], case["K"])
    greedy = agent.act_device(s, training=False)[0].clone()
    top2 = torch.topk(ref, 2, dim=1).values
    bad = (greedy.cpu() != ref.argmax(1)) & ((top2[:, 0] - top2[:, 1]) > 1e-5)
    assert not bad.any()
    q = agent.network._buf("act.q", (M, case["A"])).cpu().to(torch.float64)
    _close(q.numpy(), ref.numpy(), 1e-4, "act Q", float(ref.abs().max()))
    # the epsilon path is jb_q_act on these Q values
    agent.epsilon = 0.5
    u = torch.from_numpy(rs.uniform(size=(M, 2)).astype(np.float32)).to(DEV)
    got, _ = agent.act_device(s, training=True, noise=u)
    got = got.clone()
    q_dev = agent.network._buf("act.q", (M, case["A"]))
    want = torch.empty(M, dtype=torch.int64, device=DEV)
    C.jb_q_act(ptr(q_dev), M, case["A"], 0.5, None, ptr(u), 0, 0, None, ptr(want), None, stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert (got.cpu() != greedy.cpu()).any()
    if agent_name == "iqn":
        agent._inject_tau = None                          # drawn from the agent's Philox stream from here on
    out = agent.act(s[:5].cpu().numpy(), training=False)["action"]
    assert out.dtype == np.int64 and out.shape == (5, 1)


def test_iqn_act_chunks_count_rows_times_samples():
    from jorldy_b200.core.network import iqn
    case = dict(LEARN_CASES["iqn_cnn"], H=64)
    agent = _agent(case)
    net = agent.network
    per = iqn.ROW_BYTES_PER_PASS // (4 * net.head.D_head_out * case["N"])
    assert per == 41
    M = 2 * per + 3                                       # three chunks, the last one short
    rs = np.random.RandomState(1)
    s = torch.from_numpy(rs.randint(0, 256, size=(M, 4, 84, 84)).astype(np.uint8)).to(DEV)
    tau = rs.uniform(size=(M, case["N"])).astype(np.float32)
    agent._inject_tau = [None, None, tau]
    agent.act_device(s, training=False)
    q = agent.network._buf("act.q", (M, case["A"])).cpu().to(torch.float64)
    ref = oq.iqn_q(_params(net), s.cpu(), torch.from_numpy(tau), 64)
    _close(q.numpy(), ref.numpy(), 1e-3, "chunked act Q", float(ref.abs().max()))


# ---------------------------------------------------------------------------------------------------- 6. frames
N_LANES, PERIOD, ROUNDS = 4, 8, 6


@pytest.mark.parametrize("agent_name", ["qrdqn", "iqn"])
def test_frame_replay_learn_equals_the_stacked_twin(agent_name):
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    case = dict(agent=agent_name, head="cnn", D=[4, 84, 84], A=18, H=64, B=16, K=200, N=8)
    agent = _agent(case, buffer_size=256, start_train_step=10 ** 9)
    env = Env("seaquest", num_envs=N_LANES, seed=2, device=DEV)
    rc = ReplayCollector(env, agent, update_period=PERIOD)
    step = 0
    for _ in range(ROUNDS):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    mem = agent.memory
    assert rc.frames is not None and mem.frames is rc.frames and mem.size == N_LANES * PERIOD * ROUNDS
    twin = _agent(case, buffer_size=256)
    twin.network.flat.copy_(agent.network.flat)
    twin.target_network.flat.copy_(agent.target_network.flat)
    twin.memory.store([mem.gather_device(torch.arange(mem.size, device=DEV))])
    assert twin.memory.frames is None
    if agent_name == "iqn":
        twin._tau_ctr.copy_(agent._tau_ctr)
    rs = np.random.RandomState(4)
    for _ in range(3):
        agent._inject_idx = twin._inject_idx = rs.randint(mem.size, size=case["B"])
        assert agent.learn() == twin.learn()
    torch.cuda.synchronize()
    assert torch.equal(agent.network.flat, twin.network.flat)


# ------------------------------------------------------------------------------------------------ 7. checkpoints
@pytest.mark.parametrize("agent_name", ["qrdqn", "iqn"])
def test_checkpoint_keys_and_round_trip(tmp_path, agent_name):
    case = dict(LEARN_CASES["qrdqn_mlp_h64" if agent_name == "qrdqn" else "iqn_mlp"], H=32, B=4)
    a = _agent(case, start_train_step=1)
    rs = np.random.RandomState(1)
    s = rs.standard_normal((8, 4)).astype(np.float32)
    tr = {"state": s, "next_state": s[::-1].copy(), "reward": np.ones((8, 1)), "done": np.zeros((8, 1), dtype=bool),
          "action": a.act(s, True)["action"]}
    for step in range(1, 4):
        a.process([tr], step)
    assert a.num_learn == 3
    a.save(str(tmp_path))
    ck = torch.load(str(tmp_path / "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "optimizer"}
    if agent_name == "qrdqn":
        assert list(ck["network"]) == ["head.l.weight", "head.l.bias", "l.weight", "l.bias", "q.weight", "q.bias"]
        assert tuple(ck["network"]["q.weight"].shape) == (2 * case["K"], 32)
    else:
        assert list(ck["network"]) == ["head.l.weight", "head.l.bias", "sample_embed.weight", "sample_embed.bias",
                                       "l.weight", "l.bias", "q.weight", "q.bias"]
        assert tuple(ck["network"]["sample_embed.weight"].shape) == (32, 64)
    b = _agent(case, seed=9)
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, a.network.flat) and torch.equal(b.target_network.flat, a.network.flat)
    assert torch.equal(b.optimizer.exp_avg, a.optimizer.exp_avg)


# -------------------------------------------------------------------------------------------------- 8. end to end
@pytest.mark.parametrize("config,extra,sizes", [
    ("config.qrdqn.cartpole", ["--train.num_workers", "8", "--agent.start_train_step", "64"], (4, 2)),
    ("config.iqn.atari", ["--env.name", "seaquest", "--train.num_workers", "8", "--agent.start_train_step", "16",
                          "--agent.buffer_size", "8192", "--agent.hidden_size", "64"], ([4, 84, 84], 18)),
])
def test_sync_training_run(tmp_path, config, extra, sizes):
    """`python -m jorldy_b200.main --sync --config ...` for 512 steps; run_mode prints a traceback instead of raising, so
    the output is checked: the last step line, and a checkpoint that loads into a fresh agent with an identical state."""
    from jorldy_b200.core import Agent
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable, "-m", "jorldy_b200.main", "--sync", "--config", config, "--train.run_step", "512",
           "--train.print_period", "256", "--train.save_period", "512", *extra]
    r = subprocess.run(cmd, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith("512 step |") and "max_Q" in line for line in r.stdout.splitlines()), out[-4000:]
    ckpts = [d for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    saved = torch.load(os.path.join(ckpts[0], "ckpt"), map_location="cpu", weights_only=False)
    D, A = sizes
    name = config.split(".")[1]
    kw = dict(head="cnn", hidden_size=64) if config.endswith("atari") else {}
    fresh = Agent(name, state_size=D, action_size=A, device=DEV, **kw)
    fresh.load(ckpts[0])
    for k, v in fresh.network.state_dict().items():
        assert torch.equal(v.cpu(), saved["network"][k]), k
