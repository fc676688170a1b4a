"""Rainbow-IQN on the GPU (jb_rainbow_iqn_loss in csrc/quantile.cu, core/network/rainbow_iqn.py, core/agent/rainbow_iqn.py)
against the float64 oracle (oracle/rainbow_iqn.py), against jb_quantile_loss, float64 autograd, the stacked replay layout
and the run loop (pytest -m gpu).

Tolerances.  u = 2^-24 is fp32's unit roundoff; S_b = 1 + sum_s |r_bs| + max |next_target[b]|.
- Loss kernel (1).  The n-step fold takes 3 roundings per step on values bounded by S_b: |dy| <= 4 n u S_b = tol_b.
  a* is compared exactly: the online means on s' are built >= 0.01 apart (a warp mean of <= 256 values is within
  16 u max|x| ~ 1e-5 of the float64 mean) or exactly tied (identical columns give identical fp32 means, and the first
  index wins in both).  The quantile Huber is 1-Lipschitz in y with weights <= 1, so a dpred element moves by at most
  w_b (tol_b + (Np + 2) u) / B (the sum over j adds Np u relative, the weight and 1/(B Np) one rounding each), and the
  per-sample loss by N tol_b + (Np + 13) u L_b (N' sequential adds per quantile and an 8-warp tree, as in
  test_quantile_gpu.py).  p_b = L_b^alpha moves by alpha L_b^(alpha - 1) times that, plus 2 u p_b.  The batch loss adds
  B u of the sum.  max_Q is a warp mean (16 u max|pred|), max_logit / min_logit are selections (exact).  The mutations this
  is meant to catch (a* from the target net, the batch-mean weight, the fold in the wrong order, the weight dropped from the
  gradient) move these by 10^2..10^6 times the bounds.
- Anchor (2).  With n = 1, next_online == next_target and no weights, the kernel runs jb_quantile_loss's arithmetic in the
  same order (the same warp means, the same target rounding, gcoef = 1 / (B Np) rounded once, the same quantile_huber
  and a sequential fold of the batch loss), so dpred, loss, a*, stats[0] and stats[1] are bit-identical; a weight of 1.0
  multiplies exactly.
- Network (4).  As test_quantile_gpu.py: normwise per tensor, output 1e-4, gradients 1e-3 (MLP), 2e-3 (CNN outside the
  trunk), 2e-2 for the conv trunk and the CNN's sample_embed (sums over ~10^5 ReLU pre-activations, a few of which lie
  within fp32 rounding of 0 and take the other branch in float64).  With a random dout every gradient under a ReLU is a
  random-sign sum over rows, so one such flipped pre-activation moves it by ~1/sqrt(rows) of its scale; at the MLP's
  B N H = 2^16 pre-activations of f one flip is likely, so the MLP cases give the float64 ReLUs the GPU forward's on/off
  pattern (an element within rounding of 0 then contributes ~0 in both) and keep 1e-3 on every tensor.
- One learn (5): the same gradient bounds; loss, max_Q, max_logit, min_logit at rtol 5e-4; priorities written into the tree
  at rtol 5e-4 (alpha = 0.5 halves the loss's relative error); sampled_p / mean_p come from the same f64 tree as the
  oracle's (1e-12).  Parameters against a float64 Adam step on the kernel's own gradients, bound 1e-3 lr + 2 u |p|.
- act (7): the chunked act against the one-pass forward at 1e-4 normwise (row chunks change no sum's order, only which
  GEMM tile computes a row), and against the float64 oracle at 1e-3 like IQN's chunked act.
- Repeated learns (6), frames vs stacks (8) and checkpoints (9) are bit-exact.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import quantile as oq
from oracle import rainbow_iqn as ori
from oracle.per import SumTree

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
GAMMA = float(np.float32(0.99))
PALPHA = 0.5


def _close(got, ref, R, what, scale=None):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = max(float(np.abs(ref).max()), 1e-30) if scale is None else scale
    err = float(np.abs(got - ref).max())
    assert err <= R * scale, f"{what}: max |err| {err:.3e} > {R} * {scale:.3e}"


def _dv(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _h(x):
    return torch.from_numpy(np.asarray(x)).to(torch.float64)


# ----------------------------------------------------------------------------------------- 1. kernel vs the oracle
def _inputs(rs, B, A, N, Nn, Np, n):
    """Online means on s' >= 0.01 apart, tied at the max on every third row; on even rows the target net's best mean is
    another action than the online net's, so a* taken from the wrong net changes y."""
    qn = 2.0 * rs.standard_normal((B, A))
    ar = np.arange(B)
    top = qn.argmax(1)
    qn[ar, top] = np.sort(qn, 1)[:, -2] + 0.01 + rs.uniform(size=B) if A > 1 else qn[ar, top]
    on = qn[:, None, :] + 0.5 * rs.standard_normal((B, Nn, A))
    on = (on - on.mean(1, keepdims=True) + qn[:, None, :]).astype(np.float32)
    tie = (ar % 3 == 0) & (A > 1)
    for b in np.nonzero(tie)[0]:
        on[b, :, (top[b] + 1) % A] = on[b, :, top[b]]
    a_on = np.where(tie, np.minimum(top, (top + 1) % A), top)
    tg = 2.0 * rs.standard_normal((B, Np, A))
    if A > 1:
        alt = (a_on + 1) % A
        tg[ar % 2 == 0, :, alt[ar % 2 == 0]] += 10.0
    tg = tg.astype(np.float32)
    reward = rs.standard_normal((B, n)).astype(np.float32)
    done = (rs.uniform(size=(B, n)) < 0.3).astype(np.float32)
    a_t = rs.randint(A, size=B)
    fr = rs.uniform(size=(B, N)).astype(np.float32)
    return on, tg, reward, done, a_t, fr, a_on, tie


def _weights(rs, kind, B):
    if kind == "null":
        return None
    if kind == "ones":
        return np.ones(B)
    w = rs.uniform(0.05, 1.0, size=B)
    w[rs.randint(B)] = 1.0
    return w


def _launch(g, B, A, N, Nn, Np, n, alpha=PALPHA):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    out = dict(dpred=torch.full((B, N, A), float("nan"), device=DEV), loss=torch.full((B,), float("nan"), device=DEV),
               prio=torch.full((B,), float("nan"), dtype=torch.float64, device=DEV),
               a_star=torch.full((B,), -1, dtype=torch.int32, device=DEV), stats=torch.full((4,), float("nan"), device=DEV))
    scratch = torch.empty(4 * B, device=DEV)
    C.jb_rainbow_iqn_loss(ptr(g["p"]), ptr(g["on"]), ptr(g["tg"]), ptr(g["t"]), ptr(g["a"]), 0, ptr(g["r"]), ptr(g["d"]),
                          ptr(g.get("w")), B, A, N, Nn, Np, n, GAMMA, alpha, ptr(out["dpred"]), ptr(out["loss"]),
                          ptr(out["prio"]), ptr(out["a_star"]), ptr(out["stats"]), ptr(scratch), stream_ptr())
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("N,Nn,Np", [(1, 1, 1), (64, 64, 64), (32, 17, 8), (200, 3, 256)])
@pytest.mark.parametrize("A", [2, 18])
@pytest.mark.parametrize("B", [1, 32, 257])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("wkind", ["null", "ones", "random"])
def test_loss_kernel_matches_the_oracle(N, Nn, Np, A, B, n, wkind):
    rs = np.random.RandomState(N + 3 * Nn + 5 * Np + 7 * A + B + 11 * n + len(wkind))
    on, tg, reward, done, a_t, fr, a_on, tie = _inputs(rs, B, A, N, Nn, Np, n)
    w = _weights(rs, wkind, B)
    wh = _h(w) if w is not None else torch.ones(B, dtype=torch.float64)
    a_star, y = ori.targets(_h(on), _h(tg), _h(reward), _h(done), GAMMA)
    assert np.array_equal(a_star.numpy(), a_on)
    if A > 1 and B > 1:                      # rows where the target net would pick another action, and ties
        assert (_h(tg).mean(1).argmax(1).numpy() != a_on).any() and tie.any()
    pred = np.clip(2.0 * rs.standard_normal((B, N, A)), -8, 8)
    pred[np.arange(B), :, a_t] = y.mean(1).numpy()[:, None] + 1.5 * rs.standard_normal((B, N))
    pred = pred.astype(np.float32)
    g = {k: _dv(v) for k, v in dict(p=pred, on=on, tg=tg, t=fr, a=a_t.astype(np.int64), r=reward, d=done).items()}
    if w is not None:
        g["w"] = _dv(w)
    o = _launch(g, B, A, N, Nn, Np, n)
    dpred, stats = o["dpred"].cpu().numpy(), o["stats"].cpu().numpy()
    assert np.isfinite(dpred).all() and np.isfinite(stats).all()
    assert np.array_equal(o["a_star"].cpu().numpy(), a_on)
    S = 1 + np.abs(reward).sum(1) + np.abs(tg).reshape(B, -1).max(1)
    tol = 4 * n * U * S
    ar = np.arange(B)
    theta, tau = _h(pred)[torch.arange(B), :, torch.from_numpy(a_t)], _h(fr)
    per = oq.per_sample_loss(theta, y, tau).numpy()
    want = np.zeros((B, N, A))
    want[ar, :, a_t] = ori.grad_closed(theta, y, tau, wh).numpy()
    err = np.abs(dpred - want).reshape(B, -1).max(1)
    assert (err <= wh.numpy() * (tol + (Np + 2) * U) / B).all(), f"dpred: worst row {err.argmax()} err {err.max():.3e}"
    mask = np.ones((B, A), bool)
    mask[ar, a_t] = False
    assert np.all(dpred.transpose(0, 2, 1)[mask] == 0.0)
    loss_tol = N * tol + (Np + 13) * U * per
    assert (np.abs(o["loss"].cpu().numpy() - per) <= loss_tol).all()
    prio_ref = per ** PALPHA
    assert (np.abs(o["prio"].cpu().numpy() - prio_ref) <= PALPHA * per ** (PALPHA - 1) * loss_tol + 2 * U * prio_ref).all()
    wl = wh.numpy() * per
    assert abs(stats[0] - wl.mean()) <= (wh.numpy() * loss_tol).mean() + B * U * wl.mean() + 1e-30
    _close(stats[1], _h(pred).mean(1).max().item(), 16 * U, "max_Q", float(np.abs(pred).max()))
    assert stats[2] == pred.max() and stats[3] == pred.min()


def test_loss_kernel_rejects_out_of_range_arguments():
    from jorldy_b200._lib import JbError
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    B = 2
    x = torch.zeros(B * 19 * 257, device=DEV)
    a = torch.zeros(B, dtype=torch.int64, device=DEV)
    small = torch.zeros(16, device=DEV)
    out = torch.zeros(B * 19 * 257, device=DEV)
    for A, N, Nn, Np, n, kind in ((19, 8, 8, 8, 1, 0), (2, 257, 8, 8, 1, 0), (2, 8, 257, 8, 1, 0), (2, 8, 8, 257, 1, 0),
                                  (2, 8, 0, 8, 1, 0), (2, 0, 8, 8, 1, 0), (2, 8, 8, 0, 1, 0), (2, 8, 8, 8, 0, 0),
                                  (2, 8, 8, 8, 1, 3), (2, 8, 8, 8, 1, -1)):
        with pytest.raises(JbError):
            C.jb_rainbow_iqn_loss(ptr(x), ptr(x), ptr(x), ptr(small), ptr(a), kind, ptr(small), ptr(small), None, B, A, N,
                                  Nn, Np, n, GAMMA, PALPHA, ptr(out), ptr(small), None, None, ptr(small), ptr(small),
                                  stream_ptr())
    with pytest.raises(JbError):
        C.jb_rainbow_iqn_loss(None, ptr(x), ptr(x), ptr(small), ptr(a), 0, ptr(small), ptr(small), None, B, 2, 8, 8, 8, 1,
                              GAMMA, PALPHA, ptr(out), ptr(small), None, None, ptr(small), ptr(small), stream_ptr())


# --------------------------------------------------------------------------------------- 2. anchor: jb_quantile_loss
@pytest.mark.parametrize("N,Np", [(1, 1), (64, 64), (32, 8), (200, 256)])
@pytest.mark.parametrize("A", [2, 18])
@pytest.mark.parametrize("B", [1, 32, 257])
def test_one_step_unweighted_equals_quantile_loss(N, Np, A, B):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(300 + N + Np + A + B)
    on, _, reward, done, a_t, fr, _, _ = _inputs(rs, B, A, N, Np, Np, 1)
    pred = (2.0 * rs.standard_normal((B, N, A))).astype(np.float32)
    g = {k: _dv(v) for k, v in dict(p=pred, on=on, t=fr, a=a_t.astype(np.int64), r=reward, d=done).items()}
    g["tg"] = g["on"]                                              # the same tensor: one pass is both nets
    dq = torch.full((B, N, A), float("nan"), device=DEV)
    lq = torch.full((B,), float("nan"), device=DEV)
    aq = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    sq = torch.full((4,), float("nan"), device=DEV)
    C.jb_quantile_loss(ptr(g["p"]), 1, A, ptr(g["on"]), 1, A, ptr(g["t"]), N, ptr(g["a"]), 0, ptr(g["r"]), ptr(g["d"]), B,
                       A, N, Np, GAMMA, ptr(dq), ptr(lq), ptr(aq), ptr(sq), ptr(torch.empty(2 * B, device=DEV)),
                       stream_ptr())
    for w in (None, np.ones(B)):
        if w is not None:
            g["w"] = _dv(w)
        o = _launch(g, B, A, N, Np, Np, 1)
        assert torch.equal(o["dpred"], dq) and torch.equal(o["loss"], lq) and torch.equal(o["a_star"], aq)
        assert torch.equal(o["stats"][:2], sq[:2])


# ---------------------------------------------------------------------------------- 4. network vs float64 autograd
def _noise(rs, H, A):
    return [(rs.standard_normal(H).astype(np.float32), rs.standard_normal(o).astype(np.float32)) for o in (H, H, A, 1)]


def _noise_dev(nz):
    return [(_dv(a), _dv(b)) for a, b in nz]


def _noise_h(nz):
    return [(_h(a), _h(b)) for a, b in nz]


def _params(net):
    return {k: v.detach().cpu().to(torch.float64) for k, v in net.p.items()}


def _states(rs, head, D, n):
    if head == "cnn":
        return rs.randint(0, 256, size=(n, 4, 84, 84)).astype(np.uint8)
    return rs.standard_normal((n, D)).astype(np.float32)


def _rt(k, cnn):
    loose = k.startswith("head.conv") or (cnn and k.startswith("sample_embed."))
    return 2e-2 if loose else (2e-3 if cnn else 1e-3)


@pytest.mark.parametrize("head,D,A,H,B,N", [("mlp", 4, 2, 64, 16, 8), ("mlp", 4, 6, 512, 8, 16),
                                            ("cnn", [4, 84, 84], 18, 512, 4, 16)])
def test_network_forward_and_backward_match_autograd(head, D, A, H, B, N, monkeypatch):
    from jorldy_b200.core.network import Network
    rs = np.random.RandomState(H + A)
    net = Network("rainbow_iqn", D, A, D_em=64, D_hidden=H, head=head, device=DEV, seed=3)
    with torch.no_grad():                                          # sigma away from its init, so dsig is not dmu * eps
        for k, v in net.p.items():
            if k.startswith("sig_"):
                v.copy_(torch.from_numpy(rs.uniform(0.01, 0.2, size=tuple(v.shape)).astype(np.float32)))
    x = _states(rs, head, D, B)
    tau = rs.uniform(size=(B, N)).astype(np.float32)
    nz = _noise(rs, H, A)
    out = net.forward(_dv(x), _dv(tau), True, "t.", _noise_dev(nz)).clone()
    dout = rs.standard_normal((B * N, A)).astype(np.float32)
    net.backward(_dv(dout), "t.")
    torch.cuda.synchronize()
    p = {k: v.clone().requires_grad_(True) for k, v in _params(net).items()}
    if head == "mlp":                    # the oracle's ReLUs (psi, phi, f, xa, xv in call order) take the GPU's on/off pattern
        acts = [net._buf("t.head.h", (B, H)).view(B, H)] + [net._buf(f"t.{k}", (B * N, d)).view(B, N, d)
                                                           for k, d in (("phi", H), ("f", H), ("xa", H), ("xv", H))]
        masks = iter([(a > 0).cpu().to(torch.float64) for a in acts])
        monkeypatch.setattr(torch.nn.functional, "relu", lambda t: t * next(masks))
    ref = ori.network(p, _h(x), _h(tau), 64, _noise_h(nz))
    monkeypatch.undo()
    _close(out.cpu().numpy(), ref.detach().reshape(B * N, A).numpy(), 1e-4, "out")
    (ref.reshape(B * N, A) * _h(dout)).sum().backward()
    cnn = head == "cnn"
    for k, v in p.items():
        _close(net.g[k].cpu().numpy(), v.grad.numpy(), _rt(k, cnn), f"grad {k}", float(v.grad.abs().max()) + 1e-12)
    assert list(net.p)[:4] == ["mu_w_a1", "sig_w_a1", "mu_b_a1", "sig_b_a1"]


# ----------------------------------------------------------------------------------- 5. one eager learn vs oracle
CAP = 64
LR = 1e-3
LEARN_CASES = {
    "mlp": dict(head="mlp", D=4, A=2, H=64, B=16, N=16, n=3),
    "cnn": dict(head="cnn", D=[4, 84, 84], A=18, H=512, B=32, N=64, n=3),
}


def _agent(case, seed=0, buffer_size=CAP, **extra):
    from jorldy_b200.core import Agent
    torch.manual_seed(seed)
    kw = dict(state_size=case["D"], action_size=case["A"], hidden_size=case["H"], head=case["head"],
              optim_config={"name": "adam", "lr": LR}, gamma=0.99, buffer_size=buffer_size, batch_size=case["B"],
              run_step=1000, lr_decay=False, device=DEV, seed=seed, alpha=PALPHA, beta=0.4, n_step=case["n"],
              num_sample=case["N"], start_train_step=0)
    kw.update(extra)
    return Agent("rainbow_iqn", **kw)


def _replay(case, rs, n=CAP):
    return {"state": _states(rs, case["head"], case["D"], n), "next_state": _states(rs, case["head"], case["D"], n),
            "action": rs.randint(case["A"], size=(n, 1)).astype(np.int64),
            "reward": rs.standard_normal((n, case["n"], 1)).astype(np.float32),
            "done": rs.uniform(size=(n, case["n"], 1)) < 0.25}


def _filled(case, rs, agent):
    """The agent's PER replay and the oracle sum-tree with the same non-uniform priorities."""
    tr = _replay(case, rs)
    agent.memory.store([tr])
    ora = SumTree(CAP, agent.memory.uniform_sample_prob)
    ora.store(CAP)
    pr = rs.uniform(0.1, 2.0, size=CAP)
    leaves = np.arange(CAP) + ora.first_leaf
    agent.memory.update_priorities(_dv(leaves.astype(np.int64)), _dv(pr))
    for i, p in zip(leaves, pr):
        ora.update(p, i)
    return tr, ora


def _perturb_target(agent, rs):
    with torch.no_grad():
        for v in agent.target_network.p.values():
            v.add_(torch.from_numpy(rs.standard_normal(tuple(v.shape)).astype(np.float32)).to(DEV) * 0.05)


@pytest.mark.parametrize("name", list(LEARN_CASES))
def test_eager_learn_matches_the_float64_oracle(name):
    case = LEARN_CASES[name]
    B, N, H, A = case["B"], case["N"], case["H"], case["A"]
    rs = np.random.RandomState(5)
    agent = _agent(case)
    _perturb_target(agent, rs)
    tr, ora = _filled(case, rs, agent)
    u_a, u_b = rs.uniform(size=B), rs.uniform(size=B)
    u_a[0] = 1e-4                                                  # one uniform slot
    idx, w, sampled_p, mean_p = ora.sample(agent.beta, u_a, u_b)
    rows = idx - ora.first_leaf
    batch = {"state": torch.from_numpy(tr["state"][rows]), "next_state": torch.from_numpy(tr["next_state"][rows]),
             "action": torch.from_numpy(tr["action"][rows, 0]), "reward": torch.from_numpy(tr["reward"][rows, :, 0]),
             "done": torch.from_numpy(tr["done"][rows, :, 0].astype(np.float32))}
    taus = [rs.uniform(size=(B, N)).astype(np.float32) for _ in range(3)]
    noise = [_noise(rs, H, A) for _ in range(3)]
    pre, tgt = _params(agent.network), _params(agent.target_network)
    ref = ori.learn(pre, tgt, batch, torch.from_numpy(w), [torch.from_numpy(t) for t in taus], [_noise_h(z) for z in noise],
                    dict(D_em=64, gamma=GAMMA, alpha=PALPHA, lr=LR))
    agent._inject_u = (u_a, u_b)
    agent._inject_tau = taus + [None]
    agent._inject_noise = [_noise_dev(z) for z in noise]
    res = agent.learn()
    torch.cuda.synchronize()
    assert set(res) == {"loss", "beta", "max_Q", "max_logit", "min_logit", "sampled_p", "mean_p"}
    assert res["beta"] == 0.4 and agent.num_learn == 1
    for k, v in ref["result"].items():
        assert abs(res[k] - v) <= 5e-4 * max(abs(v), 1.0), (name, k, res[k], v)
    assert abs(res["sampled_p"] - sampled_p) <= 1e-12 * sampled_p and abs(res["mean_p"] - mean_p) <= 1e-12 * mean_p
    for i, p in zip(idx, ref["prio"].numpy()):
        ora.update(p, i)
    got_tree = agent.memory.sum_tree
    np.testing.assert_allclose(got_tree[ora.first_leaf:], ora.tree[ora.first_leaf:], rtol=5e-4)
    cnn = case["head"] == "cnn"
    for k, g in ref["grads"].items():
        _close(agent.network.g[k].cpu().numpy(), g.numpy(), _rt(k, cnn), f"grad {k}", float(g.abs().max()) + 1e-12)
    for k, p0 in pre.items():
        g = agent.network.g[k].cpu().to(torch.float64)
        want = p0 - LR * g / (g.abs() + 1e-8)
        got = agent.network.p[k].cpu().to(torch.float64)
        assert (got - want).abs().max().item() <= 1e-3 * LR + 2 * U * p0.abs().max().item(), k


# ------------------------------------------------------------------------------------------ 6. bit-reproducible
def test_two_learns_from_the_same_state_are_bit_identical():
    case = LEARN_CASES["mlp"]
    rs = np.random.RandomState(9)
    a, b = _agent(case), _agent(case)
    _perturb_target(a, rs)
    b.network.flat.copy_(a.network.flat)
    b.target_network.flat.copy_(a.target_network.flat)
    tr = _replay(case, rs)
    a.memory.store([tr]); b.memory.store([tr])
    for _ in range(3):
        a._inject_u = b._inject_u = (rs.uniform(size=case["B"]), rs.uniform(size=case["B"]))
        ra, rb = a.learn(), b.learn()                  # the same seeds and counters give the same fractions and noise
        assert ra == rb
    torch.cuda.synchronize()
    assert torch.equal(a.network.flat, b.network.flat) and torch.equal(a.memory._tree, b.memory._tree)
    assert a._tau_ctr.item() == 3 * 3 * ((case["B"] * case["N"] + 3) // 4)
    assert a.network._draw_ctr.item() == 3 * 8 and a.target_network._draw_ctr.item() == 3 * 4


# ------------------------------------------------------------------------------------------------------- 7. act
def test_act_random_before_the_start_step_then_greedy():
    case = dict(LEARN_CASES["mlp"], A=6)
    agent = _agent(case, buffer_size=128, start_train_step=100)
    rs = np.random.RandomState(3)
    M, N, H, A = 512, case["N"], case["H"], case["A"]
    s = _dv(rs.standard_normal((M, 4)).astype(np.float32))
    torch.manual_seed(11)
    got = agent.act_device(s, training=True)[0].clone()
    torch.manual_seed(11)
    assert torch.equal(got, torch.randint(0, A, (M,), device=DEV))
    assert agent._tau_ctr.item() == 0 and agent.network._draw_ctr.item() == 0
    agent.memory.store([_replay(case, rs, 100)])
    params = _params(agent.network)
    for training in (True, False):
        tau = rs.uniform(size=(M, N)).astype(np.float32)
        nz = _noise(rs, H, A)
        agent._inject_tau = [None, None, None, tau]
        ctr = agent.network._draw_ctr.item()
        greedy = agent.act_device(s, training=training, noise=_noise_dev(nz))[0].clone()
        assert agent.network._draw_ctr.item() == ctr                 # injected or mu weights: no draw
        ref = ori.network(params, s.cpu().to(torch.float64), _h(tau), 64, _noise_h(nz) if training else None).mean(1)
        q = agent.network._buf("act.q", (M, A)).cpu().to(torch.float64)
        _close(q.numpy(), ref.numpy(), 1e-4, f"act Q (training={training})", float(ref.abs().max()))
        top2 = torch.topk(ref, 2, dim=1).values
        assert not ((greedy.cpu() != ref.argmax(1)) & ((top2[:, 0] - top2[:, 1]) > 1e-5)).any()
    agent._inject_tau = None
    out = agent.act(s[:5].cpu().numpy(), training=True)["action"]
    assert out.dtype == np.int64 and out.shape == (5, 1)


def test_act_draws_noise_once_per_call_and_chunks_match_one_pass():
    from jorldy_b200.core.network import iqn
    case = dict(LEARN_CASES["cnn"], H=64)
    agent = _agent(case)
    net, N, H, A = agent.network, case["N"], case["H"], case["A"]
    agent.memory.store([_replay(case, np.random.RandomState(0))])
    per = iqn.ROW_BYTES_PER_PASS // (4 * net.head.D_head_out * N)
    assert per == 41
    rs = np.random.RandomState(1)
    M = 2 * per + 3                                                # three chunks, the last one short
    s = _dv(rs.randint(0, 256, size=(M, 4, 84, 84)).astype(np.uint8))
    for rows in (1, M):                                            # fresh noise: one draw per layer per call
        c0, t0 = net._draw_ctr.item(), agent._tau_ctr.item()
        agent.act_device(s[:rows], training=True)
        torch.cuda.synchronize()
        assert net._draw_ctr.item() - c0 == 4 and agent._tau_ctr.item() - t0 == (rows * N + 3) // 4
    tau = rs.uniform(size=(M, N)).astype(np.float32)
    nz = _noise(rs, H, A)
    agent._inject_tau = [None, None, None, tau]
    agent.act_device(s, training=True, noise=_noise_dev(nz))
    q = agent.network._buf("act.q", (M, A)).cpu().to(torch.float64)
    one = net.forward(s, _dv(tau), True, "one.", _noise_dev(nz)).cpu().to(torch.float64).view(M, N, A).mean(1)
    _close(q.numpy(), one.numpy(), 1e-4, "chunked act vs one pass", float(one.abs().max()))
    ref = ori.network(_params(net), s.cpu().to(torch.float64), _h(tau), 64, _noise_h(nz)).mean(1)
    _close(q.numpy(), ref.numpy(), 1e-3, "chunked act Q", float(ref.abs().max()))


# ---------------------------------------------------------------------------------------------------- 8. frames
def test_frame_replay_learn_equals_the_stacked_twin():
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    case = dict(head="cnn", D=[4, 84, 84], A=18, H=64, B=16, N=8, n=3)
    agent = _agent(case, buffer_size=256, start_train_step=10 ** 9)
    env = Env("seaquest", num_envs=4, seed=2, device=DEV)
    rc = ReplayCollector(env, agent, update_period=8)
    step = 0
    for _ in range(6):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    mem = agent.memory
    assert rc.frames is not None and mem.frames is rc.frames and rc.assembler is not None and mem.size > 0
    twin = _agent(case, buffer_size=256)
    twin.network.flat.copy_(agent.network.flat)
    twin.target_network.flat.copy_(agent.target_network.flat)
    twin.memory.store([mem.gather_device(torch.arange(mem.size, device=DEV))])
    assert twin.memory.frames is None and twin.memory.size == mem.size
    twin.memory._tree.copy_(mem._tree)
    twin.memory._max_priority.copy_(mem._max_priority)
    twin.beta = agent.beta
    twin._tau_ctr.copy_(agent._tau_ctr)
    twin.network._draw_ctr.copy_(agent.network._draw_ctr)
    twin.target_network._draw_ctr.copy_(agent.target_network._draw_ctr)
    rs = np.random.RandomState(4)
    for _ in range(3):
        agent._inject_u = twin._inject_u = (rs.uniform(size=case["B"]), rs.uniform(size=case["B"]))
        assert agent.learn() == twin.learn()
    torch.cuda.synchronize()
    assert torch.equal(agent.network.flat, twin.network.flat) and torch.equal(mem._tree, twin.memory._tree)


# ------------------------------------------------------------------------------------------------ 9. checkpoints
def test_checkpoint_keys_and_round_trip(tmp_path):
    case = dict(LEARN_CASES["mlp"], H=32, B=4)
    a = _agent(case, start_train_step=1, learn_period=1)
    rs = np.random.RandomState(1)
    state = rs.standard_normal((1, 4)).astype(np.float32)
    for step in range(1, 12):
        ns = rs.standard_normal((1, 4)).astype(np.float32)
        tr = {"state": state, "next_state": ns, "reward": np.ones((1, 1)), "done": np.zeros((1, 1), dtype=bool)}
        tr.update(a.act(state, True))
        tr = a.interact_callback(tr)
        if tr:
            a.process([tr], step)
        state = ns
    assert a.num_learn > 0
    a.save(str(tmp_path))
    ck = torch.load(str(tmp_path / "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "optimizer"}
    noisy = [f"{k}{lt}" for lt in ("_a1", "_v1", "_a2", "_v2") for k in ("mu_w", "sig_w", "mu_b", "sig_b")]
    assert list(ck["network"]) == noisy + ["head.l.weight", "head.l.bias", "sample_embed.weight", "sample_embed.bias",
                                           "l.weight", "l.bias"]
    assert tuple(ck["network"]["mu_w_a2"].shape) == (32, 2) and tuple(ck["network"]["sig_b_v2"].shape) == (1,)
    assert tuple(ck["network"]["sample_embed.weight"].shape) == (32, 64)
    b = _agent(case, seed=9)
    assert not torch.equal(b.network.flat, a.network.flat)
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, a.network.flat) and torch.equal(b.target_network.flat, a.network.flat)
    assert torch.equal(b.optimizer.exp_avg, a.optimizer.exp_avg)


# -------------------------------------------------------------------------------------------------- 10. end to end
@pytest.mark.parametrize("config,extra,sizes", [
    ("config.rainbow_iqn.cartpole", ["--train.num_workers", "8", "--agent.start_train_step", "64"], (4, 2)),
    ("config.rainbow_iqn.atari", ["--env.name", "seaquest", "--train.num_workers", "8", "--agent.start_train_step", "16",
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
    kw = dict(head="cnn", hidden_size=64) if config.endswith("atari") else {}
    fresh = Agent("rainbow_iqn", state_size=D, action_size=A, device=DEV, **kw)
    fresh.load(ckpts[0])
    for k, v in fresh.network.state_dict().items():
        assert torch.equal(v.cpu(), saved["network"][k]), k
