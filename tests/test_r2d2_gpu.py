"""R2D2 on the GPU (csrc/lstm.cu, csrc/r2d2.cu, core/network/r2d2.py, core/agent/r2d2.py, SequenceAssembler) against
float64 references (oracle/r2d2.py and torch autograd), the stacked replay layout and the run loop (pytest -m gpu).

Tolerances.  u = 2^-24.  A step kernel's pre-activation is an fp32 sum of K products in ascending k, within (K + 1) u of
sum_k |h_k w_k| + |xg| of the float64 value; the gates are 1-Lipschitz (sigmoid 1/4) and the cell update adds a few
roundings, so h, c and the gates are checked at (K + 8) u (S + 1)(1 + max|c_prev|), S the largest such row sum.  The
backward's recurrent product is the same bound with K = 4H over |dgates_next| |W_hh|, and the gates it multiplies come
from the fp32 forward (a few u apart from float64), hence 1e-5 of the largest gradient on top.  The loss kernel forms its
targets and sums in float64, like the oracle: only dq's final rounding (u) and the order of the sums differ, so it is
checked at 1e-6 (dq, loss) and 1e-12 (priorities).  The network and the learns are checked normwise per tensor as the
other learners' tests are: Q 1e-4, gradients 1e-3 (MLP) and 2e-2 for the conv trunk.  Repeated learns, frames against
stacks and checkpoints are bit-exact.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import r2d2 as orr
from oracle.per import SumTree

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
GAMMA = float(np.float32(0.997))
LR = 1e-4


def _dv(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _close(got, ref, R, what, scale=None):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = max(float(np.abs(ref).max()), 1e-30) if scale is None else scale
    err = float(np.abs(got - ref).max())
    assert err <= R * scale, f"{what}: max |err| {err:.3e} > {R} * {scale:.3e}"


def _C():
    from jorldy_b200._lib import C
    return C


def _s():
    return torch.cuda.current_stream().cuda_stream


def _reset(rs, kind, M):
    if kind == "none":
        return None
    r = np.ones(M, np.float32) if kind == "all" else (rs.uniform(size=M) < 0.3).astype(np.float32)
    return r


# ------------------------------------------------------------------------------------------- 1. step kernels
@pytest.mark.parametrize("M", [1, 7, 64, 257])
@pytest.mark.parametrize("H,Z", [(64, 3136 + 18), (512, 512 + 2)])
@pytest.mark.parametrize("rkind", ["none", "all", "random"])
def test_lstm_step_kernels_match_float64_autograd(M, H, Z, rkind):
    C = _C()
    rs = np.random.RandomState(M + H)
    k = 1.0 / np.sqrt(H)
    f = lambda *s: rs.uniform(-k, k, size=s).astype(np.float32)
    x = _dv(np.maximum(rs.standard_normal((M, Z)), 0).astype(np.float32))
    w_ih, w_hh, b = _dv(f(4 * H, Z)), _dv(f(4 * H, H)), _dv(f(4 * H))
    xg = torch.empty(M, 4 * H, device=DEV)
    C.jb_linear_fwd(x.data_ptr(), w_ih.data_ptr(), b.data_ptr(), xg.data_ptr(), M, Z, 4 * H, 0, _s())
    hp, cp = _dv(rs.standard_normal((M, H)).astype(np.float32) * 0.5), _dv(rs.standard_normal((M, H)).astype(np.float32))
    rnp = _reset(rs, rkind, M)
    reset = None if rnp is None else _dv(rnp)
    h, c, hpe = (torch.empty(M, H, device=DEV) for _ in range(3))
    gates = torch.empty(M, 4 * H, device=DEV)
    rp = 0 if reset is None else reset.data_ptr()
    C.jb_lstm_step_fwd(xg.data_ptr(), hp.data_ptr(), cp.data_ptr(), w_hh.data_ptr(), rp, M, H, h.data_ptr(), c.data_ptr(),
                       gates.data_ptr(), hpe.data_ptr(), _s())
    d = lambda t: t.cpu().to(torch.float64)
    keep = torch.ones(M, 1, dtype=torch.float64) if rnp is None else torch.from_numpy(1.0 - rnp).to(torch.float64)[:, None]
    hp64, cp64 = d(hp) * keep, (d(cp) * keep).requires_grad_(True)
    pre = (d(xg) + hp64 @ d(w_hh).T).requires_grad_(True)
    gi, gf, gg, go = pre.chunk(4, -1)
    c_ref = torch.sigmoid(gf) * cp64 + torch.sigmoid(gi) * torch.tanh(gg)
    h_ref = torch.sigmoid(go) * torch.tanh(c_ref)
    S = float((hp64.abs() @ d(w_hh).abs().T).max() + d(xg).abs().max())
    tol = (H + 8) * U * (S + 1) * (1 + float(cp64.detach().abs().max()))
    _close(d(h), h_ref.detach(), tol, "h", 1.0)
    _close(d(c), c_ref.detach(), tol, "c", 1.0)
    g_ref = torch.cat([torch.sigmoid(gi), torch.sigmoid(gf), torch.tanh(gg), torch.sigmoid(go)], -1)
    _close(d(gates), g_ref.detach(), tol, "gates", 1.0)
    assert torch.equal(hpe.cpu(), (hp.cpu() * keep.float()))
    # backward: the gradient of <dh_out + dgates_next W_hh, h> + <dc_next, c>, the recurrent terms dropped on reset_next rows
    dh_out = _dv(rs.standard_normal((M, H)).astype(np.float32))
    dgn = _dv(rs.standard_normal((M, 4 * H)).astype(np.float32) * 0.1)
    dcn = _dv(rs.standard_normal((M, H)).astype(np.float32))
    rn_np = _reset(rs, "random", M)
    rn = _dv(rn_np)
    dg, dc = torch.empty(M, 4 * H, device=DEV), torch.empty(M, H, device=DEV)
    C.jb_lstm_step_bwd(dh_out.data_ptr(), dgn.data_ptr(), w_hh.data_ptr(), gates.data_ptr(), cp.data_ptr(), c.data_ptr(),
                       dcn.data_ptr(), rp, rn.data_ptr(), M, H, dg.data_ptr(), dc.data_ptr(), _s())
    cross = torch.from_numpy(1.0 - rn_np).to(torch.float64)[:, None]
    dh_tot = d(dh_out) + cross * (d(dgn) @ d(w_hh))
    L = (dh_tot * h_ref).sum() + (cross * d(dcn) * c_ref).sum()
    L.backward()
    Sb = float((d(dgn).abs() @ d(w_hh).abs()).max() + d(dh_out).abs().max() + d(dcn).abs().max())
    scale = float(pre.grad.abs().max()) + 1e-30
    _close(d(dg), pre.grad, (4 * H + 8) * U * Sb / scale + 1e-5, "dgates", scale)
    sc = float(cp64.grad.abs().max()) + 1e-30
    _close(d(dc), cp64.grad, (4 * H + 8) * U * Sb / sc + 1e-5, "dc", sc)


# -------------------------------------------------------------------------------------------- 2. loss kernel
def _loss_inputs(rs, B, T, A, n):
    q = (5 * rs.standard_normal((B, T, A))).astype(np.float32)
    qn = rs.standard_normal((B, T, A)).astype(np.float32)
    qt = (30 * rs.standard_normal((B, T, A))).astype(np.float32)
    if A > 1:
        qn[::3, :, 1] = qn[::3, :, 0]                          # ties: the first index wins
        top = qn.argmax(-1)
        alt = (top + 1) % A                                   # a* disagreement: the target's best is another action
        np.put_along_axis(qt, alt[..., None], np.abs(qt).max() + 1, -1)
    qt.reshape(-1)[::5] = rs.uniform(-1e-4, 1e-4, size=qt.size)[::5]   # values near 0 ...
    qt.reshape(-1)[1::7] = 300.0 * np.sign(rs.standard_normal(qt.size))[1::7]   # ... and large |x|
    act = rs.randint(A, size=(B, T)).astype(np.int64)
    rew = rs.standard_normal((B, T + n)).astype(np.float32)
    done = (rs.uniform(size=(B, T + n)) < 0.15).astype(np.float32)
    return q, qn, qt, act, rew, done


@pytest.mark.parametrize("B", [1, 32, 64, 257])
@pytest.mark.parametrize("T", [1, 5, 80])
@pytest.mark.parametrize("n", [1, 3, 5])
@pytest.mark.parametrize("A", [2, 18])
def test_loss_kernel_matches_the_oracle(B, T, A, n):
    C = _C()
    rs = np.random.RandomState(B * 7 + T * 3 + n + A)
    q, qn, qt, act, rew, done = _loss_inputs(rs, B, T, A, n)
    dq = torch.empty(B, T, A, device=DEV)
    prio = torch.empty(B, dtype=torch.float64, device=DEV)
    stats = torch.empty(2, device=DEV)
    scratch = torch.empty(2 * B, dtype=torch.float64, device=DEV)
    dev = [_dv(a) for a in (q, qn, qt, act, rew, done)]
    h = lambda a: torch.from_numpy(a).to(torch.float64)
    for eta in (0.0, float(np.float32(0.9)), 1.0):      # eta and alpha reach the kernel as fp32
        for wkind in ("none", "ones", "random"):
            w = None if wkind == "none" else (np.ones(B) if wkind == "ones" else rs.uniform(0.05, 1.0, size=B))
            wd = None if w is None else _dv(w)
            C.jb_r2d2_loss(*[t.data_ptr() for t in dev], 0 if wd is None else wd.data_ptr(), B, T, A, n, GAMMA, 0.9, eta,
                           dq.data_ptr(), prio.data_ptr(), stats.data_ptr(), scratch.data_ptr(), _s())
            qq = h(q).requires_grad_(True)
            L, td, p = orr.loss(qq, h(qn), h(qt), torch.from_numpy(act), h(rew), h(done), None if w is None else h(w),
                                GAMMA, n, eta, float(np.float32(0.9)))
            L.backward()
            st = stats.cpu().numpy()
            _close(dq.cpu(), qq.grad, 2e-6, f"dq eta={eta} w={wkind}")
            assert abs(st[0] - L.item()) <= 1e-6 * abs(L.item()) + 1e-30, (st[0], L.item())
            assert st[1] == q[np.arange(B)[:, None], np.arange(T)[None], act].max()
            np.testing.assert_allclose(prio.cpu().numpy(), p.numpy(), rtol=1e-12)


def test_loss_kernel_rejects_out_of_range_arguments():
    from jorldy_b200._lib import JbError
    C = _C()
    B, T, A, n = 2, 3, 4, 2
    t = [torch.zeros(B, T, 19, device=DEV) for _ in range(4)]
    act = torch.zeros(B, T, dtype=torch.int64, device=DEV)
    rd = torch.zeros(B, T + n, device=DEV)
    st, sc = torch.zeros(2, device=DEV), torch.zeros(2 * B, dtype=torch.float64, device=DEV)
    p = lambda x: x.data_ptr()

    def call(A=A, n=n, T=T, q=p(t[0])):
        return C.jb_r2d2_loss(q, p(t[1]), p(t[2]), p(act), p(rd), p(rd), 0, B, T, A, n, 0.99, 0.9, 0.9, p(t[3]), 0, p(st),
                              p(sc), _s())
    assert call() == 0
    for kw in (dict(A=19), dict(n=0), dict(T=0), dict(q=0)):
        with pytest.raises(JbError):
            call(**kw)


# ----------------------------------------------------------------------------------------------- 3. network
def _params(net):
    return {k: v.detach().cpu().clone() for k, v in net.p.items()}


def _net(head, D, A, H, seed=0):
    from jorldy_b200.core.network import Network
    net = Network("r2d2", D, A, D_hidden=H, head=head, device=DEV, seed=seed)
    with torch.no_grad():                    # non-zero biases, so a dropped bias gradient shows
        rs = np.random.RandomState(seed + 1)
        for k, v in net.p.items():
            if k.endswith("bias") or "bias_" in k:
                v.copy_(_dv((0.1 * rs.standard_normal(tuple(v.shape))).astype(np.float32)))
    return net


def _states(rs, head, D, shape):
    if head == "cnn":
        return rs.randint(0, 256, size=shape + (4, 84, 84)).astype(np.uint8)
    return rs.standard_normal(shape + (D,)).astype(np.float32)


def _rt(k, cnn):
    return 2e-2 if (cnn and k.startswith("head.")) else (2e-3 if cnn else 1e-3)


@pytest.mark.parametrize("head,H,A", [("mlp", 64, 2), ("mlp", 512, 2), ("cnn", 64, 18)])
def test_network_forward_and_backward_match_autograd(head, H, A):
    rs = np.random.RandomState(H + A)
    D = 4 if head == "mlp" else [4, 84, 84]
    B, S, g0 = (3, 7, 3) if head == "mlp" else (2, 5, 2)
    net = _net(head, D, A, H)
    x = _states(rs, head, D, (B, S))
    prev = rs.randint(-1, A, size=(B, S)).astype(np.int64)
    reset = (rs.uniform(size=(B, S)) < 0.3).astype(np.float32)
    reset[0, g0] = 1.0                                   # an episode start at the first trained step
    h0 = (0.5 * rs.standard_normal((B, H))).astype(np.float32)
    c0 = rs.standard_normal((B, H)).astype(np.float32)
    q = net.forward_seq(_dv(x.reshape(B * S, *x.shape[2:])), _dv(prev), _dv(reset), _dv(h0), _dv(c0), g0)
    dq = rs.standard_normal((B, S - g0, A)).astype(np.float32)
    net.backward_seq(_dv(dq))
    torch.cuda.synchronize()
    p = {k: v.to(torch.float64).requires_grad_(True) for k, v in _params(net).items()}
    x64 = torch.from_numpy(x).to(torch.float64)
    ref = orr.network(p, x64, torch.from_numpy(prev), torch.from_numpy(reset).double(), torch.from_numpy(h0).double(),
                      torch.from_numpy(c0).double(), g0, A)
    _close(q.cpu(), ref.detach(), 1e-4, "Q")
    (ref * torch.from_numpy(dq).double()).sum().backward()
    for k, v in p.items():
        _close(net.g[k].cpu(), v.grad, _rt(k, head == "cnn"), f"grad {k}", float(v.grad.abs().max()) + 1e-12)
    # the oracle detaches the state at the end of the burn-in, so matching every gradient shows nothing flows into it
    assert torch.equal(net.g["lstm.bias_hh_l0"], net.g["lstm.bias_ih_l0"])


# ------------------------------------------------------------------------------------------------- 4. learns
LEARN_CASES = {
    "mlp": dict(head="mlp", D=4, A=18, H=64, B=8, Tb=3, T=5, n=2),
    "cnn": dict(head="cnn", D=[4, 84, 84], A=18, H=64, B=4, Tb=2, T=3, n=2),
}
CAP = 32


def _agent(case, **kw):
    from jorldy_b200.core import Agent
    args = dict(state_size=case["D"], action_size=case["A"], hidden_size=case["H"], head=case["head"],
                batch_size=case["B"], seq_len=case["T"], n_burn_in=case["Tb"], n_step=case["n"], buffer_size=CAP,
                optim_config={"name": "adam", "lr": LR, "eps": 1e-3}, gamma=0.997, alpha=0.9, beta=0.6, eta=0.9,
                clip_grad_norm=40.0, run_step=1000, lr_decay=False, start_train_step=0, device=DEV, seed=0)
    args.update(kw)
    return Agent("r2d2", **args)


def _sequences(case, rs, n):
    L, A, H = case["Tb"] + case["T"] + case["n"], case["A"], case["H"]
    done = (rs.uniform(size=(n, L)) < 0.15).astype(np.float32)
    action = rs.randint(A, size=(n, L)).astype(np.int64)
    reset = np.concatenate([np.ones((n, 1), np.float32), done[:, :-1]], 1)
    prev = np.concatenate([np.full((n, 1), -1), action[:, :-1]], 1).astype(np.int64)
    prev[reset > 0] = -1
    return {"state": _states(rs, case["head"], case["D"], (n, L)), "action": action, "prev_action": prev, "reset": reset,
            "reward": rs.standard_normal((n, L)).astype(np.float32), "done": done,
            "h0": (0.3 * rs.standard_normal((n, H))).astype(np.float32), "c0": rs.standard_normal((n, H)).astype(np.float32)}


def _filled(case, rs, agent):
    tr = _sequences(case, rs, CAP)
    agent.memory.store([{k: _dv(v) for k, v in tr.items()}])
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
            v.add_(_dv(rs.standard_normal(tuple(v.shape)).astype(np.float32)) * 0.05)


@pytest.mark.parametrize("name", list(LEARN_CASES))
def test_eager_learn_matches_the_float64_oracle(name):
    case = LEARN_CASES[name]
    B = case["B"]
    rs = np.random.RandomState(5)
    agent = _agent(case)
    _perturb_target(agent, rs)
    tr, ora = _filled(case, rs, agent)
    u_a, u_b = rs.uniform(size=B), rs.uniform(size=B)
    u_a[0] = 1e-4
    idx, w, sampled_p, mean_p = ora.sample(agent.beta, u_a, u_b)
    rows = idx - ora.first_leaf
    batch = {k: torch.from_numpy(v[rows]) for k, v in tr.items()}
    pre, tgt = _params(agent.network), _params(agent.target_network)
    hp = dict(gamma=GAMMA, n_step=case["n"], n_burn_in=case["Tb"], seq_len=case["T"], eta=0.9, alpha=0.9, lr=LR, eps=1e-3,
              clip=40.0, A=case["A"])
    ref = orr.learn(pre, tgt, batch, torch.from_numpy(w), hp)
    agent._inject_u = (u_a, u_b)
    res = agent.learn()
    torch.cuda.synchronize()
    assert set(res) == {"loss", "max_Q", "sampled_p", "mean_p", "num_learn", "num_transitions"} and res["num_learn"] == 1
    for k, v in ref["result"].items():
        assert abs(res[k] - v) <= 5e-4 * max(abs(v), 1.0), (name, k, res[k], v)
    assert abs(res["sampled_p"] - sampled_p) <= 1e-12 * sampled_p and abs(res["mean_p"] - mean_p) <= 1e-12 * mean_p
    for i, p in zip(idx, ref["prio"].numpy()):
        ora.update(p, i)
    np.testing.assert_allclose(agent.memory.sum_tree[ora.first_leaf:], ora.tree[ora.first_leaf:], rtol=5e-4)
    cnn = case["head"] == "cnn"
    for k, g in ref["grads"].items():
        _close(agent.network.g[k].cpu(), g, _rt(k, cnn), f"grad {k}", float(g.abs().max()) + 1e-12)
    gs = {k: agent.network.g[k].cpu().to(torch.float64) for k in pre}
    norm = float(torch.sqrt(sum((g * g).sum() for g in gs.values())))
    coef = min(1.0, 40.0 / (norm + 1e-6))
    for k, p0 in pre.items():
        g = gs[k] * coef
        want = p0.to(torch.float64) - LR * g / (g.abs() + 1e-3)
        got = agent.network.p[k].cpu().to(torch.float64)
        assert (got - want).abs().max().item() <= 1e-3 * LR + 2 * U * p0.abs().max().item(), k


def test_two_learns_from_the_same_state_are_bit_identical():
    case = LEARN_CASES["mlp"]
    rs = np.random.RandomState(9)
    a, b = _agent(case), _agent(case)
    _perturb_target(a, rs)
    b.target_network.flat.copy_(a.target_network.flat)
    tr = {k: _dv(v) for k, v in _sequences(case, rs, CAP).items()}
    a.memory.store([tr]); b.memory.store([tr])
    for _ in range(3):
        a._inject_u = b._inject_u = (rs.uniform(size=case["B"]), rs.uniform(size=case["B"]))
        assert a.learn() == b.learn()
    torch.cuda.synchronize()
    assert torch.equal(a.network.flat, b.network.flat) and torch.equal(a.network.grad, b.network.grad)
    assert torch.equal(a.memory._tree, b.memory._tree)


# ---------------------------------------------------------------------------------------------------- 5. act
def test_act_steps_equal_one_unroll_and_follow_per_lane_epsilons():
    case = dict(LEARN_CASES["mlp"], A=3)
    agent = _agent(case)
    rs = np.random.RandomState(2)
    N, K, A, H = 6, 9, case["A"], case["H"]
    states = rs.standard_normal((K, N, 4)).astype(np.float32)
    done = (rs.uniform(size=(K, N)) < 0.25).astype(np.float32)
    done[3] = 0
    done[3, 0] = 1                                     # one lane ends its episode: only that lane starts over
    qs, prev, reset = [], [], []
    for t in range(K):
        a, _ = agent.act_device(_dv(states[t]), training=False)
        qs.append(agent.network._buf("act.q", (N, A)).clone())
        prev.append(agent.step_inputs["prev_action"]); reset.append(agent.step_inputs["reset"])
        assert torch.equal(a, qs[-1].argmax(1))                     # training=False: greedy
        agent.end_step(_dv(done[t]))
    assert torch.equal(reset[4].cpu(), torch.tensor([1.0] + [0.0] * (N - 1)))
    assert prev[4][0].item() == -1 and (prev[4][1:] >= 0).all()
    x = _dv(states.transpose(1, 0, 2).reshape(N * K, 4))
    z = torch.zeros(N, H, device=DEV)
    q_seq = agent.network.forward_seq(x, torch.stack(prev, 1), torch.stack(reset, 1), z, z, 0, tag="seq.")
    _close(torch.stack(qs, 1).cpu(), q_seq.cpu(), 1e-5, "step-by-step act vs one unroll")
    # per-lane epsilons: lanes at epsilon 0 act greedily, lanes at epsilon 1 uniformly
    agent._eps_rows = _dv(np.array([0.0, 1.0] * (N // 2), np.float32))
    greedy_hits = np.zeros(N)
    for t in range(60):
        a, _ = agent.act_device(_dv(states[t % K]), training=True)
        greedy_hits += (a == agent.network._buf("act.q", (N, A)).argmax(1)).cpu().numpy()
        agent.end_step(torch.zeros(N, device=DEV))
    assert (greedy_hits[0::2] == 60).all() and (greedy_hits[1::2] < 60).all()


# ---------------------------------------------------------------------------------------------- 6. assembler
def test_collector_sequences_carry_the_actor_state_of_their_first_step(monkeypatch):
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    case = dict(LEARN_CASES["mlp"], A=2)
    agent = _agent(case, start_train_step=10 ** 9)
    env = Env("cartpole", num_envs=4, seed=1, device=DEV)
    snaps, acts, dones, emitted = [], [], [], []
    act0, end0, proc0 = agent.act_device, agent.end_step, agent.process

    def act(state, training=True, noise=None):
        ln = agent._lanes
        snaps.append(None if ln is None else (ln["h"].clone(), ln["c"].clone()))
        a, q = act0(state, training, noise)
        acts.append(a.clone())
        return a, q

    def end(done):
        dones.append(done.clone())
        end0(done)

    def proc(batches, step):
        emitted.extend(batches)
        return proc0(batches, step)
    monkeypatch.setattr(agent, "act_device", act)
    monkeypatch.setattr(agent, "end_step", end)
    monkeypatch.setattr(agent, "process", proc)
    rc = ReplayCollector(env, agent, update_period=16)
    step = 0
    for _ in range(6):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    L, P = agent.L, agent.store_period
    assert len(emitted) == (6 * 16 - L) // P + 1 and float(torch.cat(dones).sum()) > 0
    for k, out in enumerate(emitted):
        s0 = k * P
        snap = snaps[s0] or (torch.zeros(4, case["H"], device=DEV),) * 2
        assert torch.equal(out["h0"], snap[0]) and torch.equal(out["c0"], snap[1])
        assert torch.equal(out["action"], torch.stack(acts[s0:s0 + L], 1))
        assert torch.equal(out["done"], torch.stack(dones[s0:s0 + L], 1))
        want_reset = torch.stack([torch.ones(4, device=DEV) if s == 0 else dones[s - 1] for s in range(s0, s0 + L)], 1)
        assert torch.equal(out["reset"], want_reset)


# ------------------------------------------------------------------------------------------------- 7. frames
def test_frame_replay_learn_equals_the_stacked_twin_and_eviction_raises():
    from jorldy_b200.core import Env
    from jorldy_b200.core.buffer.frame_store import FrameEvictedError
    from jorldy_b200.core.collect import ReplayCollector
    case = dict(LEARN_CASES["cnn"], B=4)
    agent = _agent(case, buffer_size=64, start_train_step=10 ** 9)
    env = Env("seaquest", num_envs=4, seed=2, device=DEV)
    rc = ReplayCollector(env, agent, update_period=8)
    step = 0
    for _ in range(5):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    mem = agent.memory
    assert rc.frames is agent._frames and mem.frames is None and mem.size > 0
    refs = mem.fields["state"][:mem.size]
    n, L = refs.shape
    st, _ = agent._frames.gather(refs.reshape(-1), refs.reshape(-1))
    agent._frames.check()
    twin = _agent(case, buffer_size=64)
    twin.network.flat.copy_(agent.network.flat)
    twin.target_network.flat.copy_(agent.target_network.flat)
    stacked = {k: v[:mem.size] for k, v in mem.fields.items()}
    stacked["state"] = st.view(n, L, 4, 84, 84)
    twin.memory.store([stacked])
    twin.memory._tree.copy_(mem._tree)
    twin.memory._max_priority.copy_(mem._max_priority)
    twin.beta, twin.num_transitions = agent.beta, agent.num_transitions
    rs = np.random.RandomState(4)
    for _ in range(2):
        agent._inject_u = twin._inject_u = (rs.uniform(size=case["B"]), rs.uniform(size=case["B"]))
        assert agent.learn() == twin.learn()
    torch.cuda.synchronize()
    assert torch.equal(agent.network.flat, twin.network.flat) and torch.equal(mem._tree, twin.memory._tree)
    old = refs.clone()
    newest = int((old[0] & ((1 << 40) - 1)).max())
    while int(agent._frames.head.min()) <= newest + agent._frames.F:     # until every lane has overwritten those frames
        step, _ = rc.run_round(step)
    mem.fields["state"][:mem.size] = old[:1].expand(mem.size, L)
    agent._inject_u = (rs.uniform(size=case["B"]), rs.uniform(size=case["B"]))
    with pytest.raises(FrameEvictedError):
        agent.learn()


# -------------------------------------------------------------------------------------------- 8. checkpoints
def test_checkpoint_keys_and_round_trip(tmp_path):
    case = dict(LEARN_CASES["mlp"], A=2, B=2)
    a = _agent(case, start_train_step=1, learn_period=1)
    rs = np.random.RandomState(1)
    state = rs.standard_normal((1, 4)).astype(np.float32)
    for step in range(1, 40):
        ns = rs.standard_normal((1, 4)).astype(np.float32)
        tr = {"state": state, "next_state": ns, "reward": np.ones(1), "done": np.array([step % 13 == 0])}
        tr.update(a.act(state, True))
        tr = a.interact_callback(tr)
        if tr:
            a.process([tr], step)
        state = ns
    assert a.num_learn > 0
    a.save(str(tmp_path))
    ck = torch.load(str(tmp_path / "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "optimizer"}
    assert list(ck["network"]) == ["head.l.weight", "head.l.bias", "lstm.weight_ih_l0", "lstm.weight_hh_l0",
                                   "lstm.bias_ih_l0", "lstm.bias_hh_l0", "l1_a.weight", "l1_a.bias", "l1_v.weight",
                                   "l1_v.bias", "l2_a.weight", "l2_a.bias", "l2_v.weight", "l2_v.bias"]
    H = case["H"]
    assert tuple(ck["network"]["lstm.weight_ih_l0"].shape) == (4 * H, H + 2)
    b = _agent(case, seed=9)
    assert not torch.equal(b.network.flat, a.network.flat)
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, a.network.flat) and torch.equal(b.target_network.flat, a.network.flat)
    assert torch.equal(b.optimizer.exp_avg, a.optimizer.exp_avg)


# -------------------------------------------------------------------------------------------------- 9. end to end
@pytest.mark.parametrize("config,extra,sizes", [
    ("config.r2d2.cartpole", ["--train.num_workers", "8", "--agent.start_train_step", "64",
                              "--train.distributed_batch_size", "32"], (4, 2)),
    ("config.r2d2.atari", ["--env.name", "seaquest", "--train.num_workers", "8", "--agent.start_train_step", "16",
                           "--agent.buffer_size", "512", "--agent.hidden_size", "64", "--agent.batch_size", "8",
                           "--agent.seq_len", "8", "--agent.n_burn_in", "4", "--train.update_period", "16"],
     ([4, 84, 84], 18)),
])
def test_sync_training_run(tmp_path, config, extra, sizes):
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
    from jorldy_b200 import config as cfg
    D, A = sizes
    kw = dict(head="cnn", hidden_size=64) if config.endswith("atari") else {}
    fresh = Agent("r2d2", state_size=D, action_size=A, device=DEV, optim_config=cfg.load(config).optim, **kw)
    fresh.load(ckpts[0])
    for k, v in fresh.network.state_dict().items():
        assert torch.equal(v.cpu(), saved["network"][k]), k
