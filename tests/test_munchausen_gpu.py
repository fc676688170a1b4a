"""M-DQN and M-IQN on the GPU (csrc/munchausen.cuh, jb_mdqn_loss in csrc/dqn.cu, jb_munchausen_quantile_loss in
csrc/quantile.cu, core/agent/munchausen.py) against the float64 oracle (oracle/munchausen.py), against jb_td_loss and
jb_quantile_loss in the alpha = 0, tau -> 0 limit, and through the replay layouts and the run loop (pytest -m gpu).

Tolerances.  u = 2^-24 is fp32's unit roundoff; S_b = 1 + |r_b| + the largest |value| of sample b's target rows.
- Targets.  tau logpi(a_t|s) takes one rounding for q(a_t) - m and a log of a sum of A <= 18 exponentials.  Terms that
  matter (exp(x) > u) have |x| < 17, so each carries a relative error of at most (2 |x| + 2) u < 36 u and the sum < 54 u;
  times tau that is far below u S_b.  The bonus is 1-Lipschitz in tau logpi.  V' = sum_a pi'(a) (q'(s',a) - tau logpi'(a))
  has weights with relative error < 60 u and values with 3 roundings each.  So |dy| <= 128 u S_b: the per-sample bound
  tol_b.  M-IQN's q' are warp means (at most 8 sequential adds, 5 butterfly levels and a division): error
  e_b <= 16 u max|theta'|.  The bonus moves by at most 2 e_b.  pi' moves by up to 2 pi' e_b / tau per action, and V'_j by
  that times max_{a,j} |theta'_j(s',a) - q'(s',a)| (D_b); tau logpi'(a) moves by at most 2 e_b.  So M-IQN adds
  2 e_b + (1 - d) gamma (2 e_b + 2 e_b D_b / tau) to tol_b.
  Rows whose spread makes exp underflow have a one-hot pi' in both precisions, so the bound holds there too.
- Loss and gradient (1).  smooth_l1 and the quantile Huber are 1-Lipschitz in y with weights <= 1.  So a gradient element
  moves by at most tol_b / B (+ N' u / B for the sum over j), and M-IQN's per-sample loss by N tol_b + (N' + 13) u
  loss_b.  The batch loss adds B u of the sum.  max_Q is a selection (M-DQN: exact) or a warp mean (M-IQN: 16 u
  max|theta|).  The mutations the suite is meant to catch move the bonus or V' by 0.045 (clip order) up to O(1) on
  most samples, 10^2..10^4 times these bounds.
- Reduction (2).  At alpha = 0 and tau = 1e-7 with maxima >= 0.01 apart, every exponential but the max's underflows to 0,
  so pi' is exactly one-hot, tau logpi'(a*) is exactly 0 and the bonus is +-0: y is bit-identical to jb_td_loss's and
  jb_quantile_loss's, and so are dq / dpred.  The batch loss is folded in another order (a warp tree in jb_td_loss):
  B u relative.
- One learn (3): as test_quantile_gpu.py: gradients normwise per tensor at 1e-3 (MLP), 2e-3 (CNN outside the trunk),
  2e-2 for the conv trunk and for M-IQN's sample_embed on the CNN head; loss and max_Q at rtol 5e-4; parameters against
  a float64 Adam step on the kernel's own gradients, bound 1e-3 lr + 2 u |p|.  M-IQN's pi' amplifies the forward's
  rounding in q' by 1/tau (above); at init the quantile spreads D_b are ~0.1, which keeps it below 1e-4 of y.
- Repeated learns (4), frames vs stacks (6) and checkpoints (7) are bit-exact.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import munchausen as om
from oracle import nets
from oracle import quantile as oq

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
GAMMA = float(np.float32(0.99))
ALPHA, MTAU, L0 = 0.9, 0.03, -1.0
ALPHA32, MTAU32 = float(np.float32(ALPHA)), float(np.float32(MTAU))


def _close(got, ref, R, what, scale=None):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = max(float(np.abs(ref).max()), 1e-30) if scale is None else scale
    err = float(np.abs(got - ref).max())
    assert err <= R * scale, f"{what}: max |err| {err:.3e} > {R} * {scale:.3e}"


def _dv(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _h(x):
    return torch.from_numpy(np.asarray(x)).to(torch.float64)


def _current_rows(rs, B, A):
    """q'(s, .) whose taken action sits, by b % 4, at the argmax (tau logpi ~ 0), 0.5 below the max (above l_0), 1.05
    below (between l_0 / alpha and l_0: clip-then-scale gives -0.9, scale-then-clip -0.945) and 3 below (under l_0 / alpha);
    every fifth row also has an action 1000 below, whose exponential underflows."""
    a_t = rs.randint(A, size=B)
    base = rs.standard_normal(B)
    q = base[:, None] + rs.uniform(-3.0, -2.0, size=(B, A))
    ar = np.arange(B)
    if A > 1:
        a_m = (a_t + 1 + rs.randint(A - 1, size=B)) % A
        q[ar, a_m] = base
        q[ar, a_t] = base + np.array([0.2, -0.5, -1.05, -3.0])[ar % 4]
        far = (ar % 5 == 4) & (A > 2)
        a_f = (a_m + 1) % A
        a_f = np.where(a_f == a_t, (a_f + 1) % A, a_f)
        q[ar[far], a_f[far]] = base[far] - 1000.0
    return q, a_t


def _next_rows(rs, B, A):
    """q'(s', .): every third row has a tie at its max, every fifth a spread of ~1000 (exp underflows)."""
    q = 2.0 * rs.standard_normal((B, A))
    ar = np.arange(B)
    if A > 1:
        top = q.argmax(1)
        tie = ar % 3 == 0
        q[ar[tie], ((top + 1) % A)[tie]] = q[ar[tie], top[tie]]
    q[ar % 5 == 4] *= 500.0
    return q, ar % 3 == 0


# ----------------------------------------------------------------------------------------- 1. kernels vs the oracle
def _mdqn(B, A, d, seed, alpha=ALPHA, tau=MTAU, q=None, qs=None, qn=None, a_t=None):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(seed)
    if qs is None:
        qs, a_t = _current_rows(rs, B, A)
        qn, _ = _next_rows(rs, B, A)
    qs, qn = qs.astype(np.float32), qn.astype(np.float32)
    reward = rs.standard_normal(B).astype(np.float32)
    done = np.full(B, float(d), np.float32)
    y = om.mdqn_target(_h(qs), _h(qn), torch.from_numpy(a_t), _h(reward), _h(done), GAMMA, float(np.float32(alpha)),
                       float(np.float32(tau)), L0).numpy()
    if q is None:
        q = rs.standard_normal((B, A))
        q[np.arange(B), a_t] = y + rs.uniform(-1.5, 1.5, size=B)          # both branches of smooth_l1
    q = q.astype(np.float32)
    dq = torch.full((B, A), float("nan"), device=DEV)
    stats = torch.full((4,), float("nan"), device=DEV)
    scratch = torch.empty(2 * B, device=DEV)
    g = {k: _dv(v) for k, v in dict(q=q, qs=qs, qn=qn, a=a_t.astype(np.int64), r=reward, d=done).items()}
    C.jb_mdqn_loss(ptr(g["q"]), ptr(g["qs"]), ptr(g["qn"]), ptr(g["a"]), 0, ptr(g["r"]), ptr(g["d"]), B, A, GAMMA, alpha,
                   tau, L0, ptr(dq), ptr(stats), ptr(scratch), stream_ptr())
    torch.cuda.synchronize()
    return dict(q=q, qs=qs, qn=qn, a_t=a_t, reward=reward, done=done, y=y, dq=dq.cpu().numpy(), stats=stats.cpu().numpy(),
                g=g)


@pytest.mark.parametrize("A", [2, 18])
@pytest.mark.parametrize("B", [1, 32, 257])
@pytest.mark.parametrize("d", [0, 1])
def test_mdqn_kernel_matches_the_oracle(A, B, d):
    o = _mdqn(B, A, d, seed=A * 7 + B + d)
    assert np.isfinite(o["dq"]).all() and np.isfinite(o["stats"][:2]).all()
    S = 1 + np.abs(o["reward"]) + np.abs(o["qs"]).max(1) + np.abs(o["qn"]).max(1)
    tol = 128 * U * S
    ar = np.arange(B)
    diff = _h(o["q"][ar, o["a_t"]]) - _h(o["y"])
    per = torch.nn.functional.smooth_l1_loss(_h(o["q"][ar, o["a_t"]]), _h(o["y"]), reduction="none").numpy()
    want = np.zeros((B, A))
    want[ar, o["a_t"]] = diff.clamp(-1, 1).numpy() / B
    err = np.abs(o["dq"] - want).max(1)
    assert (err <= tol / B + 2 * U / B).all(), f"dq: worst row {err.argmax()} err {err.max():.3e}"
    mask = np.ones((B, A), bool)
    mask[ar, o["a_t"]] = False
    assert np.all(o["dq"][mask] == 0.0)
    assert abs(o["stats"][0] - per.mean()) <= tol.mean() + B * U * per.mean() + 1e-30
    assert o["stats"][1] == o["q"][ar, o["a_t"]].max()


def _cur_quantiles(rs, qs, n):
    noise = 0.5 * rs.standard_normal(qs.shape + (n,))
    return qs[..., None] + (noise - noise.mean(2, keepdims=True))           # per-action means stay on qs


def _next_quantiles(rs, qn, tie, n):
    th = qn[..., None] + np.clip(rs.standard_normal(qn.shape + (n,)), -3, 3)
    B, A = qn.shape
    if A > 1:                                                                # a tie of the means: identical columns
        top = qn.argmax(1)
        for b in np.nonzero(tie)[0]:
            th[b, (top[b] + 1) % A] = th[b, top[b]]
    return th


def _miqn(B, A, N, Np, Nc, d, seed, alpha=ALPHA, tau=MTAU):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(seed)
    qs, a_t = _current_rows(rs, B, A)
    qn, tie = _next_rows(rs, B, A)
    cur = _cur_quantiles(rs, qs, Nc).astype(np.float32)                   # [B, A, n] logical
    nxt = _next_quantiles(rs, qn, tie, Np).astype(np.float32)
    reward = rs.standard_normal(B).astype(np.float32)
    done = np.full(B, float(d), np.float32)
    fr = rs.uniform(size=(B, N)).astype(np.float32)
    y = om.miqn_targets(_h(cur), _h(nxt), torch.from_numpy(a_t), _h(reward), _h(done), GAMMA, float(np.float32(alpha)),
                        float(np.float32(tau)), L0)
    pred = np.clip(2.0 * rs.standard_normal((B, A, N)), -8, 8)
    pred[np.arange(B), a_t] = y.mean(1).numpy()[:, None] + 1.5 * rs.standard_normal((B, N))
    pred = pred.astype(np.float32)
    dpred = torch.full((B, N, A), float("nan"), device=DEV)
    stats = torch.full((4,), float("nan"), device=DEV)
    scratch = torch.empty(2 * B, device=DEV)
    g = {k: _dv(v) for k, v in dict(p=pred.transpose(0, 2, 1), n=nxt.transpose(0, 2, 1), c=cur.transpose(0, 2, 1),
                                     t=fr, a=a_t.astype(np.int64), r=reward, d=done).items()}
    C.jb_munchausen_quantile_loss(ptr(g["p"]), ptr(g["n"]), ptr(g["c"]), ptr(g["t"]), N, ptr(g["a"]), 0, ptr(g["r"]),
                                  ptr(g["d"]), B, A, N, Np, Nc, GAMMA, alpha, tau, L0, ptr(dpred), ptr(stats), ptr(scratch),
                                  stream_ptr())
    torch.cuda.synchronize()
    return dict(pred=pred, cur=cur, nxt=nxt, a_t=a_t, reward=reward, done=done, fr=fr, y=y,
                dpred=dpred.cpu().numpy().transpose(0, 2, 1), stats=stats.cpu().numpy(), g=g)


@pytest.mark.parametrize("N,Np,Nc", [(1, 1, 1), (64, 64, 64), (32, 8, 17), (200, 256, 3)])
@pytest.mark.parametrize("A", [2, 18])
@pytest.mark.parametrize("B", [1, 32, 257])
@pytest.mark.parametrize("d", [0, 1])
def test_miqn_kernel_matches_the_oracle(N, Np, Nc, A, B, d):
    o = _miqn(B, A, N, Np, Nc, d, seed=N + Np * 3 + Nc * 5 + A * 7 + B + d)
    assert np.isfinite(o["dpred"]).all() and np.isfinite(o["stats"][:2]).all()
    ar = np.arange(B)
    cur, nxt = _h(o["cur"]), _h(o["nxt"])
    S = 1 + np.abs(o["reward"]) + np.abs(o["cur"]).reshape(B, -1).max(1) + np.abs(o["nxt"]).reshape(B, -1).max(1)
    e = 16 * U * np.abs(o["nxt"]).reshape(B, -1).max(1) + 16 * U * np.abs(o["cur"]).reshape(B, -1).max(1)
    D = (nxt - nxt.mean(2, keepdim=True)).abs().reshape(B, -1).max(1).values.numpy()
    tol = 128 * U * S + 2 * e + (1 - o["done"]) * GAMMA * (2 * e + 2 * e * D / MTAU32)
    theta = _h(o["pred"])[torch.arange(B), torch.from_numpy(o["a_t"])]
    tau = _h(o["fr"])
    per = oq.per_sample_loss(theta, o["y"], tau).numpy()
    want = np.zeros((B, A, N))
    want[ar, o["a_t"]] = oq.grad_closed(theta, o["y"], tau).numpy()
    err = np.abs(o["dpred"] - want).reshape(B, -1).max(1)
    assert (err <= (tol + Np * U) / B).all(), f"dpred: worst row {err.argmax()} err {err.max():.3e}"
    mask = np.ones((B, A), bool)
    mask[ar, o["a_t"]] = False
    assert np.all(o["dpred"][mask] == 0.0)
    loss_tol = (N * tol + (Np + 13) * U * per).mean() + B * U * per.mean()
    assert abs(o["stats"][0] - per.mean()) <= loss_tol, (o["stats"][0], per.mean(), loss_tol)
    _close(o["stats"][1], _h(o["pred"]).mean(2).max().item(), 16 * U, "max_Q", float(np.abs(o["pred"]).max()))


def test_the_inputs_reach_every_clip_region():
    """The rows _current_rows builds put tau logpi(a_t|s) above l_0, between l_0 / alpha and l_0, and below l_0 / alpha."""
    rs = np.random.RandomState(0)
    qs, a_t = _current_rows(rs, 64, 18)
    t = om.tau_logpi(_h(qs), MTAU)[torch.arange(64), torch.from_numpy(a_t)].numpy()
    assert (t > L0).any() and ((t < L0) & (t > L0 / ALPHA)).any() and (t < L0 / ALPHA).any()
    assert np.all((np.abs(t - L0) > 0.04) & (np.abs(t - L0 / ALPHA) > 0.04))


def test_kernels_reject_out_of_range_arguments():
    from jorldy_b200._lib import JbError
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    B = 2
    x = torch.zeros(B * 19 * 257, device=DEV)
    a = torch.zeros(B, dtype=torch.int64, device=DEV)
    small = torch.zeros(8, device=DEV)
    out = torch.zeros(B * 19 * 257, device=DEV)
    for A, tau, l0 in ((19, MTAU, L0), (2, 0.0, L0), (2, -1.0, L0), (2, float("nan"), L0), (2, MTAU, 0.5)):
        with pytest.raises(JbError):
            C.jb_mdqn_loss(ptr(x), ptr(x), ptr(x), ptr(a), 0, ptr(small), ptr(small), B, A, GAMMA, ALPHA, tau, l0, ptr(out),
                           ptr(small), ptr(small), stream_ptr())
    with pytest.raises(JbError):
        C.jb_mdqn_loss(ptr(x), None, ptr(x), ptr(a), 0, ptr(small), ptr(small), B, 2, GAMMA, ALPHA, MTAU, L0, ptr(out),
                       ptr(small), ptr(small), stream_ptr())
    for A, N, Np, Nc, tau, l0 in ((19, 8, 8, 8, MTAU, L0), (2, 257, 8, 8, MTAU, L0), (2, 8, 257, 8, MTAU, L0),
                                  (2, 8, 8, 257, MTAU, L0), (2, 8, 8, 0, MTAU, L0), (2, 8, 8, 8, 0.0, L0),
                                  (2, 8, 8, 8, -0.03, L0), (2, 8, 8, 8, MTAU, 0.5)):
        with pytest.raises(JbError):
            C.jb_munchausen_quantile_loss(ptr(x), ptr(x), ptr(x), ptr(small), 0, ptr(a), 0, ptr(small), ptr(small), B, A, N,
                                          Np, Nc, GAMMA, ALPHA, tau, l0, ptr(out), ptr(small), ptr(small), stream_ptr())
    with pytest.raises(JbError):
        C.jb_munchausen_quantile_loss(ptr(x), ptr(x), None, ptr(small), 0, ptr(a), 0, ptr(small), ptr(small), B, 2, 8, 8, 8,
                                      GAMMA, ALPHA, MTAU, L0, ptr(out), ptr(small), ptr(small), stream_ptr())


# ------------------------------------------------------------------------- 2. alpha = 0, tau -> 0: DQN's and IQN's loss
def _separated(rs, B, A, scale=2.0):
    q = scale * rs.standard_normal((B, A))
    top = q.argmax(1)
    q[np.arange(B), top] = q.max(1) + 0.01 + rs.uniform(size=B)
    return q


@pytest.mark.parametrize("A", [2, 18])
@pytest.mark.parametrize("B", [1, 32, 257])
@pytest.mark.parametrize("d", [0, 1])
def test_mdqn_reduces_to_td_loss(A, B, d):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(100 + A + B + d)
    qs, qn = 2.0 * rs.standard_normal((B, A)), _separated(rs, B, A)
    a_t = rs.randint(A, size=B)
    q = 2.0 * rs.standard_normal((B, A))
    o = _mdqn(B, A, d, 0, alpha=0.0, tau=1e-7, q=q, qs=qs, qn=qn, a_t=a_t)
    g = o["g"]
    dq = torch.full((B, A), float("nan"), device=DEV)
    stats = torch.full((4,), float("nan"), device=DEV)
    C.jb_td_loss(ptr(g["q"]), None, ptr(g["qn"]), ptr(g["a"]), 0, ptr(g["r"]), ptr(g["d"]), None, B, A, GAMMA, 0.0, 1, 0,
                 0, 0, ptr(dq), None, ptr(stats), stream_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(o["dq"], dq.cpu().numpy())
    st = stats.cpu().numpy()
    assert abs(o["stats"][0] - st[0]) <= B * U * abs(st[0]) and o["stats"][1] == st[1]


@pytest.mark.parametrize("N,Np,Nc", [(1, 1, 1), (64, 64, 64), (32, 8, 17)])
@pytest.mark.parametrize("A", [2, 18])
@pytest.mark.parametrize("B", [1, 32, 257])
def test_miqn_reduces_to_quantile_loss(N, Np, Nc, A, B):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(200 + N + Np + Nc + A + B)
    qn = _separated(rs, B, A)
    nxt = (qn[..., None] + 0.5 * rs.standard_normal((B, A, Np)))
    nxt = nxt - nxt.mean(2, keepdims=True) + qn[..., None]                   # means stay >= 0.01 apart in fp32
    nxt = nxt.astype(np.float32).transpose(0, 2, 1)
    cur = rs.standard_normal((B, Nc, A)).astype(np.float32)
    pred = (2.0 * rs.standard_normal((B, N, A))).astype(np.float32)
    fr = rs.uniform(size=(B, N)).astype(np.float32)
    a_t = rs.randint(A, size=B).astype(np.int64)
    reward = rs.standard_normal(B).astype(np.float32)
    done = (rs.uniform(size=B) < 0.3).astype(np.float32)
    g = {k: _dv(v) for k, v in dict(p=pred, n=nxt, c=cur, t=fr, a=a_t, r=reward, d=done).items()}
    dm, dq = (torch.full((B, N, A), float("nan"), device=DEV) for _ in range(2))
    sm, sq = (torch.full((4,), float("nan"), device=DEV) for _ in range(2))
    scratch = torch.empty(2 * B, device=DEV)
    loss = torch.empty(B, device=DEV)
    C.jb_munchausen_quantile_loss(ptr(g["p"]), ptr(g["n"]), ptr(g["c"]), ptr(g["t"]), N, ptr(g["a"]), 0, ptr(g["r"]),
                                  ptr(g["d"]), B, A, N, Np, Nc, GAMMA, 0.0, 1e-7, L0, ptr(dm), ptr(sm), ptr(scratch),
                                  stream_ptr())
    C.jb_quantile_loss(ptr(g["p"]), 1, A, ptr(g["n"]), 1, A, ptr(g["t"]), N, ptr(g["a"]), 0, ptr(g["r"]), ptr(g["d"]), B,
                       A, N, Np, GAMMA, ptr(dq), ptr(loss), None, ptr(sq), ptr(scratch), stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(dm, dq)
    a, b = sm.cpu().numpy(), sq.cpu().numpy()
    assert abs(a[0] - b[0]) <= B * U * abs(b[0]) and a[1] == b[1]


# ----------------------------------------------------------------------------------- 3. one eager learn vs oracle
CAP = 64
LR = 1e-3
LEARN_CASES = {
    "m_dqn_mlp_h64": dict(agent="m_dqn", head="mlp", D=4, A=2, H=64, B=16),
    "m_dqn_mlp_h512": dict(agent="m_dqn", head="mlp", D=4, A=2, H=512, B=32),
    "m_dqn_cnn": dict(agent="m_dqn", head="cnn", D=[4, 84, 84], A=18, H=512, B=32),
    "m_iqn_mlp": dict(agent="m_iqn", head="mlp", D=4, A=2, H=64, B=16, N=16),
    "m_iqn_cnn": dict(agent="m_iqn", head="cnn", D=[4, 84, 84], A=18, H=512, B=32, N=64),
}


def _agent(case, seed=0, buffer_size=CAP, **extra):
    from jorldy_b200.core import Agent
    torch.manual_seed(seed)
    kw = dict(state_size=case["D"], action_size=case["A"], hidden_size=case["H"], head=case["head"],
              optim_config={"name": "adam", "lr": LR}, gamma=0.99, buffer_size=buffer_size, batch_size=case["B"],
              run_step=1000, lr_decay=False, device=DEV, seed=seed, alpha=ALPHA, tau=MTAU, l_0=L0)
    if case["agent"] == "m_iqn":
        kw.update(num_sample=case["N"])
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
    """A target net that differs from the online one, so that the bonus, pi' and y depend on which net produced them."""
    with torch.no_grad():
        for k, v in agent.target_network.p.items():
            v.add_(torch.from_numpy(rs.standard_normal(tuple(v.shape)).astype(np.float32)).to(DEV) * 0.05)


@pytest.mark.parametrize("name", list(LEARN_CASES))
def test_eager_learn_matches_the_float64_oracle(name):
    case = LEARN_CASES[name]
    rs = np.random.RandomState(5)
    agent = _agent(case)
    assert (agent.m_alpha, agent.m_tau, agent.m_l0, agent.alpha) == (ALPHA, MTAU, L0, 0.0)
    _perturb_target(agent, rs)
    tr = _replay(case, rs)
    agent.memory.store([tr])
    idx = rs.randint(CAP, size=case["B"])
    batch = {"state": torch.from_numpy(tr["state"][idx]), "next_state": torch.from_numpy(tr["next_state"][idx]),
             "action": torch.from_numpy(tr["action"][idx, 0]),
             "reward": torch.from_numpy(tr["reward"][idx, 0].astype(np.float32)),
             "done": torch.from_numpy(tr["done"][idx, 0].astype(np.float32))}
    pre, tgt = _params(agent.network), _params(agent.target_network)
    hp = dict(gamma=GAMMA, lr=LR, alpha=ALPHA32, tau=MTAU32, l_0=L0)
    if case["agent"] == "m_dqn":
        ref = om.mdqn_learn(pre, tgt, batch, hp)
    else:
        B, N = case["B"], case["N"]
        taus = [rs.uniform(size=(B, N)).astype(np.float32) for _ in range(3)]
        agent._inject_tau = [taus[0], taus[1], None, taus[2]]
        ref = om.miqn_learn(pre, tgt, batch, *(torch.from_numpy(t) for t in taus), dict(hp, D_em=64))
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
@pytest.mark.parametrize("agent_name", ["m_dqn", "m_iqn"])
def test_two_learns_from_the_same_state_are_bit_identical(agent_name):
    case = dict(LEARN_CASES[agent_name + "_" + ("mlp_h64" if agent_name == "m_dqn" else "mlp")])
    rs = np.random.RandomState(9)
    a, b = _agent(case), _agent(case)
    _perturb_target(a, rs)
    b.network.flat.copy_(a.network.flat)
    b.target_network.flat.copy_(a.target_network.flat)
    tr = _replay(case, rs)
    a.memory.store([tr]); b.memory.store([tr])
    for _ in range(3):
        a._inject_idx = b._inject_idx = rs.randint(CAP, size=case["B"])
        ra, rb = a.learn(), b.learn()                  # M-IQN: the same seed and counter give the same three draws
        assert ra == rb
    torch.cuda.synchronize()
    assert torch.equal(a.network.flat, b.network.flat)
    if agent_name == "m_iqn":
        assert a._tau_ctr.item() == b._tau_ctr.item() == 3 * 3 * ((case["B"] * case["N"] + 3) // 4)


# ------------------------------------------------------------------------------------------------------- 5. act
@pytest.mark.parametrize("agent_name", ["m_dqn", "m_iqn"])
def test_act_greedy_and_epsilon_paths(agent_name):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    case = dict(LEARN_CASES[agent_name + "_" + ("mlp_h64" if agent_name == "m_dqn" else "mlp")], A=18)
    agent = _agent(case)
    rs = np.random.RandomState(3)
    M = 2048
    s = torch.from_numpy(rs.standard_normal((M, 4)).astype(np.float32)).to(DEV)
    params = _params(agent.network)
    if agent_name == "m_iqn":
        tau = rs.uniform(size=(M, case["N"])).astype(np.float32)
        agent._inject_tau = [None, None, tau, None]
        ref = oq.iqn_q(params, s.cpu(), torch.from_numpy(tau), 64)
    else:
        ref = nets.discrete_q_network(params, s.cpu().to(torch.float64))
    greedy = agent.act_device(s, training=False)[0].clone()
    top2 = torch.topk(ref, 2, dim=1).values
    bad = (greedy.cpu() != ref.argmax(1)) & ((top2[:, 0] - top2[:, 1]) > 1e-5)
    assert not bad.any()
    q = agent.network._buf("act.q", (M, case["A"])).cpu().to(torch.float64)
    _close(q.numpy(), ref.numpy(), 1e-4, "act Q", float(ref.abs().max()))
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
    if agent_name == "m_iqn":
        agent._inject_tau = None
    out = agent.act(s[:5].cpu().numpy(), training=False)["action"]
    assert out.dtype == np.int64 and out.shape == (5, 1)


# ---------------------------------------------------------------------------------------------------- 6. frames
N_LANES, PERIOD, ROUNDS = 4, 8, 6


@pytest.mark.parametrize("agent_name", ["m_dqn", "m_iqn"])
def test_frame_replay_learn_equals_the_stacked_twin(agent_name):
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    case = dict(agent=agent_name, head="cnn", D=[4, 84, 84], A=18, H=64, B=16, N=8)
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
    if agent_name == "m_iqn":
        twin._tau_ctr.copy_(agent._tau_ctr)
    rs = np.random.RandomState(4)
    for _ in range(3):
        agent._inject_idx = twin._inject_idx = rs.randint(mem.size, size=case["B"])
        assert agent.learn() == twin.learn()
    torch.cuda.synchronize()
    assert torch.equal(agent.network.flat, twin.network.flat)


# ------------------------------------------------------------------------------------------------ 7. checkpoints
@pytest.mark.parametrize("agent_name", ["m_dqn", "m_iqn"])
def test_checkpoint_keys_and_round_trip(tmp_path, agent_name):
    case = dict(LEARN_CASES[agent_name + "_" + ("mlp_h64" if agent_name == "m_dqn" else "mlp")], H=32, B=4)
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
    if agent_name == "m_dqn":
        assert list(ck["network"]) == ["head.l.weight", "head.l.bias", "l.weight", "l.bias", "q.weight", "q.bias"]
        assert tuple(ck["network"]["q.weight"].shape) == (2, 32)
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
    ("config.m_dqn.cartpole", ["--train.num_workers", "8", "--agent.start_train_step", "64"], (4, 2)),
    ("config.m_iqn.atari", ["--env.name", "seaquest", "--train.num_workers", "8", "--agent.start_train_step", "16",
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
