"""RND-PPO on the GPU (pytest -m gpu): jb_rnd_ppo_loss, jb_rnd_loss and jb_adv_mix against float64 and against PPO's
kernels, the four-head layers, eager learns against the oracle's learn (oracle/rnd_ppo.py), the host path against the
resident path, the CUDA-graph path against eager, the persistent PPO kernel staying off, checkpoints, parallel.attach
and end-to-end runs of main --sync.

Tolerances (fp32 kernels against float64):
  loss gradients               : atol 1e-7 + 2e-5 * max|grad|;  losses: rtol 1e-5, atol 1e-6
  parameters after a learn     : atol 0.1 * lr (Adam normalises the update to ~lr)
  Adam moments                 : atol 1e-3 * max|moment| + tiny, rtol 5e-3
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import icm_ppo as oi
from oracle import rnd_ppo as orr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
FW = 256


def _C():
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    return C, ptr, stream_ptr


# ------------------------------------------------------------------------------------------ 1. the two-critic loss
def _ppo_inputs(rs, B, A, cont, regime):
    NT = B + 3
    nout = 2 * A + 2 if cont else A + 2
    npol = nout - 2
    out = rs.standard_normal((B, nout)).astype(np.float32)
    idx = rs.permutation(NT)[:B].astype(np.int32)
    action = rs.uniform(-0.9, 0.9, (NT, A)).astype(np.float32) if cont else rs.randint(0, A, NT).astype(np.int32)
    adv = rs.standard_normal(NT).astype(np.float32)
    ret, ret_i = rs.standard_normal(NT).astype(np.float32), rs.standard_normal(NT).astype(np.float32)
    lpo = rs.uniform(-2, -0.1, (NT, A) if cont else NT).astype(np.float32)
    v_old, v_i_old = rs.standard_normal(NT).astype(np.float32), rs.standard_normal(NT).astype(np.float32)
    if regime == "tie":          # every value inside its clip: v_clip = v, so each stream's two critic means tie
        v_old[idx] = out[:, npol] + 0.0625
        v_i_old[idx] = out[:, npol + 1] - 0.03125
    else:                        # values inside and outside each clip
        v_old[idx] = out[:, npol] + rs.uniform(-0.3, 0.3, B).astype(np.float32)
        v_i_old[idx] = out[:, npol + 1] + rs.uniform(-0.3, 0.3, B).astype(np.float32)
    return dict(out=out, idx=idx, action=action, adv=adv, ret=ret, v_old=v_old, ret_i=ret_i, v_i_old=v_i_old, lpo=lpo)


def _run_rnd_ppo(c, A, cont, hp=(0.1, 0.5, 0.01)):
    C, ptr, sp = _C()
    t = {k: torch.from_numpy(v).to(DEV) for k, v in c.items()}
    B, nout = c["out"].shape
    dout = torch.full((B, nout), float("nan"), device=DEV)
    stats = torch.full((8 + 4 * ((B + 255) // 256),), float("nan"), device=DEV)
    acc = torch.tensor([0, 0, 0, -float("inf"), float("inf"), 0, 0, 0], dtype=torch.float32, device=DEV)
    C.jb_rnd_ppo_loss(int(cont), ptr(t["out"]), ptr(t["idx"]), ptr(t["action"]), ptr(t["adv"]), ptr(t["ret"]),
                      ptr(t["v_old"]), ptr(t["ret_i"]), ptr(t["v_i_old"]), ptr(t["lpo"]), B, A, nout, *hp, ptr(dout),
                      ptr(stats), ptr(acc), sp())
    torch.cuda.synchronize()
    return dout.cpu().numpy(), stats.cpu().numpy(), acc.cpu().numpy()


@pytest.mark.parametrize("regime", ["mixed", "tie"])
@pytest.mark.parametrize("B", [1, 7, 256, 257, 2048])
@pytest.mark.parametrize("cont,A", [(False, 2), (False, 4), (False, 18), (True, 1), (True, 3), (True, 8)])
def test_rnd_ppo_loss_matches_the_float64_oracle(cont, A, B, regime):
    rs = np.random.RandomState(B * 13 + A + (100 if cont else 0) + (7 if regime == "tie" else 0))
    c = _ppo_inputs(rs, B, A, cont, regime)
    dout, stats, acc = _run_rnd_ppo(c, A, cont)
    d = lambda a: torch.from_numpy(np.asarray(a)).double()
    i = c["idx"]
    out = d(c["out"]).requires_grad_(True)
    act = d(c["action"][i]) if cont else d(c["action"][i]).view(-1, 1)
    col = lambda k: d(c[k][i]).view(B, -1)
    loss, aux = orr.ppo_loss(out, act, col("adv"), col("ret"), col("v_old"), col("ret_i"), col("v_i_old"), col("lpo"), A,
                             cont, 0.1, 0.5, 0.01)
    loss.backward()
    g = out.grad.numpy()
    np.testing.assert_allclose(dout, g, rtol=0, atol=1e-7 + 2e-5 * np.abs(g).max())
    exp = [aux[k].item() for k in ("actor_loss", "critic_loss", "entropy_loss", "max_ratio", "min_prob", "critic_e",
                                   "critic_i")]
    np.testing.assert_allclose(stats[:7], exp, rtol=1e-5, atol=1e-6)
    np.testing.assert_array_equal(acc[:5], stats[:5])
    assert acc[5] == 1.0


@pytest.mark.parametrize("B", [1, 7, 256, 257, 2048])
@pytest.mark.parametrize("cont,A", [(False, 2), (False, 18), (True, 1), (True, 8)])
def test_rnd_ppo_loss_is_bit_identical_to_ppo_loss_without_the_intrinsic_stream(cont, A, B):
    C, ptr, sp = _C()
    rs = np.random.RandomState(B + A)
    c = _ppo_inputs(rs, B, A, cont, "mixed")
    nout = c["out"].shape[1]
    c["ret_i"][c["idx"]] = c["v_i_old"][c["idx"]] = c["out"][:, -1]         # ret_i = v_i = v_old_i
    dout, stats, acc = _run_rnd_ppo(c, A, cont)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in c.items()}
    po = t["out"][:, :nout - 1].contiguous()
    pd = torch.full((B, nout - 1), float("nan"), device=DEV)
    pst = torch.full((8 + 4 * ((B + 255) // 256),), float("nan"), device=DEV)
    pacc = torch.tensor([0, 0, 0, -float("inf"), float("inf"), 0, 0, 0], dtype=torch.float32, device=DEV)
    C.jb_ppo_loss(int(cont), ptr(po), ptr(t["idx"]), ptr(t["action"]), ptr(t["adv"]), ptr(t["ret"]), ptr(t["v_old"]),
                  ptr(t["lpo"]), B, A, nout - 1, 0.1, 0.5, 0.01, ptr(pd), ptr(pst), ptr(pacc), sp())
    torch.cuda.synchronize()
    np.testing.assert_array_equal(dout[:, :nout - 1], pd.cpu().numpy())
    assert (dout[:, -1] == 0).all()
    np.testing.assert_array_equal(stats[:5], pst.cpu().numpy()[:5])
    np.testing.assert_array_equal(acc[:6], pacc.cpu().numpy()[:6])
    assert stats[6] == 0.0 and stats[5] == stats[1]


def test_rnd_prepass_matches_ppo_prepass():
    """log_prob_old and v are PPO's pre-pass bit for bit (the same device function); v_i is the last column."""
    C, ptr, sp = _C()
    rs = np.random.RandomState(3)
    for cont, A in ((False, 3), (False, 18), (True, 1), (True, 8)):
        M = 1000
        nout = 2 * A + 2 if cont else A + 2
        out = torch.from_numpy(rs.standard_normal((M, nout)).astype(np.float32)).to(DEV)
        act = torch.from_numpy(rs.uniform(-1, 1, (M, A)).astype(np.float32) if cont
                               else rs.randint(0, A, M).astype(np.int32)).to(DEV)
        v, vi, lp = (torch.empty(M, device=DEV) for _ in range(3))
        lp = torch.empty(M, A if cont else 1, device=DEV)
        C.jb_rnd_prepass(int(cont), ptr(out), ptr(act), M, A, nout, ptr(v), ptr(vi), ptr(lp), sp())
        po = out[:, :nout - 1].contiguous()
        pv, plp = torch.empty(M, device=DEV), torch.empty_like(lp)
        fn = C.jb_ppo_prepass_continuous if cont else C.jb_ppo_prepass_discrete
        fn(ptr(po), ptr(act), M, A, nout - 1, ptr(pv), ptr(plp), sp())
        torch.cuda.synchronize()
        assert torch.equal(v, pv) and torch.equal(lp, plp) and torch.equal(vi, out[:, -1])


# --------------------------------------------------------------------------------------- 2. the distillation loss
def _run_rnd_loss(p, tgt, idx, reward_only=False):
    C, ptr, sp = _C()
    B = p.shape[0]
    tp, tt, ti = (torch.from_numpy(x).to(DEV) for x in (p, tgt, idx))
    ri = torch.full((B,), float("nan"), device=DEV)
    dp = torch.full((B, FW), float("nan"), device=DEV)
    stats = torch.full((1 + (B + 7) // 8,), float("nan"), device=DEV)
    acc = torch.zeros(2, device=DEV)
    if reward_only:
        C.jb_rnd_loss(ptr(tp), ptr(tt), ptr(ti), B, FW, ptr(ri), 0, 0, 0, sp())
    else:
        C.jb_rnd_loss(ptr(tp), ptr(tt), ptr(ti), B, FW, ptr(ri), ptr(dp), ptr(stats), ptr(acc), sp())
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (ri, dp, stats, acc)]


@pytest.mark.parametrize("B", [1, 7, 256, 257, 2048])
def test_rnd_loss_matches_float64_with_duplicate_indices(B):
    rs = np.random.RandomState(B)
    NT = B + 5
    p = rs.standard_normal((B, FW)).astype(np.float32)
    tgt = rs.standard_normal((NT, FW)).astype(np.float32)
    idx = rs.randint(0, NT, B).astype(np.int32)
    if B > 1:
        idx[1] = idx[0]                                  # at least one duplicate
    ri, dp, stats, acc = _run_rnd_loss(p, tgt, idx)
    P, Tg = torch.from_numpy(p).double(), torch.from_numpy(tgt[idx]).double()
    r_ref, l_ref = orr.rnd_loss(P, Tg)
    g = orr.closed_form(P, Tg).numpy()
    np.testing.assert_allclose(ri, r_ref.numpy(), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(dp, g, rtol=0, atol=1e-6 * np.abs(g).max())
    np.testing.assert_allclose(stats[0], float(l_ref), rtol=1e-5)
    assert acc[0] == stats[0] and acc[1] == 1.0
    ri2, dp2, stats2, _ = _run_rnd_loss(p, tgt, idx, reward_only=True)
    np.testing.assert_array_equal(ri2, ri)
    assert np.isnan(dp2).all() and np.isnan(stats2).all()


# ------------------------------------------------------------------------------------------------ 3. advantage mix
@pytest.mark.parametrize("T", [1, 5, 64, 200, 2048])
def test_adv_mix_matches_float64_and_is_gae_at_coefficients_one_zero(T):
    C, ptr, sp = _C()
    rs = np.random.RandomState(T)
    N = 37
    r, d = rs.standard_normal(N * T).astype(np.float32), (rs.uniform(size=N * T) < 0.05).astype(np.float32)
    v, nv = rs.standard_normal(N * T).astype(np.float32), rs.standard_normal(N * T).astype(np.float32)
    ai = rs.standard_normal(N * T).astype(np.float32)
    tr, td, tv, tnv, tai = (torch.from_numpy(x).to(DEV) for x in (r, d, v, nv, ai))
    ae, ret, ref_adv = (torch.empty(N * T, device=DEV) for _ in range(3))
    C.jb_gae(ptr(tr), ptr(td), ptr(tv), ptr(tnv), 0, N, T, 0.99, 0.95, 0, ptr(ae), ptr(ret), sp())
    C.jb_gae(ptr(tr), ptr(td), ptr(tv), ptr(tnv), 0, N, T, 0.99, 0.95, 1, ptr(ref_adv), ptr(ret), sp())
    one_zero = torch.empty(N * T, device=DEV)
    C.jb_adv_mix(ptr(ae), ptr(tai), N, T, 1.0, 0.0, 1, ptr(one_zero), sp())
    for std in (0, 1):
        mixed = torch.empty(N * T, device=DEV)
        C.jb_adv_mix(ptr(ae), ptr(tai), N, T, 2.0, 1.0, std, ptr(mixed), sp())
        torch.cuda.synchronize()
        exp = orr.adv_mix(ae.cpu().double(), tai.cpu().double(), T, 2.0, 1.0, bool(std) and T > 1).numpy().reshape(-1)
        if std and T == 1:
            exp = np.zeros_like(exp)                     # one step: (a - a) / (0 + 1e-7)
        np.testing.assert_allclose(mixed.cpu().numpy(), exp, rtol=1e-5, atol=1e-5)
    torch.cuda.synchronize()
    assert torch.equal(one_zero, ref_adv)


# ------------------------------------------------------------------------------------------------ 4. four heads
@pytest.mark.parametrize("A", [1, 3, 8])
def test_four_head_layers_match_float64(A):
    from jorldy_b200.core.network import layers as L
    rs = np.random.RandomState(A)
    M, H = 300, 96
    h = torch.from_numpy(np.maximum(rs.standard_normal((M, H)), 0).astype(np.float32)).to(DEV)
    sizes = (A, A, 1, 1)
    ws = [torch.from_numpy(rs.standard_normal((n, H)).astype(np.float32)).to(DEV) for n in sizes]
    bs = [torch.from_numpy(rs.standard_normal(n).astype(np.float32)).to(DEV) for n in sizes]
    nout = 2 * A + 2
    out = torch.empty(M, nout, device=DEV)
    L.heads_fwd(h, list(zip(ws, bs)), out)
    dout = torch.from_numpy(rs.standard_normal((M, nout)).astype(np.float32)).to(DEV)
    dh = torch.empty(M, H, device=DEV)
    L.heads_bwd_dx(dout, h, list(zip(ws, bs)), dh)
    dws, dbs = [torch.empty_like(w) for w in ws], [torch.empty_like(b) for b in bs]
    L.heads_bwd_dw(dout, h, list(zip(dws, dbs)))
    torch.cuda.synchronize()
    W, Bb, Hd, D = torch.cat(ws).cpu().double(), torch.cat(bs).cpu().double(), h.cpu().double(), dout.cpu().double()
    np.testing.assert_allclose(out.cpu().numpy(), (Hd @ W.T + Bb).numpy(), rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(dh.cpu().numpy(), ((D @ W) * (Hd > 0)).numpy(), rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(torch.cat(dws).cpu().numpy(), (D.T @ Hd).numpy(), rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(torch.cat(dbs).cpu().numpy(), D.sum(0).numpy(), rtol=1e-5, atol=1e-4)


def test_three_head_entry_points_equal_the_array_form():
    from jorldy_b200.core.network import layers as L
    C, ptr, sp = _C()
    rs = np.random.RandomState(9)
    M, H = 257, 512
    h = torch.from_numpy(np.maximum(rs.standard_normal((M, H)), 0).astype(np.float32)).to(DEV)
    ws = [torch.from_numpy(rs.standard_normal((n, H)).astype(np.float32)).to(DEV) for n in (3, 3, 1)]
    bs = [torch.from_numpy(rs.standard_normal(n).astype(np.float32)).to(DEV) for n in (3, 3, 1)]
    dout = torch.from_numpy(rs.standard_normal((M, 7)).astype(np.float32)).to(DEV)
    o1, o2 = torch.empty(M, 7, device=DEV), torch.empty(M, 7, device=DEV)
    C.jb_heads_fwd(ptr(h), M, H, *sum([[ptr(w), ptr(b), w.shape[0]] for w, b in zip(ws, bs)], []), ptr(o1), sp())
    L.heads_fwd(h, list(zip(ws, bs)), o2)
    d1, d2 = torch.empty(M, H, device=DEV), torch.empty(M, H, device=DEV)
    C.jb_heads_bwd_dx(ptr(dout), ptr(h), M, H, *sum([[ptr(w), w.shape[0]] for w in ws], []), ptr(d1), sp())
    L.heads_bwd_dx(dout, h, list(zip(ws, bs)), d2)
    g1 = [(torch.empty_like(w), torch.empty_like(b)) for w, b in zip(ws, bs)]
    g2 = [(torch.empty_like(w), torch.empty_like(b)) for w, b in zip(ws, bs)]
    C.jb_heads_bwd_dw(ptr(dout), ptr(h), M, H, *sum([[ptr(w), ptr(b), w.shape[0]] for w, b in g1], []), sp())
    L.heads_bwd_dw(dout, h, g2)
    torch.cuda.synchronize()
    assert torch.equal(o1, o2) and torch.equal(d1, d2)
    for (a, b), (c, d) in zip(g1, g2):
        assert torch.equal(a, c) and torch.equal(b, d)


# ------------------------------------------------------------------------------------------------ 5. rejections
def test_new_entry_points_reject_bad_arguments():
    import ctypes
    from jorldy_b200._lib import JbError
    C, ptr, sp = _C()
    buf = torch.zeros(1 << 16, device=DEV)
    ib = torch.zeros(4096, dtype=torch.int32, device=DEV)
    p, ip = ptr(buf), ptr(ib)

    def loss(cont=0, B=8, A=2, nout=4, out=p, ret_i=p, vi=p, dout=p, stats=p):
        C.jb_rnd_ppo_loss(cont, out, 0, ip, p, p, p, ret_i, vi, p, B, A, nout, 0.1, 0.5, 0.01, dout, stats, 0, sp())
    loss()
    loss(cont=1, A=3, nout=8)
    for kw in (dict(B=0), dict(A=0), dict(A=19, nout=21), dict(cont=1, A=9, nout=20), dict(nout=3), dict(cont=1, nout=5),
               dict(out=0), dict(ret_i=0), dict(vi=0), dict(dout=0), dict(stats=0)):
        with pytest.raises(JbError):
            loss(**kw)

    def prepass(cont=0, M=8, A=2, nout=4, v=p, vi=p, lp=p):
        C.jb_rnd_prepass(cont, p, ip, M, A, nout, v, vi, lp, sp())
    prepass()
    for kw in (dict(M=0), dict(A=19, nout=21), dict(nout=3), dict(cont=1, A=2, nout=5), dict(vi=0), dict(lp=0)):
        with pytest.raises(JbError):
            prepass(**kw)

    def rnd(B=8, F=FW, pp=p, t=p, ri=p, dp=p, stats=p):
        C.jb_rnd_loss(pp, t, 0, B, F, ri, dp, stats, 0, sp())
    rnd()
    rnd(dp=0, stats=0)
    for kw in (dict(B=0), dict(F=128), dict(pp=0), dict(t=0), dict(stats=0), dict(dp=0, ri=0)):
        with pytest.raises(JbError):
            rnd(**kw)

    def mix(N=4, T=8, a=p, b=p, o=p):
        C.jb_adv_mix(a, b, N, T, 2.0, 1.0, 1, o, sp())
    mix()
    for kw in (dict(N=0), dict(T=0), dict(a=0), dict(b=0), dict(o=0)):
        with pytest.raises(JbError):
            mix(**kw)

    arr = lambda xs, t=ctypes.c_void_p: (t * len(xs))(*xs)
    C.jb_heads_fwd_n(p, 4, 32, 4, arr([p] * 4), arr([p] * 4), arr([1] * 4, ctypes.c_int), p, sp())
    torch.cuda.synchronize()
    for n_heads, n in ((0, [1]), (5, [1] * 5), (4, [8, 8, 8, 9]), (2, [0, 0])):
        with pytest.raises(JbError):
            C.jb_heads_fwd_n(p, 4, 32, n_heads, arr([p] * len(n)), arr([p] * len(n)), arr(n, ctypes.c_int), p, sp())
    with pytest.raises(JbError):
        C.jb_heads_fwd_n(p, 4, 32, 2, arr([p, 0]), arr([p, p]), arr([1, 1], ctypes.c_int), p, sp())


# ------------------------------------------------------------------------------------------------- 6. learn
CASES = {
    "cartpole_h64": dict(seed=41, N=4, T=32, D=4, A=2, H=64, continuous=False, batch_size=32, n_epoch=2, lr=2.5e-4),
    "cartpole_h512": dict(seed=42, N=8, T=64, D=4, A=2, H=512, continuous=False, batch_size=256, n_epoch=2, lr=2.5e-4),
    "hopper": dict(seed=43, N=4, T=64, D=11, A=3, H=256, continuous=True, batch_size=64, n_epoch=2, lr=3e-4),
}
RND_KW = dict(gamma_i=0.99, extrinsic_coeff=2.0, intrinsic_coeff=1.0, obs_normalize=True, ri_normalize=True,
              batch_norm=True, non_episodic=True)


def _agent(case, **kw):
    from jorldy_b200.core import Agent
    net = "continuous_policy_value" if case["continuous"] else "discrete_policy_value"
    args = dict(RND_KW, **kw)
    return Agent("rnd_ppo", state_size=case["D"], action_size=case["A"], hidden_size=case["H"], network=net,
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


def _snapshot(agent):
    cpu = lambda d: {k: v.detach().cpu().clone() for k, v in d.items()}
    return cpu(agent.network.p), cpu(agent.rnd.target.p), cpu(agent.rnd.predictor.p), cpu(agent.rnd.predictor.buffers)


def _check_learn_against_oracle(agent, case, rkw, learns=2):
    params, tgt, pred, bufs = _snapshot(agent)
    tgt0 = {k: v.clone() for k, v in tgt.items()}
    ss = orr.new_state(case["D"], case["N"])
    opt_state = None
    for learn in range(learns):
        batch, perms = _batch(case, learn)
        res = _learn(agent, case, batch, perms)
        ref = orr.learn(params, tgt, pred, bufs, batch, _hp(case), rkw, perms, case["lr"], ss, opt_state=opt_state)
        params, pred, bufs, opt_state = ref["params"], ref["predictor"], ref["buffers"], ref["opt_state"]
        for k, v in ref["params"].items():
            np.testing.assert_allclose(agent.network.p[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=0.1 * case["lr"],
                                       err_msg=k)
        # BatchNorm cancels fc1's bias: its float64 gradient is 0 and the fp32 one is round-off, which Adam turns into steps
        # of up to ~lr.  fc1.bias, and the running mean that carries it, are held to that bound: lr per step taken so far.
        drift = case["lr"] * (learn + 1) * case["n_epoch"] * -(-case["N"] * case["T"] // case["batch_size"])
        for k, v in ref["predictor"].items():
            atol = drift if (k == "fc1.bias" and rkw["batch_norm"]) else 0.1 * case["lr"]
            np.testing.assert_allclose(agent.rnd.predictor.p[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=atol, err_msg=k)
        for k, v in ref["buffers"].items():
            got = agent.rnd.predictor.buffers[k].cpu()
            if v.dtype == torch.int64:
                assert int(got) == int(v), k
            else:
                atol = drift if k.endswith("running_mean") else 1e-5
                np.testing.assert_allclose(got.numpy(), v.numpy(), rtol=1e-4, atol=atol, err_msg=k)
        for k, v in tgt0.items():
            assert torch.equal(agent.rnd.target.p[k].cpu(), v), k            # the target is never updated
        assert set(res) == set(ref["result"])
        for k, v in ref["result"].items():
            np.testing.assert_allclose(res[k], v, rtol=2e-4, atol=2e-4, err_msg=k)
        if rkw["obs_normalize"]:
            np.testing.assert_allclose(agent.rms_obs.mean.cpu().numpy(), ss["rms_obs"].mean, rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(agent.rms_obs.var.cpu().numpy(), ss["rms_obs"].var, rtol=1e-9)
        if rkw["ri_normalize"]:
            np.testing.assert_allclose(float(agent.rms_ri.var), float(ss["rms_ri"].var), rtol=1e-3)
            np.testing.assert_allclose(agent.rewems.cpu().numpy(), ss["rewems"], rtol=1e-3, atol=1e-7)
        st = opt_state["state"]
        P = len(agent.network.p)
        for opt, names, off in ((agent.optimizer, list(agent.network.p), 0),
                                (agent.rnd_optimizer, list(agent.rnd.predictor.p), P)):
            m, v = opt._slot_views(opt.exp_avg), opt._slot_views(opt.exp_avg_sq)
            for i, k in enumerate(names):
                if k == "fc1.bias" and opt is agent.rnd_optimizer and rkw["batch_norm"]:
                    continue        # BatchNorm cancels fc1's bias: its gradient is 0 in float64 and fp32 round-off here
                for got, key in ((m[i], "exp_avg"), (v[i], "exp_avg_sq")):
                    r = st[off + i][key].numpy()
                    np.testing.assert_allclose(got.cpu().numpy(), r, rtol=5e-3, atol=1e-3 * np.abs(r).max() + 1e-12,
                                               err_msg=f"{key} {k}")


@pytest.mark.parametrize("name", list(CASES))
def test_two_eager_learns_match_the_float64_oracle(name):
    case = CASES[name]
    _check_learn_against_oracle(_agent(case, use_cuda_graph=False), case, RND_KW)


@pytest.mark.parametrize("kw", [dict(non_episodic=False),
                                dict(obs_normalize=False, ri_normalize=False, batch_norm=False)])
def test_learns_with_episodic_intrinsic_stream_or_without_normalisation_and_batch_norm(kw):
    case = CASES["cartpole_h64"]
    agent = _agent(case, use_cuda_graph=False, **kw)
    if not kw.get("batch_norm", True):
        assert not agent.rnd.predictor.buffers and "bn1.weight" not in agent.rnd.predictor.p
    _check_learn_against_oracle(agent, case, dict(RND_KW, **kw))


def test_eager_learn_on_atari_frames_with_the_cnn_rnd_matches_the_float64_oracle():
    """A = 18, the CNN head and the CNN RND on uint8 frame stacks, one epoch of 2 Adam steps.  A ReLU input within fp32
    round-off of 0 can take the other side in float64, so parameters are compared normwise against the update."""
    from jorldy_b200.core import Agent
    N, T, B, A, lr = 4, 8, 16, 18, 2.5e-4
    case = dict(continuous=False, A=A, T=T, batch_size=B, n_epoch=1)
    rkw = dict(RND_KW, obs_normalize=False)
    agent = Agent("rnd_ppo", state_size=[4, 84, 84], action_size=A, hidden_size=64, network="discrete_policy_value",
                  head="cnn", rnd_network="rnd_cnn", optim_config={"name": "adam", "lr": lr}, run_step=1000,
                  lr_decay=False, device=DEV, batch_size=B, n_step=T, n_epoch=1, use_cuda_graph=False, **rkw)
    rs = np.random.RandomState(8)
    state = torch.from_numpy(rs.randint(0, 256, (N * T, 4, 84, 84)).astype(np.uint8))
    nxt = torch.from_numpy(rs.randint(0, 256, (N * T, 4, 84, 84)).astype(np.uint8))
    action = torch.from_numpy(rs.randint(0, A, (N * T, 1)).astype(np.float32))
    reward = torch.from_numpy(rs.standard_normal((N * T, 1)).astype(np.float32))
    done = torch.from_numpy((rs.uniform(size=(N * T, 1)) < 0.1).astype(np.float32))
    perms = [rs.permutation(N * T)]
    params, tgt, pred, bufs = _snapshot(agent)
    agent._inject_perms = perms
    res = agent._learn_tensors(state.to(DEV), action.reshape(-1).to(torch.int32).to(DEV), reward.reshape(-1).to(DEV),
                               done.reshape(-1).to(DEV), next_state=nxt.to(DEV))
    torch.cuda.synchronize()
    batch = dict(state=state.double(), next_state=nxt.double(), action=action, reward=reward, done=done)
    ref = orr.learn(params, tgt, pred, bufs, batch, _hp(case), rkw, perms, lr, orr.new_state(1, N))
    # Below the predictor's BatchNorm the gradient reaching fc1's input sums to 0 over the rows, so the trunk's bias
    # gradients are what the ReLU masks leave of a cancelling sum, and fc1's bias gets only round-off: those are held to
    # 5e-2 of their update, fc1.bias is skipped, everything else to 2e-2.
    for which, start, got_p, ref_p in (("network", params, agent.network.p, ref["params"]),
                                       ("predictor", pred, agent.rnd.predictor.p, ref["predictor"])):
        for k, v in ref_p.items():
            if which == "predictor" and k == "fc1.bias":
                continue
            tol = 5e-2 if which == "predictor" and k.startswith("head.") and k.endswith(".bias") else 2e-2
            upd = (v - start[k].double()).norm().item()
            err = (got_p[k].cpu().double() - v).norm().item()
            assert err <= tol * upd + 1e-9, (which, k, err, upd)
    for k, v in tgt.items():
        assert torch.equal(agent.rnd.target.p[k].cpu(), v), k
    for k, v in ref["buffers"].items():
        got = agent.rnd.predictor.buffers[k].cpu()
        if v.dtype == torch.int64:
            assert int(got) == int(v), k
        elif k.endswith("running_var"):
            np.testing.assert_allclose(got.numpy(), v.numpy(), rtol=1e-3, atol=1e-5, err_msg=k)
    for k, v in ref["result"].items():
        np.testing.assert_allclose(res[k], v, rtol=1e-3, atol=1e-3, err_msg=k)


def _state(g):
    return [g.network.flat, g.rnd.predictor.flat, g.rnd.target.flat, *g.rnd.buffer_tensors(), *g.optimizer.state_tensors(),
            *g.rnd_optimizer.state_tensors(), g._acc, g._rnd_acc, *g.rms_obs.tensors(), *g.rms_ri.tensors(), g.rewems]


def test_host_learn_equals_learn_rollout_on_the_same_steps():
    """The resident path reads V(s') and the RND input from the rollout's next-state rows, the host path from its
    transitions: the same steps give the same learn bit for bit."""
    from jorldy_b200.core import Agent, Env
    from jorldy_b200.core.collect import RolloutCollector
    kw = dict(state_size=4, action_size=2, hidden_size=64, batch_size=64, n_step=32, n_epoch=2, device=DEV, run_step=1000,
              lr_decay=False, use_cuda_graph=False)
    a, b = Agent("rnd_ppo", **kw), Agent("rnd_ppo", **kw)
    b.network.load_state_dict(a.network.state_dict())
    b.rnd.load_state_dict(a.rnd.state_dict())
    ro = RolloutCollector(Env("cartpole", num_envs=16, seed=4), a, use_cuda_graph=False).collect()
    torch.cuda.synchronize()
    assert ro.done.bool().any()
    N, T = ro.N, ro.T
    perms = [np.random.RandomState(e).permutation(N * T) for e in range(2)]
    a._inject_perms = b._inject_perms = perms
    state, nxt = ro.state.view(N * T, -1).clone(), ro.next_state.view(N * T, -1).clone()
    act, rew, done = ro.action.view(N * T).clone(), ro.reward.view(N * T).clone(), ro.done.view(N * T).clone()
    rb = b._learn_tensors(state, act, rew, done, next_state=nxt)
    ra = a.learn_rollout(ro)
    torch.cuda.synchronize()
    assert ra == rb
    for x, y in zip(_state(a), _state(b)):
        assert torch.equal(x, y)


def test_graph_learn_is_bit_identical_to_eager_and_reproducible(monkeypatch):
    import jorldy_b200.core.agent.ppo as ppo_mod
    monkeypatch.setattr(ppo_mod, "GRAPH_CHUNK", 2)
    case = dict(CASES["cartpole_h64"], N=8, T=40, batch_size=24)          # 13 full minibatches + a tail of 8
    torch.manual_seed(0)
    agents = [_agent(case, use_cuda_graph=g) for g in (True, False)]
    torch.manual_seed(0)
    agents.append(_agent(case, use_cuda_graph=True))                         # a second seeded run
    for a in agents[1:2]:
        a.network.load_state_dict(agents[0].network.state_dict())
        a.rnd.load_state_dict(agents[0].rnd.state_dict())
    assert torch.equal(agents[2].network.flat, agents[0].network.flat)
    assert torch.equal(agents[2].rnd.predictor.flat, agents[0].rnd.predictor.flat)
    results = []
    for a in agents:
        r = []
        for learn in range(2):
            batch, perms = _batch(case, learn)
            r.append(_learn(a, case, batch, perms))
        results.append(r)
    assert agents[0]._graphs and not agents[1]._graphs
    for a, r in zip(agents[1:], results[1:]):
        assert r == results[0]
        for x, y in zip(_state(a), _state(agents[0])):
            assert torch.equal(x, y)


def test_the_persistent_ppo_kernel_is_never_used():
    case = CASES["cartpole_h64"]
    from jorldy_b200.core.agent import ppo_fused
    agent = _agent(case, use_fused=True)
    assert agent.use_fused is False
    batch, perms = _batch(case)
    _learn(agent, case, batch, perms)
    assert agent._fused == {}
    from jorldy_b200.core import Agent                      # PPO at the same settings would take it
    p = Agent("ppo", state_size=4, action_size=2, hidden_size=64, batch_size=32, n_step=32, device=DEV, run_step=1000)
    assert ppo_fused.supported(p, 32)


# ------------------------------------------------------------------------------------------ 7. checkpoint, attach
def test_checkpoint_round_trip_and_layout(tmp_path):
    case = CASES["hopper"]
    a = _agent(case, use_cuda_graph=False)
    batch, perms = _batch(case)
    _learn(a, case, batch, perms)
    a.save(str(tmp_path))
    ck = torch.load(str(tmp_path / "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "rnd", "optimizer"}
    P, Q = len(a.network.p), len(a.rnd.predictor.p)
    assert ck["optimizer"]["param_groups"][0]["params"] == list(range(P + Q))
    assert sorted(ck["optimizer"]["state"]) == list(range(P + Q))
    assert list(ck["network"])[-2:] == ["v_i.weight", "v_i.bias"]
    keys = list(ck["rnd"])
    assert keys[:4] == ["target.fc1.weight", "target.fc1.bias", "target.fc2.weight", "target.fc2.bias"]
    assert keys[4:11] == ["predictor.fc1.weight", "predictor.fc1.bias", "predictor.bn1.weight", "predictor.bn1.bias",
                          "predictor.bn1.running_mean", "predictor.bn1.running_var", "predictor.bn1.num_batches_tracked"]
    b = _agent(case, seed=9)
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, a.network.flat) and torch.equal(b.rnd.predictor.flat, a.rnd.predictor.flat)
    assert torch.equal(b.rnd.target.flat, a.rnd.target.flat)
    for x, y in zip(b.rnd.buffer_tensors() + b.optimizer.state_tensors() + b.rnd_optimizer.state_tensors(),
                    a.rnd.buffer_tensors() + a.optimizer.state_tensors() + a.rnd_optimizer.state_tensors()):
        assert torch.equal(x, y)


def test_attach_keeps_rnd_ppo_a_replica():
    from jorldy_b200.core import parallel
    a = _agent(CASES["cartpole_h64"])
    with pytest.warns(UserWarning, match="replicas only .*RND-PPO"):
        parallel.attach(a, 2)
    assert a.world_size == 1 and a.allreduce is None


# -------------------------------------------------------------------------------------------------- 8. end to end
@pytest.mark.parametrize("config,extra", [
    ("config.rnd_ppo.cartpole", ["--train.num_workers", "8", "--agent.n_step", "32"]),
    ("config.rnd_ppo.mujoco", ["--env.name", "hopper", "--train.num_workers", "16", "--agent.n_step", "32",
                               "--agent.batch_size", "64", "--agent.hidden_size", "64", "--train.update_period", "32",
                               "--train.distributed_batch_size", "64"]),
    ("config.rnd_ppo.atari", ["--env.name", "seaquest", "--train.num_workers", "16", "--agent.n_step", "32",
                              "--agent.hidden_size", "64"]),
])
def test_sync_training_run_with_save_and_load(tmp_path, config, extra):
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
    assert {"network", "rnd", "optimizer"} == set(saved)
    r2 = subprocess.run(cmd + ["--train.load_path", ckpts[0]],
                        cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    assert "Traceback" not in r2.stdout + r2.stderr, (r2.stdout + r2.stderr)[-4000:]
    assert "Load model from" in r2.stdout, r2.stdout[-4000:]
