"""Discrete-action SAC on the GPU (csrc/actor_critic.cu jb_sacd_*, core/agent/ddpg.py SACDiscrete) against the float64
oracle (oracle/sac_discrete.py), the eager path, the stacked replay layout and the run loop (pytest -m gpu).

Tolerances.  u = 2^-24 is fp32's unit roundoff.
- Kernels (1): every output is a sum of at most A + 4 <= 22 rounded products per row, plus a fixed-order sum over B rows
  for the stats, and expf / logf within 2 ulp.  The standard bound gamma_n = n u / (1 - n u) on such sums gives a
  relative error of at most ~22 u * (sum |terms|) / |result|, and the B-row means add ~B u / sqrt(B) (pairwise tree of
  256 lanes).  With the inputs drawn here (|z| <= 8, |q| <= 3) sum |terms| / max |result| stays below ~20, so the
  normwise bound 22 * 20 * u = 2.6e-5 holds with margin under R = 1e-4: every check is max |got - ref| <= R * scale,
  scale = max |ref| of that output (and 1 for the entropy stats, which are O(ln A)).  A wrong kernel (dz without the
  -L_b term, max in place of min over the target critics, the target without (1 - d)) moves an output by O(0.01..1) of
  its scale; a wrong target_entropy (ln(A - 1)) moves alpha_loss in learn() (2).
- One learn against the float64 oracle (2): the fp32 forward and backward contract over K <= 12800 terms (conv1's weight
  gradient at B=32); their normwise error grows at worst like K u = 7.6e-4 and in practice like sqrt(K) u.  Gradients
  are checked normwise per tensor at 2e-3 (CNN) / 5e-4 (MLP), result-dict entries at rtol 5e-4 + atol 5e-4 * scale.
  The conv layers' gradients get 2e-2: the trunk has ~7e5 ReLU pre-activations per forward at B=32, and about one in
  10^6 lies within fp32 rounding of zero, so over the 9 network passes a few take the other branch in float64.  Such an
  element's value is ~0 on both sides (the forward does not move), but its gradient term is kept on one side and
  dropped on the other; against a conv weight gradient summed over >= 1568 rows that term is ~1/sqrt(1568) = 2.5e-2 of
  a typical element and far less of the largest one.
  Post-step parameters are checked against a float64 Adam step on the kernel's OWN gradients (for Adam's first step,
  p - lr g / (|g| + eps)): near |g| ~ eps a first Adam step turns rounding-level gradient differences into O(lr)
  parameter differences, so a comparison with the oracle's parameters would test the rounding, not the step; the bound
  is 1e-3 lr + 2 u |p|.  log_alpha / alpha follow the oracle over 3 learns at rtol 1e-5 (each Adam step on the scalar
  is lr * sign-like, exact up to the rounding of its inputs).
- Graph vs eager (3), frames vs stacks (5) and checkpoints (6) are bit-exact.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import sac_discrete as osd

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def _close(got, ref, R, what, scale=None):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = max(float(np.abs(ref).max()), 1e-30) if scale is None else scale
    err = float(np.abs(got - ref).max())
    assert err <= R * scale, f"{what}: max |err| {err:.3e} > {R} * {scale:.3e}"


# --------------------------------------------------------------------------------------------- 1. kernels vs the oracle
@pytest.mark.parametrize("A", [2, 4, 18])
@pytest.mark.parametrize("B", [1, 64, 257])
@pytest.mark.parametrize("d", [0, 1])
@pytest.mark.parametrize("alpha", [math.exp(-2.0), 1.0])
def test_kernels_match_the_oracle(A, B, d, alpha):
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    rs = np.random.RandomState(A * 1000 + B * 10 + d)
    f32 = lambda *s, sc=1.0: (sc * rs.standard_normal(s)).clip(-8, 8).astype(np.float32)
    z, nz = f32(B, A, sc=2.5), f32(B, A, sc=2.5)
    z[0] = 0.0                                            # equal logits
    q1, q2, nq1, nq2 = (f32(B, A).clip(-3, 3) for _ in range(4))
    action = rs.randint(A, size=B).astype(np.int64)
    reward = f32(B)
    done = np.full(B, float(d), np.float32)
    gamma, te = 0.99, osd.target_entropy(A)
    dv = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    t = {k: dv(v) for k, v in dict(z=z, nz=nz, q1=q1, q2=q2, nq1=nq1, nq2=nq2, a=action, r=reward, d=done).items()}
    al = torch.tensor([alpha], dtype=torch.float32, device=DEV)
    dq1, dq2, dz = (torch.empty(B, A, device=DEV) for _ in range(3))
    st = torch.full((16,), float("nan"), device=DEV)
    C.jb_sacd_critic_loss(ptr(t["q1"]), ptr(t["q2"]), ptr(t["nq1"]), ptr(t["nq2"]), ptr(t["nz"]), ptr(t["a"]), ptr(t["r"]),
                          ptr(t["d"]), ptr(al), B, A, gamma, ptr(dq1), ptr(dq2), ptr(st), stream_ptr())
    C.jb_sacd_actor(ptr(t["z"]), ptr(t["q1"]), ptr(t["q2"]), ptr(al), np.float32(te), B, A, ptr(dz), st.data_ptr() + 16,
                    stream_ptr())
    torch.cuda.synchronize()
    h = lambda x: torch.from_numpy(x).to(torch.float64)
    al64 = float(np.float32(alpha))
    y = osd.target(h(nz), h(nq1), h(nq2), h(reward), h(done), float(np.float32(gamma)), al64)
    l1, l2, rdq1, rdq2 = osd.critic_closed(h(q1), h(q2), torch.from_numpy(action), y)
    rdz, rst = osd.actor_closed(h(z), h(q1), h(q2), al64, te)
    R = 1e-4
    got = st.cpu().numpy().astype(np.float64)
    ysc = float(y.abs().max())
    _close(got[2], y.max().item(), R, "max_Q", ysc)
    # the target itself, recovered from dq at the taken action: y = q1[a] - dq1[a] * B / 2
    gy = q1[np.arange(B), action] - dq1.cpu().numpy()[np.arange(B), action].astype(np.float64) * B / 2
    _close(gy, y.numpy(), R, "target", ysc + np.abs(q1).max())
    _close(got[0], l1.item(), R, "critic_loss1")
    _close(got[1], l2.item(), R, "critic_loss2")
    _close(dq1.cpu().numpy(), rdq1.numpy(), R, "dq1")
    _close(dq2.cpu().numpy(), rdq2.numpy(), R, "dq2")
    assert (dq1.cpu().numpy() != 0).sum() <= B and (dq2.cpu().numpy() != 0).sum() <= B     # only the taken action
    _close(dz.cpu().numpy(), rdz.numpy(), R, "dz")
    qsc = float(np.abs(np.minimum(q1, q2)).max()) + alpha * 20
    _close(got[4], rst["actor_loss"], R, "actor_loss", qsc)
    _close(got[5], rst["mean_Q"], R, "mean_Q", qsc)
    _close(got[6], rst["entropy"], R, "entropy", 1.0)
    _close(got[7], rst["entropy_gap"], R, "entropy - target_entropy", 1.0)


# --------------------------------------------------------------------------------- 2. one eager learn vs float64 oracle
CAP = 64
LEARN_CASES = {
    "mlp_h64": dict(head="mlp", D=4, A=2, H=64, B=16, dynamic=True),
    "mlp_h512": dict(head="mlp", D=4, A=2, H=512, B=64, dynamic=False),
    "cnn": dict(head="cnn", D=[4, 84, 84], A=18, H=512, B=32, dynamic=True),
}
LR = dict(actor_lr=3e-4, critic_lr=1e-3, alpha_lr=2e-3)


def _agent(case, seed=0, graph=False, buffer_size=CAP, **extra):
    from jorldy_b200.core import Agent
    torch.manual_seed(seed)
    optim = dict(actor="adam", critic="adam", alpha="adam", **LR)
    kw = dict(state_size=case["D"], action_size=case["A"], hidden_size=case["H"], actor="discrete_policy",
              critic="discrete_q_network", head=case["head"], optim_config=optim, use_dynamic_alpha=case["dynamic"],
              gamma=0.99, tau=5e-3, buffer_size=buffer_size, batch_size=case["B"], run_step=1000, lr_decay=False,
              device=DEV, seed=seed, use_cuda_graph=graph)
    kw.update(extra)
    agent = Agent("sac", **kw)
    with torch.no_grad():
        agent.actor.p["pi.weight"].mul_(150.0)             # a policy far from uniform: pi and logpi both matter
    return agent


def _replay(case, rs):
    A, n = case["A"], CAP
    if case["head"] == "cnn":
        s = rs.randint(0, 256, size=(n, 4, 84, 84)).astype(np.uint8)
        ns = rs.randint(0, 256, size=(n, 4, 84, 84)).astype(np.uint8)
    else:
        s = rs.standard_normal((n, case["D"])).astype(np.float32)
        ns = rs.standard_normal((n, case["D"])).astype(np.float32)
    return {"state": s, "next_state": ns, "action": rs.randint(A, size=(n, 1)).astype(np.int64),
            "reward": rs.standard_normal((n, 1)), "done": rs.uniform(size=(n, 1)) < 0.25}


def _params(net):
    return {k: v.detach().cpu().to(torch.float64) for k, v in net.p.items()}


def _nets(agent):
    return {"actor": agent.actor, "critic1": agent.critics[0], "critic2": agent.critics[1],
            "target_critic1": agent.target_critics[0], "target_critic2": agent.target_critics[1]}


@pytest.mark.parametrize("name", list(LEARN_CASES))
def test_eager_learn_matches_the_float64_oracle(name):
    case = LEARN_CASES[name]
    rs = np.random.RandomState(5)
    agent = _agent(case)
    assert agent.action_type == "discrete" and agent.target_entropy == 0.98 * math.log(case["A"])
    tr = _replay(case, rs)
    agent.memory.store([tr])
    hp = dict(gamma=0.99, use_dynamic_alpha=case["dynamic"], A=case["A"], **LR)
    opt_state, cnn = None, case["head"] == "cnn"
    alpha_in = agent.alpha.item()
    for i in range(3):
        idx = rs.randint(CAP, size=case["B"])
        batch = {"state": torch.from_numpy(tr["state"][idx]), "next_state": torch.from_numpy(tr["next_state"][idx]),
                 "action": torch.from_numpy(tr["action"][idx, 0]),
                 "reward": torch.from_numpy(tr["reward"][idx, 0].astype(np.float32)),
                 "done": torch.from_numpy(tr["done"][idx, 0].astype(np.float32))}
        pre = {k: _params(n) for k, n in _nets(agent).items()}
        la_pre = agent.log_alpha.flat[0].item()
        ref = osd.learn(pre["actor"], pre["critic1"], pre["critic2"], pre["target_critic1"], pre["target_critic2"],
                        torch.tensor([la_pre], dtype=torch.float64), alpha_in, batch, hp, opt_state)
        opt_state = ref["opt_state"]
        agent._inject_idx = idx
        res = agent.learn()
        torch.cuda.synchronize()
        assert set(res) == {"critic_loss1", "critic_loss2", "actor_loss", "alpha_loss", "max_Q", "mean_Q", "alpha", "entropy"}
        for k, v in ref["result"].items():
            sc = max(abs(v), 1.0)
            assert abs(res[k] - v) <= 5e-4 * abs(v) + 5e-4 * sc, (name, i, k, res[k], v)
        # gradients of this learn, normwise per tensor
        for net, key in (("actor", "actor_grads"), ("critic1", "critic1_grads"), ("critic2", "critic2_grads")):
            for k, g in ref[key].items():
                R = (2e-2 if k.startswith("head.") else 2e-3) if cnn else 5e-4
                _close(_nets(agent)[net].g[k].cpu().numpy(), g.numpy(), R, f"learn {i} grad {net}.{k}", float(g.abs().max()) + 1e-12)
        if i == 0:                  # Adam's first step on the kernel's own gradients, in float64
            for net in ("actor", "critic1", "critic2"):
                lr = LR["actor_lr"] if net == "actor" else LR["critic_lr"]
                for k, p0 in pre[net].items():
                    g = _nets(agent)[net].g[k].cpu().to(torch.float64)
                    want = p0 - lr * g / (g.abs() + 1e-8)
                    got = _nets(agent)[net].p[k].cpu().to(torch.float64)
                    assert (got - want).abs().max().item() <= 1e-3 * lr + 2 * U * p0.abs().max().item(), (net, k)
        # the temperature: alpha handed out = exp(log_alpha before this learn's step); the next learn uses it
        assert abs(res["alpha"] - math.exp(la_pre)) <= 1e-6 * math.exp(la_pre)
        np.testing.assert_allclose(agent.log_alpha.flat[0].item(), ref["log_alpha"].item(), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(agent.alpha.item(), ref["alpha"], rtol=1e-5)
        if case["dynamic"] and i > 0:
            assert agent.log_alpha.flat[0].item() != la_pre and abs(alpha_in - math.exp(la_pre)) > 0   # the lag
        alpha_in = agent.alpha.item()
        # soft update as process() does it after every learn: bit-exact
        want = {t: tau_mix(pre[t], _nets(agent)[c]) for t, c in (("target_critic1", "critic1"), ("target_critic2", "critic2"))}
        agent.update_target_soft()
        for t, w in want.items():
            for k, v in w.items():
                assert torch.equal(_nets(agent)[t].p[k].cpu(), v), (t, k)
    if not case["dynamic"]:
        assert agent.log_alpha.flat[0].item() == np.float32(-2.0) and abs(res["alpha"] - math.exp(-2.0)) < 1e-6


def tau_mix(target64, online, tau=5e-3):
    """t := tau * p + (1 - tau) * t in fp32 (two rounded products, one rounded sum), on the CPU."""
    return {k: tau * online.p[k].cpu() + (1 - tau) * target64[k].to(torch.float32) for k in target64}


# ------------------------------------------------------------------------------------------- 3. graph learn == eager
@pytest.mark.parametrize("name", ["mlp", "cnn"])
def test_cuda_graph_learn_is_bit_identical_to_eager(name):
    case = dict(head="mlp", D=4, A=4, H=64, B=32, dynamic=True) if name == "mlp" else \
        dict(head="cnn", D=[4, 84, 84], A=18, H=64, B=16, dynamic=True)
    rs = np.random.RandomState(11)
    a, b = _agent(case, graph=True), _agent(case, graph=False)
    for x, y in zip(_nets(a).values(), _nets(b).values()):
        y.flat.copy_(x.flat)
    tr = _replay(case, rs)
    a.memory.store([tr]); b.memory.store([tr])
    for i in range(4):
        a._inject_idx = b._inject_idx = rs.randint(CAP, size=case["B"])
        ra, rb = a.learn(), b.learn()
        assert ra == rb, (i, ra, rb)
        a.update_target_soft(); b.update_target_soft()
    torch.cuda.synchronize()
    for (k, x), y in zip(_nets(a).items(), _nets(b).values()):
        assert torch.equal(x.flat, y.flat), k
    assert torch.equal(a.log_alpha.flat, b.log_alpha.flat) and torch.equal(a.alpha, b.alpha)
    assert len(a._graphs) == 1 and not b._graphs


# ----------------------------------------------------------------------------------------------------------- 4. act
def test_act_greedy_and_injected_uniforms_match_the_oracle():
    case = dict(head="mlp", D=4, A=18, H=64, B=8, dynamic=False)
    agent = _agent(case)
    rs = np.random.RandomState(3)
    M = 4096
    s = torch.from_numpy(rs.standard_normal((M, 4)).astype(np.float32)).to(DEV)
    greedy, _ = agent.act_device(s, training=False)
    z = agent.actor._buf("act.z", (M, 18)).cpu().to(torch.float64)
    assert greedy.shape == (M, 1) and greedy.dtype == torch.int64
    assert torch.equal(greedy.view(-1).cpu(), osd.act(z))
    u = rs.uniform(size=M).astype(np.float32)
    got, _ = agent.act_device(s, training=True, noise=torch.from_numpy(u).to(DEV))
    want = osd.act(z, torch.from_numpy(u))
    diff = (got.view(-1).cpu() != want).nonzero().view(-1)
    # a row may differ only when u * sum(pi) lies within fp32 rounding of a CDF step
    pi = torch.softmax(z, -1)
    margin = (u[:, None] * pi.sum(-1, keepdim=True).numpy() - pi.cumsum(-1).numpy())
    for m in diff.tolist():
        assert np.abs(margin[m]).min() < 1e-5, m
    assert len(diff) <= 2
    # the numpy act() path: int64 [N, 1]
    out = agent.act(s[:5].cpu().numpy(), training=False)["action"]
    assert out.dtype == np.int64 and out.shape == (5, 1)


def test_philox_draws_follow_pi():
    """Chi-square of 10^5 draws from one 18-action row against pi (the seed is fixed, so this is deterministic)."""
    from scipy.stats import chisquare
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    M, A = 100_000, 18
    z = torch.linspace(-1.5, 1.0, A, dtype=torch.float32)
    logits = z.repeat(M, 1).to(DEV).contiguous()
    ctr = torch.zeros(M, dtype=torch.int64, device=DEV)
    act = torch.empty(M, 1, dtype=torch.int64, device=DEV)
    C.jb_sacd_act(ptr(logits), M, A, None, 7, 0, ptr(ctr), 0, ptr(act), stream_ptr())
    counts = np.bincount(act.view(-1).cpu().numpy(), minlength=A)
    pi = torch.softmax(z.to(torch.float64), -1).numpy()
    assert chisquare(counts, pi * M).pvalue > 1e-3
    assert torch.all(ctr == 1)


def test_graph_replays_draw_fresh_actions():
    case = dict(head="mlp", D=4, A=18, H=64, B=8, dynamic=False)
    agent = _agent(case)
    with torch.no_grad():
        agent.actor.p["pi.weight"].zero_()                  # uniform policy: every action equally likely
    s = torch.zeros(2048, 4, device=DEV)
    agent.act_device(s, True)                              # warm-up allocates the workspaces
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        action, _ = agent.act_device(s, True)
    g.replay()
    first = action.clone()
    g.replay()
    torch.cuda.synchronize()
    assert not torch.equal(first, action)
    assert first.min().item() >= 0 and first.max().item() < 18


# ------------------------------------------------------------------------------------------------------- 5. frames
N_LANES, PERIOD, ROUNDS = 4, 8, 6
FCASE = dict(head="cnn", D=[4, 84, 84], A=18, H=64, B=16, dynamic=True)


def _collected(frames):
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    agent = _agent(FCASE, graph=True, buffer_size=256, start_train_step=10 ** 9)
    env = Env("seaquest", num_envs=N_LANES, seed=2, device=DEV)
    assert env.action_size == 18
    if not frames:
        env.frame_stack = False
    rc = ReplayCollector(env, agent, update_period=PERIOD)
    step = 0
    for _ in range(ROUNDS):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    return agent, env, rc


def test_frame_replay_learn_equals_the_stacked_twin():
    agent, _, rc = _collected(frames=True)
    mem = agent.memory
    assert rc.frames is not None and mem.frames is rc.frames and mem.fields["state"].dtype == torch.int64
    assert mem.fields["action"].dtype == torch.int64 and mem.size == N_LANES * PERIOD * ROUNDS
    twin = _agent(FCASE, graph=True, buffer_size=256)
    for x, y in zip(_nets(agent).values(), _nets(twin).values()):
        y.flat.copy_(x.flat)
    twin.memory.store([mem.gather_device(torch.arange(mem.size, device=DEV))])
    assert twin.memory.frames is None
    rs = np.random.RandomState(4)
    for _ in range(3):
        agent._inject_idx = twin._inject_idx = rs.randint(mem.size, size=FCASE["B"])
        ra, rb = agent.learn(), twin.learn()
        assert ra == rb
    torch.cuda.synchronize()
    for (k, x), y in zip(_nets(agent).items(), _nets(twin).values()):
        assert torch.equal(x.flat, y.flat), k


def test_evicted_frame_raises_in_learn():
    from jorldy_b200.core.buffer.frame_store import FrameEvictedError
    agent, env, rc = _collected(frames=True)
    fs = agent.memory.frames
    for _ in range(fs.F + 4):                               # push past the ring without storing into the replay
        next_obs, _, done = env.step_device(None)
        fs.push(env.obs, next_obs, done, env.auto_reset)
    agent._inject_idx = np.arange(FCASE["B"])
    with pytest.raises(FrameEvictedError):
        agent.learn()


# -------------------------------------------------------------------------------------------------- 6. checkpoints
def test_checkpoint_round_trip_keeps_the_sac_layout(tmp_path):
    case = dict(head="mlp", D=4, A=3, H=32, B=4, dynamic=True)
    a = _agent(case, start_train_step=1, buffer_size=64)
    rs = np.random.RandomState(1)
    s = rs.standard_normal((8, 4)).astype(np.float32)
    tr = {"state": s, "next_state": s[::-1].copy(), "reward": np.ones((8, 1)), "done": np.zeros((8, 1), dtype=bool),
          "action": a.act(s, True)["action"]}
    for step in range(1, 4):
        a.process([tr], step)
    a.save(str(tmp_path))
    ck = torch.load(str(tmp_path / "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"actor", "actor_optimizer", "critic1", "critic2", "critic_optimizer1", "critic_optimizer2", "log_alpha",
                       "alpha_optimizer"}
    assert list(ck["actor"]) == ["head.l.weight", "head.l.bias", "l.weight", "l.bias", "pi.weight", "pi.bias"]
    assert list(ck["critic1"]) == ["head.l.weight", "head.l.bias", "l.weight", "l.bias", "q.weight", "q.bias"]
    b = _agent(case, seed=9)
    b.load(str(tmp_path))
    assert torch.equal(b.actor.flat, a.actor.flat)
    assert torch.equal(b.critics[0].flat, a.critics[1].flat)           # critic2's weights land in critic1
    assert torch.equal(b.target_critics[0].flat, a.critics[1].flat)
    assert torch.equal(b.log_alpha.flat, a.log_alpha.flat)
    for k, v in b.actor.state_dict().items():
        assert torch.equal(v.cpu(), ck["actor"][k])


# -------------------------------------------------------------------------------------------------- 7. end to end
@pytest.mark.parametrize("config,extra,sizes", [
    ("config.sac_discrete.cartpole", ["--train.num_workers", "8", "--agent.start_train_step", "64"], (4, 2)),
    ("config.sac_discrete.atari", ["--env.name", "seaquest", "--train.num_workers", "8", "--agent.start_train_step", "16",
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
    assert any(line.startswith("512 step |") and "critic_loss1" in line for line in r.stdout.splitlines()), out[-4000:]
    ckpts = [d for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    saved = torch.load(os.path.join(ckpts[0], "ckpt"), map_location="cpu", weights_only=False)
    D, A = sizes
    kw = dict(head="cnn", hidden_size=64) if config.endswith("atari") else {}
    fresh = Agent("sac", state_size=D, action_size=A, actor="discrete_policy", critic="discrete_q_network",
                  use_dynamic_alpha=True, device=DEV, **kw)
    fresh.load(ckpts[0])
    for k, v in fresh.actor.state_dict().items():
        assert torch.equal(v.cpu(), saved["actor"][k]), k
    for k, v in fresh.critics[0].state_dict().items():
        assert torch.equal(v.cpu(), saved["critic2"][k]), k
    assert torch.equal(fresh.log_alpha.flat[:1].cpu(), saved["log_alpha"].reshape(1))
