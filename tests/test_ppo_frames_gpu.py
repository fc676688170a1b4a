"""PPO on Atari frames (pytest -m gpu): conv1's im2col read from the frame ring (jb_im2col_u8_frames), the frame rollout
(buffer/rollout_buffer.py FrameRollout) filled by RolloutCollector, learn_rollout() on it, and a short training run.

The frame path changes what is stored, never what is computed: the kernel, the collector and learn_rollout() are
checked bit for bit against the gathered stacks, the env and the stacked-input learner.  One learn is also checked
against float64 (test_learn_vs_float64), with tolerances derived as in test_atari_learner_gpu.py
(u = 2^-24, TOL_NET = 7.7e3 u):
  * Gradients of every minibatch, normwise per tensor: TOL_NET (1 + kappa).  TOL_NET bounds the fp32 network's forward
    and backward (the longest chain here, conv1 256 + conv2 512 + conv3 576 + l 3136 + heads 64 terms forward and
    conv1's weight gradient over 16 x 400 rows backward, is shorter than the Ape-X chain that bound was derived for).
    The loss gradient also carries the pre-pass: the advantage and the critic residual v - ret are differences of
    values each within TOL_NET max|v| of exact, so their error relative to their own scale is multiplied by
    kappa = (max|v| + max|ret|) / max|ret - v|, measured on the float64 reference.  As in test_atari_learner_gpu.py
    the float64 network takes the kernels' ReLU masks, after asserting that every disagreement sits within
    TOL_NET max|pre-activation| of zero: a pre-activation within rounding of zero passes or blocks a whole gradient.
  * Each minibatch is recomputed in float64 at the kernel's own parameters before that step, so the comparison does
    not follow a diverged trajectory: the first Adam step is lr g / (|g| + eps), which for |g| ~ eps turns a
    rounding-level gradient difference into an O(lr) parameter difference.
  * Result dict: each statistic is a mean, max or min of per-row terms that are products of at most two quantities
    carrying the error above (ratio x advantage, residual^2), so |got - ref| <= 4 TOL_NET (1 + kappa) S with
    S = max(1, |ref|, max|ret|) the scale of the terms.
  * Parameters and Adam state after all 8 steps: the float64 optimizer twin of test_atari_learner_gpu.py stepped on the
    kernel's own gradients, with its elementwise bounds (KU = 128 u per update)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle_done_steps(seed, n, steps):
    """done[e, k] of the first `steps` steps of auto-reset lanes 0..n-1, from the CPU restatement of the generator."""
    from oracle import frames as of
    out = np.zeros((n, steps), bool)
    for e in range(n):
        f = 1                                            # the reset consumed frame 0
        for k in range(steps):
            _, d = of.events(seed, e, f)
            out[e, k] = d
            f += 2 if d else 1
    return out


def _ppo(T, B, H=64, n_epoch=3, seed=0, **kw):
    from jorldy_b200.core import Agent
    return Agent("ppo", state_size=[4, 84, 84], action_size=4, hidden_size=H, head="cnn", n_step=T, batch_size=B,
                 n_epoch=n_epoch, optim_config={"name": "adam", "lr": 2.5e-4}, run_step=1000, lr_decay=False, device=DEV,
                 seed=seed, **kw)


# ---------------------------------------------------------------------------------------------- 1. the im2col kernel
KN, KT, KSEED = 128, 8, 0      # seed 0 ends episodes of lanes 74, 45 and 91 at steps 0, 1 and 6


@pytest.fixture(scope="module")
def ring():
    """Two rollouts of KT steps of KN lanes on a ring of frames_per_rollout(KT) frames.  Returns the store, the state and
    next references [2KT, KN] (step-major) and the (step, lane) of the states right after an auto-reset."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.buffer.frame_store import FrameStore, frames_per_rollout
    done = _oracle_done_steps(KSEED, KN, 2 * KT)
    after_reset = [(k + 1, e) for e, k in zip(*np.nonzero(done.T)[::-1]) if k + 1 < 2 * KT]
    assert len(after_reset) >= 3
    env = Env("breakout", num_envs=KN, seed=KSEED, device=DEV)
    env.reset_device()
    fs = FrameStore(KN, frames_per_rollout(KT), DEV)
    fs.start(env.obs)
    s_refs, n_refs, dones = [], [], []
    for _ in range(2 * KT):
        next_obs, _, d = env.step_device(None)
        dones.append(d.clone())
        s, x = fs.push(env.obs, next_obs, d, env.auto_reset)
        s_refs.append(s)
        n_refs.append(x)
    assert np.array_equal(torch.stack(dones, 1).cpu().numpy() > 0.5, done)
    return fs, torch.stack(s_refs), torch.stack(n_refs), after_reset


def _reference_col(fs, refs, idx, M):
    """jb_frame_gather of the stacks refs[idx[i]] (idx None: refs[0..M-1]) followed by jb_im2col_u8."""
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    if idx is None:
        stacks, _ = fs.gather(refs[:M], refs[:M])
    else:
        stacks, _ = fs.gather(refs, refs, idx.to(torch.int64))
    col = torch.empty(M * 400, 256, device=DEV)
    C.jb_im2col_u8(ptr(stacks), M, 4, 84, 84, 8, 8, 4, ptr(col), stream_ptr())
    return col, stacks


@pytest.mark.parametrize("M", [1, 7, 256])
@pytest.mark.parametrize("mode", ["null_idx", "idx"])
def test_im2col_frames_equals_gather_then_im2col(ring, M, mode):
    """idx NULL: the second rollout's first stacks (t = 0, 1 of every lane reach 3 frames back into the first rollout).
    idx: unordered draws over every reference of both rollouts with duplicates, the after-reset stacks among them."""
    from jorldy_b200.core.buffer.frame_store import FrameRows
    fs, s_refs, n_refs, after_reset = ring
    if mode == "null_idx":
        refs, idx = s_refs[KT:KT + 2].reshape(-1).contiguous(), None
    else:
        refs = torch.cat([s_refs.reshape(-1), n_refs.reshape(-1)])
        rs = np.random.RandomState(M)
        pick = rs.randint(0, refs.shape[0], M)
        if M > 1:
            forced = [k * KN + e for k, e in after_reset][:M - 1]
            pick[:len(forced)] = forced
            pick[-1] = pick[0]                             # a duplicate
        idx = torch.as_tensor(pick, dtype=torch.int32, device=DEV)
    fs.status.zero_()
    col = torch.full((M * 400, 256), float("nan"), device=DEV)
    FrameRows(fs, refs).im2col(idx, M, col)
    want, stacks = _reference_col(fs, refs, idx, M)
    fs.check()
    assert torch.equal(col, want)
    if mode == "null_idx" and M > 1:
        assert any(bool((stacks[i] != stacks[i, 3:]).any()) for i in range(M))   # not every stack is a reset stack
    if mode == "idx" and M > 1:                            # the after-reset stacks are the first frame tiled x4
        assert bool((stacks[0] == stacks[0, :1]).all())


def test_im2col_frames_evicted_reference_zeroes_and_raises():
    """The short ring of test_evicted_reference_raises_on_the_host (F = 8): the first step's references are overwritten
    after 12 steps; their rows are zero (as gather + im2col gives), the resident ones are the stacks', and the status
    word raises on the host."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.buffer.frame_store import FrameEvictedError, FrameRows, FrameStore
    env = Env("breakout", num_envs=2, seed=1, device=DEV)
    env.reset_device()
    fs = FrameStore(2, 8, DEV)
    fs.start(env.obs)
    refs = []
    for _ in range(12):
        next_obs, _, done = env.step_device(None)
        refs.append(fs.push(env.obs, next_obs, done, env.auto_reset)[0])
    rows = torch.cat([refs[-1], refs[0]])                # resident, resident, evicted, evicted
    col = torch.full((4 * 400, 256), float("nan"), device=DEV)
    FrameRows(fs, rows).im2col(None, 4, col)
    with pytest.raises(FrameEvictedError):
        fs.check()
    want, _ = _reference_col(fs, rows, None, 4)
    assert torch.equal(col, want)
    assert int(torch.count_nonzero(col[800:]).item()) == 0 and int(torch.count_nonzero(col[:800]).item()) > 0


# ------------------------------------------------------------------------------------------------- 2. the collector
CN, CT, CSEED = 256, 8, 0      # seed 0: episode ends inside rollouts and at the last step of one (see the asserts)


@pytest.mark.parametrize("use_graph", [False, True])
def test_collector_rollouts_equal_a_lockstep_env(use_graph):
    """Three collect() calls.  Every (n, t) stack rebuilt from the rollout equals the observation of an independent env
    with the same seed stepped in lockstep (the generator ignores actions); so do rewards, dones and last_next_state.
    The CUDA-graph collector runs one warm-up rollout before its capture, so its three rollouts are env steps T..4T."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.buffer import FrameRollout
    from jorldy_b200.core.collect import RolloutCollector
    lo = CT if use_graph else 0
    done = _oracle_done_steps(CSEED, CN, lo + 3 * CT)[:, lo:]
    ks = np.nonzero(done)[1]
    assert any(k % CT < CT - 1 for k in ks) and any(k % CT == CT - 1 and k < 2 * CT for k in ks)
    agent = _ppo(CT, 64)
    col = RolloutCollector(Env("breakout", num_envs=CN, seed=CSEED, device=DEV), agent, use_cuda_graph=use_graph)
    assert isinstance(col.rollout, FrameRollout) and not hasattr(col.rollout, "state")
    twin = Env("breakout", num_envs=CN, seed=CSEED, device=DEV)
    twin.reset_device()
    for r in range(3):
        ro = col.collect()
        if use_graph and r == 0:
            for _ in range(CT):
                twin.step_device(None)
        states, rewards, dones = [], [], []
        for _ in range(CT):
            states.append(twin.obs.clone())
            next_obs, rew, d = twin.step_device(None)
            rewards.append(rew.clone())
            dones.append(d.clone())
        refs = ro.state_ref.reshape(-1)
        got, _ = ro.frames.gather(refs, refs)
        last, _ = ro.frames.gather(ro.last_next_state, ro.last_next_state)
        ro.frames.check()
        assert torch.equal(got.view(CN, CT, 4, 84, 84), torch.stack(states, 1)), f"rollout {r} states"
        assert torch.equal(last, next_obs), f"rollout {r} last_next_state"
        assert torch.equal(ro.reward, torch.stack(rewards, 1)) and torch.equal(ro.done, torch.stack(dones, 1))
        assert np.array_equal(ro.done.cpu().numpy() > 0.5, done[:, r * CT:(r + 1) * CT])


# ------------------------------------------------------------------------------------ 3. learn against the stacked twin
@pytest.mark.parametrize("use_graph", [False, True])
def test_learn_rollout_equals_learn_on_materialised_stacks(use_graph):
    """16 envs x 32 steps, B = 24: 21 full minibatches (16 of them in one CUDA graph on the graph path) and a ragged
    tail of 8, over 3 epochs.  learn_rollout() on the frame rollout and _learn_tensors() on its gathered uint8 stacks
    give the same results, parameters and Adam state, bit for bit."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import RolloutCollector
    N, T, B = 16, 32, 24
    a = _ppo(T, B, use_cuda_graph=use_graph)
    b = _ppo(T, B, use_cuda_graph=use_graph)
    b.network.load_state_dict(a.network.state_dict())
    ro = RolloutCollector(Env("breakout", num_envs=N, seed=5, device=DEV), a, use_cuda_graph=False).collect()
    refs = ro.state_ref.reshape(-1)
    stacks, _ = ro.frames.gather(refs, refs)
    last, _ = ro.frames.gather(ro.last_next_state, ro.last_next_state)
    action, reward, done = ro.action.reshape(-1).clone(), ro.reward.reshape(-1).clone(), ro.done.reshape(-1).clone()
    rs = np.random.RandomState(11)
    perms = [rs.permutation(N * T) for _ in range(3)]
    a._inject_perms = b._inject_perms = perms
    for _ in range(2):                                   # the second learn replays the captured graphs
        ra = a.learn_rollout(ro)
        rb = b._learn_tensors(stacks, action, reward, done, last_next_state=last)
        assert ra == rb
        ro.t = T
    torch.cuda.synchronize()
    assert bool(a._graphs) == use_graph
    assert torch.equal(a.network.flat, b.network.flat)
    assert all(torch.equal(x, y) for x, y in zip(a.optimizer.state_tensors(), b.optimizer.state_tensors()))


# ------------------------------------------------------------------------------------------- 4. learn against float64
U = 2.0 ** -24
TOL_NET = 7.7e3 * U


def _masked_policy_value(masks):
    """oracle.nets.discrete_policy_value with the kernels' ReLU masks (masks[0..3]: conv1..3 and l; post-ReLU kernel
    activations of the same rows)."""
    import torch.nn.functional as F
    from test_atari_learner_gpu import _relu_mask

    def f(p, x):
        h = x / 255.0
        for li, (name, stride) in enumerate((("conv1", 4), ("conv2", 2), ("conv3", 1))):
            pre = F.conv2d(h, p[f"head.{name}.weight"], p[f"head.{name}.bias"], stride=stride)
            h = pre * _relu_mask(pre, masks[li], name)
        pre = F.linear(h.reshape(x.shape[0], -1), p["l.weight"], p["l.bias"])
        h = pre * _relu_mask(pre, masks[3], "l")
        pi = torch.exp(F.log_softmax(F.linear(h, p["pi.weight"], p["pi.bias"]), dim=-1))
        return pi, F.linear(h, p["v.weight"], p["v.bias"])
    return f


def test_learn_vs_float64(monkeypatch):
    """N=4, T=16, H=64, A=4, B=16, 2 epochs (8 Adam steps, the eager minibatch path) on a collected frame rollout."""
    from oracle import nets as onets
    from oracle import ppo as oppo
    from test_atari_learner_gpu import _OptTwin, _normwise
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import RolloutCollector
    N, T, B, E, LR = 4, 16, 16, 2, 2.5e-4
    agent = _ppo(T, B, n_epoch=E, seed=21)
    net = agent.network
    ro = RolloutCollector(Env("breakout", num_envs=N, seed=2, device=DEV), agent, use_cuda_graph=False).collect()
    refs = ro.state_ref.reshape(-1)
    stacks, _ = ro.frames.gather(refs, refs)
    last, _ = ro.frames.gather(ro.last_next_state, ro.last_next_state)
    p0 = {k: v.detach().cpu().clone() for k, v in net.p.items()}
    rs = np.random.RandomState(4)
    perms = [rs.permutation(N * T) for _ in range(E)]
    agent._inject_perms = perms

    steps = []                                             # per Adam step: parameters before it, its gradients, masks
    orig_step = agent.optimizer.step
    layers = net.head.layers

    def step(max_norm=None):
        masks = [net._buf(f"mb{B}.head.y{li}", (B * oh * ow, co)).view(B, oh, ow, co).permute(0, 3, 1, 2).cpu()
                 for li, (_, _, co, _, _, _, (oh, ow)) in enumerate(layers)]
        masks.append(net._buf(f"mb{B}.h2", (B, net.D_hidden)).cpu())
        steps.append(({k: v.detach().cpu().double() for k, v in net.p.items()},
                      [net.g[k].detach().clone() for k in net.p], masks))
        return orig_step(max_norm=max_norm)
    agent.optimizer.step = step
    res = agent.learn_rollout(ro)
    torch.cuda.synchronize()
    assert len(steps) == E * (N * T // B)

    # float64 pre-pass and GAE through oracle/ppo.learn (forward only: the ReLU masks do not matter there)
    nxt = stacks.view(N, T, 4, 84, 84).clone()
    nxt[:, :-1] = nxt[:, 1:].clone()                       # V(s') of row (n, t) is V(state[n, t+1]); masked where done
    nxt[:, -1] = last
    batch = {"state": stacks.cpu().double(), "next_state": nxt.view(N * T, 4, 84, 84).cpu().double(),
             "action": ro.action.reshape(-1, 1).cpu().double(), "reward": ro.reward.reshape(-1, 1).cpu().double(),
             "done": ro.done.reshape(-1, 1).cpu().double()}
    hp = {"continuous": False, "n_step": T, "gamma": agent.gamma, "lambda": agent._lambda, "standardize": True,
          "batch_size": B, "n_epoch": E, "eps_clip": agent.epsilon_clip, "vf_coef": agent.vf_coef,
          "ent_coef": agent.ent_coef, "clip_grad_norm": agent.clip_grad_norm}
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        pre = oppo.learn({k: v.double() for k, v in p0.items()}, batch, hp, perms, lr=LR, max_minibatches=1)
        value, ret, adv, logp = pre["value"], pre["ret"], pre["adv"], pre["log_prob_old"]
        kappa = (value.abs().max() + ret.abs().max()).item() / (ret - value).abs().max().item()
        tol = TOL_NET * (1 + kappa)
        stats = {k: [] for k in ("actor_loss", "critic_loss", "entropy_loss", "max_ratio", "min_prob")}
        for j, (pj, grads, masks) in enumerate(steps):
            idx = np.asarray(perms[j // (N * T // B)])[(j % (N * T // B)) * B:][:B]
            p = {k: v.clone().requires_grad_(True) for k, v in pj.items()}
            monkeypatch.setattr(onets, "discrete_policy_value", _masked_policy_value(masks))
            loss, aux = oppo.minibatch_loss(p, batch["state"][idx], batch["action"][idx], value[idx], ret[idx], adv[idx],
                                            logp[idx], False, hp["eps_clip"], hp["vf_coef"], hp["ent_coef"])
            monkeypatch.undo()
            loss.backward()
            for k, g in zip(net.p, grads):
                _normwise(g, p[k].grad, tol, f"step {j} grad {k}")
            for k in stats:
                stats[k].append(aux[k].item())
    finally:
        torch.set_default_dtype(prev)
    ref = {"actor_loss": np.mean(stats["actor_loss"]), "critic_loss": np.mean(stats["critic_loss"]),
           "entropy_loss": np.mean(stats["entropy_loss"]), "max_ratio": max(stats["max_ratio"]),
           "min_prob": min(stats["min_prob"]), "mean_ret": pre["mean_ret"]}
    scale_ret = ret.abs().max().item()
    for k, v in ref.items():
        bound = 4 * tol * max(1.0, abs(v), scale_ret)
        assert abs(res[k] - v) <= bound, f"{k}: {res[k]} vs float64 {v} (bound {bound:.2e})"

    twin = _OptTwin("adam", list(p0.values()), LR, 1e-8)
    for _, grads, _ in steps:
        twin.step(grads, agent.clip_grad_norm)
    state = agent.optimizer.state_dict()["state"]
    for i, k in enumerate(net.p):
        twin.check(i, net.p[k], state[i], k)


# ------------------------------------------------------------------------------------------------------ 5. end to end
def test_sync_training_run_on_frames(tmp_path):
    """`python -m jorldy_b200.main --sync --config config.ppo.atari` (the built-in Atari configs name no game, so
    --env.name picks one): 16 envs, 512 steps.  run_mode prints a traceback instead of raising, so the output is
    checked: the last step line, and a checkpoint that loads into a fresh agent with an identical state_dict."""
    from jorldy_b200.core import Agent
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable, "-m", "jorldy_b200.main", "--sync", "--config", "config.ppo.atari", "--env.name", "breakout",
           "--train.num_workers", "16", "--train.run_step", "512", "--train.print_period", "256",
           "--train.save_period", "512"]
    r = subprocess.run(cmd, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith("512 step |") for line in r.stdout.splitlines()), out[-4000:]
    ckpts = [os.path.join(d, "ckpt") for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    saved = torch.load(ckpts[0], map_location="cpu", weights_only=False)["network"]
    fresh = Agent("ppo", state_size=[4, 84, 84], action_size=4, network="discrete_policy_value", head="cnn", device=DEV,
                  run_step=512)
    fresh.load(os.path.dirname(ckpts[0]))
    got = fresh.network.state_dict()
    assert sorted(got) == sorted(saved)
    for k, v in saved.items():
        assert torch.equal(got[k].cpu(), v), k
