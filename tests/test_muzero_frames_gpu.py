"""MuZero on Atari frames on the GPU: the frame + action-plane im2col against a gather and a materialised 8-channel
jb_im2col_u8, its eviction status, the CNN representation and one learn against the float64 oracle (oracle/muzero.py),
reproducibility, the graph act against its eager twin, the collector's windows, checkpoints and an end-to-end
`jorldy_b200.main --sync` run on `config.muzero.atari`."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import muzero_frames as omf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
POS_MASK = (1 << 40) - 1


def _C():
    from jorldy_b200.core.dev import C
    return C


def ptr(t):
    return 0 if t is None else t.data_ptr()


def _agent(A=4, **kw):
    from jorldy_b200.core import Agent
    args = dict(state_size=[4, 84, 84], action_size=A, head="cnn", hidden_size=32, latent_size=16, num_simulation=4,
                num_unroll=3, td_steps=4, value_support=5, reward_support=1, batch_size=16, buffer_size=256,
                start_train_step=0, optim_config={"name": "adam", "lr": 1e-3}, run_step=1000, lr_decay=False,
                device=DEV, seed=3)
    args.update(kw)
    return Agent("muzero", **args)


def _filled_store(n, F, steps, seed, p_done=0.25):
    """A FrameStore of n lanes after `steps` pushes of random frames with random auto-resets; returns it and the
    state references of every step, int64 [steps * n], step-major."""
    from jorldy_b200.core.buffer.frame_store import FrameStore
    g = torch.Generator().manual_seed(seed)
    rnd = lambda: torch.randint(0, 256, (n, 4, 84, 84), generator=g, dtype=torch.uint8).to(DEV)
    store = FrameStore(n, F, DEV)
    store.start(rnd())
    refs = []
    for _ in range(steps):
        done = (torch.rand(n, generator=g) < p_done).float().to(DEV)
        s, _ = store.push(rnd(), rnd(), done, True)
        refs.append(s.clone())
    return store, torch.cat(refs)


def _planes_f32(store, refs, actions, A):
    """The kernel's plane values, computed independently: a / A rounded once to f32 (the f64 quotient of two small
    integers rounds to the same f32 as an IEEE f32 division; torch's CUDA division by a scalar multiplies by the
    reciprocal, which does not) where frame k follows an action, else 0."""
    p = refs & POS_MASK
    lane = refs >> 40
    f = store.first[lane, p % store.F]
    live = (p.view(-1, 1) - 3 + torch.arange(4, device=DEV)) > f.view(-1, 1)
    q = torch.as_tensor((actions.cpu().numpy().astype(np.float64) / A).astype(np.float32)).to(DEV)
    return torch.where(live, q, torch.zeros((), device=DEV)), p, f


def _im2col_reference(store, refs, actions, A, idx):
    """jb_frame_gather, then jb_im2col_u8 over a materialised [M, 8, 84, 84] input whose planes are written into the
    column matrix as the f32 values they hold."""
    C = _C()
    sel = torch.arange(refs.shape[0], device=DEV) if idx is None else idx.long()
    stacks, _ = store.gather(refs, refs, None if idx is None else idx.long())
    M = stacks.shape[0]
    x8 = torch.cat([stacks, torch.zeros_like(stacks)], 1).contiguous()
    col = torch.empty(M * 400, 512, device=DEV)
    C.jb_im2col_u8(ptr(x8), M, 8, 84, 84, 8, 8, 4, ptr(col), 0)
    planes, _, _ = _planes_f32(store, refs[sel], actions[sel], A)
    col.view(M, 400, 8, 64)[:, :, 4:, :] = planes.view(M, 1, 4, 1)
    return col, stacks


@pytest.mark.parametrize("M", [1, 7, 256])
@pytest.mark.parametrize("idx_kind", ["null", "duplicated", "unordered"])
def test_im2col_frames_actions_bit_equal_to_gather_and_im2col(M, idx_kind):
    from jorldy_b200.core.buffer.frame_store import FrameActionRows
    n, A = 4, 18
    store, refs = _filled_store(n, 256, 60, seed=M)
    g = torch.Generator().manual_seed(M + 1)
    src = refs[torch.randperm(refs.shape[0], generator=g)[:M].to(DEV)] if M <= refs.shape[0] else \
        refs[torch.randint(0, refs.shape[0], (M,), generator=g).to(DEV)]
    actions = torch.randint(0, A, (M, 4), generator=g).to(DEV)
    idx = {"null": None, "duplicated": torch.randint(0, M, (M,), generator=g).to(DEV),
           "unordered": torch.randperm(M, generator=g).to(DEV)}[idx_kind]
    idx = None if idx is None else idx.to(torch.int32).contiguous()
    src = src.contiguous()
    col = torch.full((M * 400, 512), float("nan"), device=DEV)
    FrameActionRows(store, src, actions, A).im2col(idx, M, col)
    ref, _ = _im2col_reference(store, src, actions, A, idx)
    torch.cuda.synchronize()
    assert torch.equal(col, ref)
    store.check()
    # the checked rows include stacks that reach back across a reset (a zero plane next to a non-zero one)
    planes, p, f = _planes_f32(store, src, actions, A)
    if M == 256:
        assert bool(((p - 3 < f) & (p > f)).any())


def test_im2col_frames_actions_evicted_reference_is_zero_filled_and_raised():
    from jorldy_b200.core.buffer.frame_store import FrameActionRows, FrameEvictedError
    store, refs = _filled_store(2, 8, 40, seed=5, p_done=0.0)
    src = torch.stack([refs[0], refs[-2]]).contiguous()          # the first is long overwritten, the second resident
    actions = torch.ones(2, 4, dtype=torch.int64, device=DEV)
    col = torch.full((2 * 400, 512), float("nan"), device=DEV)
    FrameActionRows(store, src, actions, 4).im2col(None, 2, col)
    with pytest.raises(FrameEvictedError):
        store.check()
    assert torch.equal(col[:400], torch.zeros(400, 512, device=DEV))
    ref, _ = _im2col_reference(store, src[1:], actions[1:], 4, None)
    assert torch.equal(col[400:], ref)


def _oracle_input(store, refs, actions, A):
    stacks, _ = store.gather(refs, refs)
    planes, _, _ = _planes_f32(store, refs, actions, A)
    return omf.frame_action_input(stacks.cpu().numpy(), planes.double().cpu())


def test_representation_on_frames_fwd_bwd_vs_float64():
    from jorldy_b200.core.buffer.frame_store import FrameActionRows
    A, M = 18, 32
    agent = _agent(A=A, latent_size=32)
    net = agent.network
    store, refs = _filled_store(4, 256, 40, seed=11)
    g = torch.Generator().manual_seed(12)
    src = refs[torch.randperm(refs.shape[0], generator=g)[:M].to(DEV)].contiguous()
    actions = torch.randint(0, A, (M, 4), generator=g).to(DEV)
    ds = torch.randn(M, net.Hs, generator=g).to(DEV)
    h1, pre, s = (torch.empty(M, d, device=DEV) for d in (net.D_repr, net.Hs, net.Hs))
    net.represent(FrameActionRows(store, src, actions, A), h1, pre, s, tag="t.")
    dpre, dh1 = torch.empty_like(pre), torch.empty_like(h1)
    net.scale_bwd(pre, ds, dpre)
    net.represent_bwd(None, h1, dpre, dh1, tag="t.")
    torch.cuda.synchronize()
    p = {k: v.double().cpu().requires_grad_(True) for k, v in net.state_dict().items()}
    x = _oracle_input(store, src, actions, A)
    ref = omf.represent(p, x)
    (ref * ds.double().cpu()).sum().backward()
    np.testing.assert_allclose(s.cpu().numpy(), ref.detach().numpy(), atol=2e-4)
    names = [k for k in p if k.startswith("head.") or k.startswith("h.")]
    assert names == ["head.conv1.weight", "head.conv1.bias", "head.conv2.weight", "head.conv2.bias", "head.conv3.weight",
                     "head.conv3.bias", "h.l.weight", "h.l.bias"]
    assert tuple(net.p["head.conv1.weight"].shape) == (32, 8, 8, 8)
    for k in names:
        gr = p[k].grad.numpy()
        np.testing.assert_allclose(net.g[k].double().cpu().numpy(), gr, rtol=2e-3, atol=2e-3 * float(np.abs(gr).max()),
                                   err_msg=k)


def _stored_windows(agent, store, refs, W, seed):
    """W windows on `store`'s references, with random prev_actions and the flat fields of tests/test_muzero_gpu.py."""
    rng = np.random.default_rng(seed)
    K, n, A = agent.K, agent.n_step, agent.action_size
    L = K + n + 1
    done = np.zeros((W, L), dtype=np.float32)
    done[::2, K // 2 + 1] = 1
    pol = rng.random((W, L, A)).astype(np.float32)
    bt = dict(reward=rng.normal(size=(W, L)).astype(np.float32), done=done,
              root_value=(rng.normal(size=(W, L)) * 5).astype(np.float32),
              policy=(pol / pol.sum(-1, keepdims=True)).astype(np.float32), action=rng.integers(0, A, (W, L)))
    w = {k: torch.as_tensor(v).to(DEV) for k, v in bt.items()}
    w["state"] = refs[torch.as_tensor(rng.integers(0, refs.shape[0], W)).to(DEV)].contiguous()
    w["prev_actions"] = torch.as_tensor(rng.integers(0, A, (W, 4))).to(DEV)
    agent._frames = store
    agent.memory.store([w])


def test_one_learn_on_frames_vs_oracle():
    A = 18
    agent = _agent(A=A)
    store, refs = _filled_store(4, 256, 40, seed=21)
    _stored_windows(agent, store, refs, 64, seed=0)
    u_a = np.random.default_rng(1).random(agent.batch_size)
    u_b = np.random.default_rng(2).random(agent.batch_size)
    ua, ub = (torch.as_tensor(u, dtype=torch.float64, device=DEV) for u in (u_a, u_b))
    batch, weights, idx, _ = agent.memory.sample_device(agent.beta, agent.batch_size, ua, ub)
    agent.memory._sample_ctr -= 1
    agent._inject_per_u = (u_a, u_b)
    params = {k: v.double().cpu() for k, v in agent.network.state_dict().items()}
    hp = dict(K=agent.K, n=agent.n_step, V=agent.V, R=agent.R, gamma=agent.gamma, value_loss_coef=agent.value_loss_coef,
              alpha=agent.alpha, A=A)
    bt = {k: v.cpu().numpy() for k, v in batch.items() if k not in ("state", "prev_actions")}
    bt["state"] = _oracle_input(store, batch["state"], batch["prev_actions"], A)
    lr = 1e-3
    new, st, prio, grads = omf.learn(params, bt, weights.cpu().numpy(), hp, lr, 5.0)
    res = agent.learn()
    torch.cuda.synchronize()
    assert set(res) == {"loss", "value_loss", "reward_loss", "policy_loss", "sampled_p", "mean_p", "num_learn"}
    for k in ("loss", "value_loss", "reward_loss", "policy_loss"):
        assert abs(res[k] - st[k]) < 1e-4 * max(1.0, abs(st[k])), (k, res[k], st[k])
    for k, g in grads.items():
        np.testing.assert_allclose(agent.network.g[k].double().cpu().numpy(), g.numpy(), rtol=2e-3,
                                   atol=2e-3 * float(g.abs().max()) + 1e-7, err_msg=k)
    for k, v in new.items():
        # Adam's first step is lr * g / (|g| + eps), close to lr * sign(g): entries whose gradient is within the f32
        # error of zero may step either way, so they get 2 lr; the others must match closely
        got, want, g = agent.network.p[k].double().cpu().numpy(), v.numpy(), grads[k].abs().numpy()
        firm = g > 1e-2 * g.max()
        np.testing.assert_allclose(got[firm], want[firm], rtol=1e-4, atol=5e-5, err_msg=k)
        np.testing.assert_allclose(got, want, atol=2 * lr + 1e-6, err_msg=k)
    tree = agent.memory._tree.cpu().numpy()
    last = {int(i): j for j, i in enumerate(idx.cpu().numpy())}
    for i, j in last.items():
        np.testing.assert_allclose(tree[i], prio[j].item(), rtol=1e-4, atol=1e-5)


def test_two_learns_on_frames_are_bit_identical():
    outs = []
    for _ in range(2):
        agent = _agent()
        store, refs = _filled_store(4, 256, 40, seed=31)
        _stored_windows(agent, store, refs, 64, seed=3)
        agent._inject_per_u = (np.linspace(0.01, 0.99, 16), np.linspace(0.02, 0.98, 16))
        r1 = agent.learn()
        r2 = agent.learn()
        outs.append((agent.network.flat.clone(), agent.optimizer.exp_avg.clone(), r1, r2))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][2:] == outs[1][2:]


def _attached(agent, N, seed):
    """attach_frames on an N-lane frame-stack env stand-in, then a few pushes with resets."""
    env = types.SimpleNamespace(frame_stack=True, num_envs=N)
    store = agent.attach_frames(env)
    g = torch.Generator().manual_seed(seed)
    rnd = lambda: torch.randint(0, 256, (N, 4, 84, 84), generator=g, dtype=torch.uint8).to(DEV)
    store.start(rnd())
    for _ in range(5):
        store.push(rnd(), rnd(), (torch.rand(N, generator=g) < 0.3).float().to(DEV), True)
    return store, rnd


def test_graph_act_on_frames_bit_identical_to_eager_with_fresh_noise():
    N = 32
    res = []
    for graph in (True, False):
        agent = _agent(use_cuda_graph=graph)
        store, rnd = _attached(agent, N, seed=4)
        g = torch.Generator().manual_seed(8)
        steps = []
        for t in range(4):
            hist = agent._hist.clone()
            a, v = agent.act_device(rnd(), training=True)
            st = agent._search_state(N)
            steps.append((a.clone(), v.clone(), agent.step_inputs["policy"].clone(), st["p"][:, 0].clone(),
                          agent.step_inputs["prev_actions"].clone(), agent._hist.clone(), hist))
            store.push(rnd(), rnd(), (torch.rand(N, generator=g) < 0.3).float().to(DEV), True)
        res.append(steps)
        if graph:
            assert (N, True) in agent._graphs
    for s1, s2 in zip(*res):
        for x1, x2 in zip(s1, s2):
            assert torch.equal(x1, x2)
    for a, _, _, _, prev, hist_after, hist_before in res[0]:
        assert torch.equal(prev, hist_before)                       # the root saw the history before the act
        assert torch.equal(hist_after, torch.cat([hist_before[:, 1:], a.view(-1, 1)], 1))
    priors = [s[3] for s in res[0]]
    assert all(not torch.equal(priors[i], priors[i + 1]) for i in range(3))


def test_collector_windows_on_frames_match_a_step_record():
    """Every stored window equals the step-by-step record: its reference gathers the stack acted on, its prev_actions
    are the lane's last four actions before that step, and its fields are what act and env.step_device gave; some
    windows run across an episode end."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    N, T = 512, 24
    env = Env("breakout", num_envs=N, seed=0)
    agent = _agent(start_train_step=10 ** 9, buffer_size=N * T, use_cuda_graph=False)
    col = ReplayCollector(env, agent, update_period=1)
    step_device, rec = env.step_device, []

    def recorded_step(action):
        out = step_device(action)
        rec[-1].update(reward=out[1].view(-1).clone(), done=out[2].view(-1).clone())
        return out
    env.step_device = recorded_step
    for _ in range(T):
        rec.append({"state": env.obs.clone(), "prev_actions": agent._hist.clone()})
        col.run_round(0)
        rec[-1].update(action=agent._search_state(N)["action"].clone(),
                       root_value=agent.step_inputs["root_value"].clone(), policy=agent.step_inputs["policy"].clone())
    L = agent.L
    assert agent.memory.size == (T - L + 1) * N
    for t in range(T):                   # the history is the last four actions, whatever the episode boundaries
        want = torch.stack([rec[t - 4 + k]["action"] if t - 4 + k >= 0 else torch.zeros(N, dtype=torch.int64,
                                                                                          device=DEV) for k in range(4)], 1)
        assert torch.equal(rec[t]["prev_actions"], want), t
    spans_episode_end = False
    for t0 in range(T - L + 1):
        w = agent.memory.gather_device(torch.arange(t0 * N, (t0 + 1) * N, device=DEV))
        stacks, _ = agent._frames.gather(w["state"], w["state"])
        assert torch.equal(stacks, rec[t0]["state"]), t0
        assert torch.equal(w["prev_actions"], rec[t0]["prev_actions"]), t0
        for i in range(L):
            for k in ("action", "reward", "done", "root_value", "policy"):
                assert torch.equal(w[k][:, i], rec[t0 + i][k]), (t0, i, k)
        spans_episode_end |= bool((w["done"][:, :L - 1] != 0).any())
    agent._frames.check()
    assert spans_episode_end


def test_checkpoint_round_trip_on_frames(tmp_path):
    agent = _agent()
    store, refs = _filled_store(4, 256, 40, seed=41)
    _stored_windows(agent, store, refs, 64, seed=4)
    agent.learn()
    agent.save(str(tmp_path))
    ck = torch.load(os.path.join(tmp_path, "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck) == {"network", "optimizer"} and list(ck["network"]) == list(agent.network.p)
    assert tuple(ck["network"]["head.conv1.weight"].shape) == (32, 8, 8, 8)
    assert tuple(ck["network"]["h.l.weight"].shape) == (16, 3136)
    b = _agent(seed=9)
    b.load(str(tmp_path))
    assert torch.equal(b.network.flat, agent.network.flat)
    assert torch.equal(b.optimizer.exp_avg, agent.optimizer.exp_avg)


def test_sync_training_run_on_atari_with_save_and_load(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    final = 200
    base = [sys.executable, "-m", "jorldy_b200.main", "--sync", "--config", "config.muzero.atari", "--env.name",
            "breakout", "--train.run_step", str(final), "--train.print_period", str(final // 2), "--train.save_period",
            str(final), "--train.num_workers", "8", "--train.update_period", "4", "--agent.start_train_step", "40",
            "--agent.batch_size", "16", "--agent.buffer_size", "2048", "--agent.num_simulation", "4",
            "--agent.hidden_size", "64", "--agent.latent_size", "32"]
    r = subprocess.run(base, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert "Traceback" not in out, out[-4000:]
    assert any(line.startswith(f"{final} step |") for line in r.stdout.splitlines()), out[-4000:]
    assert any("policy_loss" in line for line in r.stdout.splitlines() if " step |" in line), out[-4000:]
    ckpts = [d for d, _, files in os.walk(tmp_path / "logs") if "ckpt" in files]
    assert len(ckpts) == 1, ckpts
    r2 = subprocess.run(base + ["--train.load_path", ckpts[0]], cwd=tmp_path / "logs", env=env, capture_output=True,
                        text=True, timeout=900)
    out2 = r2.stdout + r2.stderr
    assert "Traceback" not in out2 and "Load model from" in out2, out2[-4000:]
