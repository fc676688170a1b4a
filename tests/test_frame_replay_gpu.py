"""Single-frame Atari replay (core/buffer/frame_store.py, csrc/frame_ring.cu) vs the env, the CPU oracle and the duplicated
stack layout (pytest -m gpu).  Every comparison is bit-exact: the layout changes what is stored, never what is sampled."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _oracle_dones(seed, n, T, auto_reset):
    """Episode ends of the first T steps of lanes 0..n-1, from the CPU restatement of the generator."""
    from oracle import frames as of
    count = 0
    for e in range(n):
        f = 1                                            # the reset consumed frame 0
        for _ in range(T):
            _, d = of.events(seed, e, f)
            count += int(d)
            f += 2 if (d and auto_reset) else 1
    return count


# ------------------------------------------------------------------------------------------- 1. stacks equal the env
@pytest.mark.parametrize("n,T,seed,min_dones", [(16, 300, 29, 8), (1, 250, 9, 2)])
def test_gathered_stacks_equal_the_env(n, T, seed, min_dones):
    """Every state / next_state the env produced comes back from its frame references, including reset stacks (first
    frame tiled x4), terminal next_states (the stack before the auto-reset) and, for one env, episodes that continue
    through a done."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.buffer.frame_store import FrameStore
    dones = _oracle_dones(seed, n, T, auto_reset=n > 1)
    assert dones >= min_dones
    env = Env("breakout", num_envs=n, seed=seed, device=DEV)
    assert env.auto_reset == (n > 1)
    env.reset_device()
    fs = FrameStore(n, 2 * T + 8, DEV)
    fs.start(env.obs)
    states, nexts, s_refs, n_refs, gpu_dones = [], [], [], [], 0
    for _ in range(T):
        states.append(env.obs.clone())
        next_obs, _, done = env.step_device(None)
        nexts.append(next_obs.clone())
        gpu_dones += int(done.sum().item())
        s, x = fs.push(env.obs, next_obs, done, env.auto_reset)
        s_refs.append(s)
        n_refs.append(x)
    assert gpu_dones == dones
    st, nx = fs.gather(torch.cat(s_refs), torch.cat(n_refs))
    fs.check()
    assert torch.equal(st, torch.cat(states))
    assert torch.equal(nx, torch.cat(nexts))
    if not env.auto_reset:                              # one env: a done does not start an episode, so every step acts on
        assert torch.equal(torch.cat(n_refs)[:-n], torch.cat(s_refs)[n:])     # the previous step's next_state


# ---------------------------------------------------------------- 2. ring contents equal the oracle loop and the stack twin
N, P, ROUNDS, CAP, SEED = 16, 4, 12, 400, 68          # 48 steps of 16 lanes into 400 slots: the ring wraps; seed 68 ends
                                                      # episodes at steps 8, 18, 36 and 40


def _agent(name, seed=3):
    from jorldy_b200.core import Agent
    kw = dict(state_size=[4, 84, 84], action_size=4, hidden_size=128, head="cnn", buffer_size=CAP, batch_size=16, n_step=3,
              start_train_step=10 ** 9, device=DEV, run_step=1000, lr_decay=False, seed=seed)
    if name == "ape_x":
        kw.update(network="dueling", num_workers=N)
    if name == "rainbow":
        kw.update(v_min=-1, v_max=10, num_support=51)
    return Agent(name, **kw)


def _collect(name, frames):
    """ROUNDS rounds of a ReplayCollector; frames=False keeps the duplicated stack layout (the path of a non-frame env)."""
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    torch.manual_seed(0)                                  # Rainbow's warm-up actions come from torch.randint
    agent = _agent(name)
    env = Env("breakout", num_envs=N, seed=SEED, device=DEV)
    if not frames:
        env.frame_stack = False
    rc = ReplayCollector(env, agent, update_period=P)
    assert (rc.frames is not None) == frames
    step = 0
    for _ in range(ROUNDS):
        step, _ = rc.run_round(step)
    torch.cuda.synchronize()
    return agent


def _oracle_ring(apex):
    """oracle.frames.FramesBatch through one oracle.collect.NStepWindow per lane, written step-major into CAP slots."""
    from oracle import collect as oc
    from oracle.frames import FramesBatch
    env = FramesBatch(N, seed=SEED, stream_base=0, auto_reset=True)
    obs = env.reset()
    wins = [oc.NStepWindow(3, apex=apex, gamma=0.99) for _ in range(N)]
    rows = []
    for _ in range(P * ROUNDS):
        state = obs.copy()
        next_obs, reward, done = env.step()
        for i in range(N):
            tr = {"state": state[i:i + 1], "action": np.zeros((1, 1), np.int64), "reward": reward[i:i + 1],
                  "done": done[i:i + 1], "next_state": next_obs[i:i + 1]}
            if apex:
                tr["q"] = np.zeros(1, np.float32)
            out = wins[i].push(tr)
            if out:
                rows.append(out)
        obs = env.obs
    ring = [None] * CAP
    for k, r in enumerate(rows):
        ring[k % CAP] = r
    return ring, len(rows)


@pytest.mark.parametrize("name", ["multistep", "rainbow", "ape_x"])
def test_ring_contents_equal_oracle_loop_and_stack_twin(name):
    agent = _collect(name, frames=True)
    twin = _collect(name, frames=False)
    mem, tmem = agent.memory, twin.memory
    assert mem.frames is not None and tmem.frames is None
    ring, emitted = _oracle_ring(name == "ape_x")
    assert emitted > CAP and mem.size == tmem.size == CAP and mem.buffer_index == tmem.buffer_index
    assert mem.fields["state"].dtype == torch.int64 and mem.fields["state"].dim() == 1
    idx = torch.arange(CAP, device=DEV)
    got, ref = mem.gather_device(idx), tmem.gather_device(idx)
    mem.check_frames()
    assert list(got) == list(ref)
    for k in ref:
        assert torch.equal(got[k], ref[k]), k
    state, nxt = got["state"].cpu().numpy(), got["next_state"].cpu().numpy()
    reward, done = got["reward"].cpu().numpy(), got["done"].cpu().numpy()
    resets = 0
    for j, r in enumerate(ring):
        np.testing.assert_array_equal(state[j], r["state"][0], err_msg=f"state slot {j}")
        np.testing.assert_array_equal(nxt[j], r["next_state"][0], err_msg=f"next_state slot {j}")
        np.testing.assert_array_equal(reward[j].reshape(-1), np.asarray(r["reward"], np.float32).reshape(-1))
        np.testing.assert_array_equal(done[j].reshape(-1) > 0.5, np.asarray(r["done"]).reshape(-1))
        resets += int((state[j] == state[j][:1]).all())
    assert resets > 0 and (done > 0.5).any()            # reset stacks and episode ends are among the compared slots
    if name in ("rainbow", "ape_x"):
        assert torch.equal(mem._tree, tmem._tree) and torch.equal(mem._max_priority, tmem._max_priority)


# --------------------------------------------------------------------------------------------- 3. learn() is unchanged
@pytest.mark.parametrize("name", ["rainbow", "ape_x"])
def test_learn_is_unchanged_by_the_layout(name):
    """The frame-store agent's materialised transitions, stored into a duplicated-layout twin with store(): the same
    injected PER uniforms give the same results, parameters, priorities and tree, bit for bit."""
    agent = _collect(name, frames=True)
    mem = agent.memory
    twin = _agent(name)
    twin.network.load_state_dict(agent.network.state_dict())
    twin.target_network.load_state_dict(agent.target_network.state_dict())
    for attr in ("beta", "epsilon", "num_transitions"):  # host bookkeeping the collection advanced
        if hasattr(agent, attr):
            setattr(twin, attr, getattr(agent, attr))
    rows = mem.gather_device(torch.arange(CAP, device=DEV))
    if name == "ape_x":
        rows["priority"] = mem._tree[mem.first_leaf_index:].clone()
    twin.memory.store([rows])
    assert twin.memory.frames is None and twin.memory.size == CAP
    # the tree's internal sums depend on the order of its updates, not on the layout: start both from the same tree
    twin.memory._tree.copy_(mem._tree)
    twin.memory._max_priority.copy_(mem._max_priority)
    rs = np.random.RandomState(7)
    for _ in range(4):
        u = (rs.rand(agent.batch_size), rs.rand(agent.batch_size))
        agent._inject_u = twin._inject_u = u
        ra, rb = agent.learn(), twin.learn()
        assert ra == rb
    torch.cuda.synchronize()
    assert torch.equal(agent.network.flat, twin.network.flat)
    assert torch.equal(mem._tree, twin.memory._tree) and torch.equal(mem._max_priority, twin.memory._max_priority)


# ------------------------------------------------------------------------------------------ 4. no silent stale frames
def test_evicted_reference_raises_on_the_host():
    from jorldy_b200.core import Env
    from jorldy_b200.core.buffer.frame_store import FrameEvictedError, FrameStore, frames_per_lane
    F = frames_per_lane(8, 2, 0, margin=0)
    assert F == 8
    env = Env("breakout", num_envs=2, seed=1, device=DEV)
    env.reset_device()
    fs = FrameStore(2, F, DEV)
    fs.start(env.obs)
    refs = []
    for _ in range(12):
        next_obs, _, done = env.step_device(None)
        refs.append(fs.push(env.obs, next_obs, done, env.auto_reset))
    s, x = refs[-1]
    fs.gather(s, x)                                       # resident: no error
    fs.check()
    s, x = refs[0]                                        # 12+ frames pushed since: overwritten in a ring of 8
    st, _ = fs.gather(s, x)
    with pytest.raises(FrameEvictedError):
        fs.check()
    assert int(st.max().item()) == 0                      # never the frames of another position


# ------------------------------------------------------------------------------- 5. stacked stores into an attached ring
def test_storing_stacks_into_a_frame_replay_raises():
    from jorldy_b200.core import Env
    from jorldy_b200.core.collect import ReplayCollector
    agent = _agent("multistep")
    ReplayCollector(Env("breakout", num_envs=4, seed=0, device=DEV), agent, update_period=1)
    assert agent.memory.frames is not None
    tr = {"state": np.zeros((1, 4, 84, 84), np.uint8), "action": np.zeros((1, 1), np.int64),
          "reward": np.zeros((1, 3), np.float64), "done": np.zeros((1, 3), bool), "next_state": np.zeros((1, 4, 84, 84), np.uint8)}
    with pytest.raises(ValueError, match="frame"):
        agent.memory.store([tr])
    assert agent.memory.size == 0
