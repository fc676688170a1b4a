"""Resident rollout collection: act -> env.step -> write transition, for every env at once, with
no host hop.  Replaces the per-actor loop of jorldy/manager/distributed_manager.py:76-92
(`Actor.run`) and its gather in run_mode.py:180-187: the N ray actors become N rows of one batched
launch sequence, and the whole T-step rollout is captured in ONE CUDA graph (per-row Philox
counters and the env's own episode counters advance on the device, so every replay draws fresh
randomness).
"""
import torch

from .buffer import DeviceRollout, EpisodeRing, FrameRollout, frame_store
from .dev import capture_after_warmup


class RolloutCollector:
    def __init__(self, env, agent, n_step=None, use_cuda_graph=True):
        self.env, self.agent = env, agent
        self.T = n_step or agent.n_step
        # Atari-shaped envs: every frame is pushed once and the rollout stores frame references (buffer/frame_store.py)
        self.frames = bool(getattr(env, "frame_stack", False))
        if self.frames:
            self.rollout = FrameRollout(env.num_envs, self.T, env.action_size, env.action_type, device=agent.device,
                                        next_state=getattr(agent, "needs_next_state", False))
        else:
            self.rollout = DeviceRollout(env.num_envs, self.T, env.state_size, env.action_size, env.action_type,
                                         device=agent.device, next_state=getattr(agent, "needs_next_state", False))
        self.use_cuda_graph = use_cuda_graph
        self._graph = None
        # kernels of OUR library per env step: mlp_in_fwd + gemm + heads_fwd + act + env_step (the
        # rollout-row copies are torch plumbing and not counted)
        self.launches_per_collect = 5 * self.T
        env.reset_device()
        if self.frames:
            self.rollout.start(env.obs)

    def _collect_eager(self):
        env, agent, ro = self.env, self.agent, self.rollout
        ro.clear()
        for t in range(self.T):
            if not self.frames:
                ro.state[:, t].copy_(env.obs)                  # state acted on (pre-step observation)
            action = agent.act_device(env.obs, training=True)
            next_obs, reward, done = env.step_device(action)   # env.obs <- post-reset observation
            ro.t = t
            if self.frames:
                next_obs = ro.push(env.obs, next_obs, done, env.auto_reset)
            ro.write_after_step(action, reward, done, next_obs)

    def collect(self):
        """Fills self.rollout with T steps of all envs; returns it."""
        if not self.use_cuda_graph:
            self._collect_eager()
            return self.rollout
        if self._graph is None:
            self._graph = capture_after_warmup(self._collect_eager)      # the T-step sequence
        self._graph.replay()
        self.rollout.t = self.T
        return self.rollout


class EpisodeCollector:
    """Whole-episode collection for REINFORCE: a round is n_round steps of act -> env.step_device -> ring write for
    every env, captured in ONE CUDA graph like RolloutCollector's (the ring's write column advances on the device);
    use_cuda_graph=False runs the same launches eagerly.  The ring holds L = env.max_steps - 1 + n_round steps per env
    (EpisodeRing), so an env needs a time limit."""

    def __init__(self, env, agent, n_round, use_cuda_graph=True):
        if getattr(env, "frame_stack", False):
            raise NotImplementedError("episode rings of frame stacks are not implemented: an episode can outlive any "
                                      "frame store that fits on the device")
        max_steps = getattr(env, "max_steps", None)
        if not max_steps:
            raise ValueError(f"{type(env).__name__} has no max_steps time limit: an unfinished episode could outgrow "
                             "any episode ring")
        self.env, self.agent, self.T = env, agent, int(n_round)
        self.ring = EpisodeRing(env.num_envs, EpisodeRing.capacity(max_steps, self.T), env.state_size, env.action_size,
                                env.action_type, device=agent.device)
        self.use_cuda_graph = use_cuda_graph
        self._graph = None
        env.reset_device()

    def _collect_eager(self):
        env, agent, ring = self.env, self.agent, self.ring
        for _ in range(self.T):
            ring.write_state(env.obs)
            action = agent.act_device(env.obs, training=True)
            next_obs, reward, done = env.step_device(action)
            ring.write_after_step(action, reward, done)

    def collect(self):
        """Appends n_round steps of every env to self.ring; returns it."""
        if not self.use_cuda_graph:
            self._collect_eager()
            return self.ring
        if self._graph is None:
            self._graph = capture_after_warmup(self._collect_eager)      # the warm-up's steps are this round's
            return self.ring
        self._graph.replay()
        return self.ring


class NStepAssembler:
    """Device-side n-step transition assembly for N batched envs.

    Same windows as the reference's per-actor deques — multistep.py:90-104 / rainbow.py:294-308 (window of
    n steps, next_state = last step's next_state) and ape_x.py:174-199 (window of n+1, next_state = the
    (n+1)-th step's state, actor-side priority |G_n - q_0|) — including their behaviour of NOT clearing at
    episode ends (windows straddle episodes and rely on the (1-done) mask).  One ring [N, L, ...] per field.

    trajectory=True emits the whole window instead (MPO's Retrace learner): state [N, n+1, ...] (s_0 .. s_{n-1} and the
    last step's next_state), and action, reward, done, log_mu [N, n, ...], oldest step first.  Inside a window s_{t+1}
    is the next state of step t wherever done_t = 0, so no per-step next_state is stored.
    """

    def __init__(self, n_step, apex=False, gamma=0.99, trajectory=False):
        self.n, self.apex, self.gamma, self.trajectory = n_step, apex, gamma, trajectory
        self.L = n_step + 1 if apex else n_step
        self.hist, self.count, self.pos = None, 0, 0

    def push(self, tr):
        """tr: dict of device tensors with leading dim N.  Returns an assembled batch dict or None."""
        if self.hist is None:
            self.hist = {k: torch.zeros((v.shape[0], self.L) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)
                         for k, v in tr.items()}
        for k, v in tr.items():
            self.hist[k][:, self.pos].copy_(v)
        newest = self.pos
        self.pos = (self.pos + 1) % self.L
        self.count = min(self.count + 1, self.L)
        if self.count < self.L:
            return None
        oldest = self.pos                  # after the increment, pos points at the oldest entry
        order = [(oldest + i) % self.L for i in range(self.L)]
        h = self.hist
        if self.trajectory:
            sel = torch.as_tensor(order, device=h["reward"].device)
            out = {k: h[k].index_select(1, sel) for k in ("action", "reward", "done", "log_mu")}
            out["state"] = torch.cat([h["state"].index_select(1, sel), h["next_state"][:, newest:newest + 1]], dim=1)
            return out
        out = {"state": h["state"][:, oldest].clone(), "action": h["action"][:, oldest].clone()}
        if self.apex:
            out["next_state"] = h["state"][:, newest].clone()
            steps = order[:-1]
        else:
            out["next_state"] = h["next_state"][:, newest].clone()
            steps = order
        sel = torch.as_tensor(steps, device=h["reward"].device)
        out["reward"] = h["reward"].index_select(1, sel).unsqueeze(-1)      # [N, n, 1]
        out["done"] = h["done"].index_select(1, sel).unsqueeze(-1)
        if self.apex:
            g = h["q"][:, newest].clone()
            for i in reversed(range(self.n)):
                s = steps[i]
                g = h["reward"][:, s] + (1 - h["done"][:, s]) * self.gamma * g
            out["priority"] = (g - h["q"][:, oldest]).abs().to(torch.float64).unsqueeze(-1)
        return out


class SequenceAssembler:
    """Device-side assembly of R2D2's replayed sequences for N batched lanes (Kapturowski et al., ICLR 2019).

    Each lane keeps a ring of L = n_burn_in + seq_len + n_step steps.  Once L steps have been pushed, the N windows of the
    last L steps are emitted every store_period = seq_len // 2 steps (windows overlap by L - store_period steps).  Like
    NStepAssembler's windows, they are not cut at episode ends: `reset` marks the steps that start an episode, and the
    learner's unroll zeroes the recurrent state there, exactly where the actor did.

    push(tr) takes the step's fields, each with leading dim N: state (or int64 frame references), action, prev_action
    (-1 at an episode's first step), reset (f32), reward, done, and, at the steps where starts_window() is true, the
    actor's (h0, c0) from before the step.  Only those snapshots are kept (at most ceil(L / store_period) + 1 of them),
    never an [N, L, H] history.  An emitted window holds every field as [N, L, ...] oldest step first, plus h0 / c0 [N, H]
    of its first step.
    """

    FIELDS = ("state", "action", "prev_action", "reset", "reward", "done")

    def __init__(self, n_burn_in, seq_len, n_step):
        self.L = int(n_burn_in) + int(seq_len) + int(n_step)
        self.period = max(1, int(seq_len) // 2)
        self.hist, self.t, self.pos, self.snap = None, 0, 0, {}

    def starts_window(self):
        """True if the next pushed step is the first step of a window (its pre-step (h, c) must come with it)."""
        return self.t % self.period == 0

    def push(self, tr):
        if self.hist is None:
            self.hist = {k: torch.zeros((tr[k].shape[0], self.L) + tuple(tr[k].shape[1:]), dtype=tr[k].dtype,
                                        device=tr[k].device) for k in self.FIELDS}
        if self.starts_window():
            self.snap[self.t] = (tr["h0"].clone(), tr["c0"].clone())
        for k in self.FIELDS:
            self.hist[k][:, self.pos].copy_(tr[k])
        self.pos = (self.pos + 1) % self.L
        self.t += 1
        start = self.t - self.L
        if start < 0 or start % self.period:
            return None
        sel = torch.as_tensor([(self.pos + i) % self.L for i in range(self.L)], device=self.hist["reward"].device)
        out = {k: v.index_select(1, sel) for k, v in self.hist.items()}
        out["h0"], out["c0"] = self.snap.pop(start)
        return out


class ReplayCollector:
    """Off-policy resident loop: `update_period` batched env steps feeding the HBM replay, then one
    agent.process() (the reference's sync loop, run_mode.py:180-187: one learn per round whatever the
    number of transitions that arrived — SURVEY.md row D3)."""

    def __init__(self, env, agent, update_period):
        self.env, self.agent, self.update_period = env, agent, update_period
        n = getattr(agent, "n_step", 1)
        apex = type(agent).__name__ == "ApeX"
        trajectory = getattr(agent, "trajectory_windows", False)      # MPO: whole windows with the behaviour log mu
        # recurrent agents (R2D2) bring their own sequence assembler and frame store
        self.sequences = getattr(agent, "sequence_assembler", None)
        self.assembler = NStepAssembler(n, apex, agent.gamma, trajectory) \
            if (n > 1 or apex or trajectory) and self.sequences is None else None
        if apex or self.sequences is not None:
            agent.set_actor_epsilons(env.num_envs, total=max(agent.num_workers, env.num_envs, 2))
        env.reset_device()
        # Atari-shaped envs: every frame is pushed once and the replay stores frame references (buffer/frame_store.py)
        if self.sequences is not None:
            self.frames = agent.attach_frames(env)
        else:
            self.frames = frame_store.attach(env, agent.memory, n)
        if self.frames is not None:
            self.frames.start(env.obs)

    def run_round(self, step):
        env, agent = self.env, self.agent
        batches = []
        for _ in range(self.update_period):
            state = env.obs if self.frames is not None else env.obs.clone()
            action, q_sel = agent.act_device(agent._net_input(state), True)
            next_obs, reward, done = env.step_device(action)
            if self.frames is not None:
                state, next_state = self.frames.push(env.obs, next_obs, done, env.auto_reset)
            else:
                next_state = next_obs.clone()
            if self.sequences is not None:
                tr = dict(agent.step_inputs, state=state, action=action.clone(), reward=reward.view(-1).clone(),
                          done=done.view(-1).clone())
                agent.end_step(tr["done"])
                out = self.sequences.push(tr)
                if out is not None:
                    batches.append(out)
                continue
            tr = {"state": state, "action": action.view(action.shape[0], -1).clone(), "reward": reward.clone(), "done": done.clone(),
                  "next_state": next_state}
            if self.assembler is not None:
                if self.assembler.apex:
                    tr["q"] = q_sel.clone()
                if self.assembler.trajectory:
                    tr["log_mu"] = q_sel.view(-1).clone()
                out = self.assembler.push({k: (v.view(v.shape[0]) if k in ("reward", "done") else v) for k, v in tr.items()})
                if out is not None:
                    batches.append(out)
            else:
                tr["reward"] = tr["reward"].view(-1, 1)
                tr["done"] = tr["done"].view(-1, 1)
                batches.append(tr)
        step += self.update_period
        result = agent.process(batches, step) if batches else {}
        return step, result
