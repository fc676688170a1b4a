"""On-policy rollout storage.

`RolloutBuffer` keeps the reference's list semantics for host transitions
(jorldy/core/buffer/rollout_buffer.py:6-24: store appends, sample stacks everything and clears).
`DeviceRollout` is the HBM-resident [N, T, ...] structure-of-arrays the batched collect kernels
write straight into (no host hop): actor-major like the reference's concatenation order
(distributed_manager.py:30), so GAE's `view(-1, n_step)` rows are envs.  `FrameRollout` is its variant for
Atari-shaped frame stacks, with states kept as single-frame references (buffer/frame_store.py).
"""
import numpy as np
import torch

from ..dev import require_cuda
from .base import BaseBuffer
from .frame_store import FrameRows, FrameStore, frames_per_rollout


class RolloutBuffer(BaseBuffer):
    def __init__(self):
        super().__init__()
        self.buffer = list()

    def store(self, transitions):
        if self.first_store:
            self.check_dim(transitions[0])
        self.buffer += transitions

    def sample(self):
        transitions = self.stack_transition(self.buffer)
        self.buffer.clear()
        return transitions

    def sample_batched(self):
        """For transitions whose leading dim is a batch of N envs (one dict per time step): returns
        arrays laid out [N*T, ...] actor-major, i.e. what N reference actors would have produced."""
        out = {}
        for key in self.buffer[0].keys():
            arr = np.stack([np.asarray(b[key]) for b in self.buffer], axis=1)   # [N, T, ...]
            out[key] = arr.reshape((-1,) + arr.shape[2:])
        self.buffer.clear()
        return out

    @property
    def size(self):
        return len(self.buffer)


class DeviceRollout:
    """next_state=True keeps every step's next state in next_state [N, T, D] (the env's terminal observation at done
    steps, not the post-reset one), for learners that read s' per row (ICM-PPO); otherwise only last_next_state."""

    def __init__(self, num_envs, n_step, state_size, action_size, action_type, device=None, next_state=False):
        dev = require_cuda(device)
        N, T = num_envs, n_step
        self.N, self.T, self.device = N, T, dev
        self.state = torch.zeros(N, T, state_size, dtype=torch.float32, device=dev)
        if action_type == "discrete":
            self.action = torch.zeros(N, T, dtype=torch.int32, device=dev)
        else:
            self.action = torch.zeros(N, T, action_size, dtype=torch.float32, device=dev)
        self.reward = torch.zeros(N, T, dtype=torch.float32, device=dev)
        self.done = torch.zeros(N, T, dtype=torch.float32, device=dev)
        self.last_next_state = torch.zeros(N, state_size, dtype=torch.float32, device=dev)
        self.next_state = torch.zeros(N, T, state_size, dtype=torch.float32, device=dev) if next_state else None
        self.t = 0

    def next_rows(self):
        """The N*T next states, actor-major, or None when the rollout does not keep them."""
        return None if self.next_state is None else self.next_state.view(self.N * self.T, -1)

    def write(self, state, action, reward, done, next_state):
        t = self.t
        self.state[:, t].copy_(state)
        if self.action.dtype == torch.int32:
            self.action[:, t].copy_(action.view(self.N))
        else:
            self.action[:, t].copy_(action.view(self.N, -1))
        self.reward[:, t].copy_(reward)
        self.done[:, t].copy_(done)
        if self.next_state is not None:
            self.next_state[:, t].copy_(next_state)
        if t == self.T - 1:
            self.last_next_state.copy_(next_state)
        self.t = t + 1

    def write_after_step(self, action, reward, done, next_state):
        """Second half of a transition (the pre-step state was already copied into state[:, t])."""
        t = self.t
        if self.action.dtype == torch.int32:
            self.action[:, t].copy_(action.view(self.N))
        else:
            self.action[:, t].copy_(action.view(self.N, -1))
        self.reward[:, t].copy_(reward)
        self.done[:, t].copy_(done)
        if self.next_state is not None:
            self.next_state[:, t].copy_(next_state)
        if t == self.T - 1:
            self.last_next_state.copy_(next_state)
        self.t = t + 1

    @property
    def full(self):
        return self.t >= self.T

    def clear(self):
        self.t = 0


class FrameRollout(DeviceRollout):
    """DeviceRollout of a frame-stack env (`env.frame_stack`, uint8 [N,4,84,84] observations): every frame is pushed once
    into a per-env ring of frames_per_rollout(T) frames, and the rollout keeps int64 frame references instead of states:
    state_ref [N, T] and last_next_state [N] (the last step's next state).  That is 7-14 KB per env step on the ring
    against 28 KB as a uint8 stack and 113 KB as fp32.  action / reward / done are DeviceRollout's.  The learner reads
    the states through `rows()` / `last_rows()` (buffer/frame_store.py FrameRows).  next_state=True also keeps every step's
    next-state reference in next_ref [N, T] (the terminal stack at done steps), read through `next_rows()`; these stacks
    lie in the same window of the ring as the states, so frames_per_rollout(T) keeps them resident too."""

    def __init__(self, num_envs, n_step, action_size, action_type, device=None, next_state=False):
        dev = require_cuda(device)
        N, T = num_envs, n_step
        self.N, self.T, self.device = N, T, dev
        self.frames = FrameStore(N, frames_per_rollout(T), dev)
        self.state_ref = torch.zeros(N, T, dtype=torch.int64, device=dev)
        if action_type == "discrete":
            self.action = torch.zeros(N, T, dtype=torch.int32, device=dev)
        else:
            self.action = torch.zeros(N, T, action_size, dtype=torch.float32, device=dev)
        self.reward = torch.zeros(N, T, dtype=torch.float32, device=dev)
        self.done = torch.zeros(N, T, dtype=torch.float32, device=dev)
        self.last_next_state = torch.zeros(N, dtype=torch.int64, device=dev)
        self.next_state = None
        self.next_ref = torch.zeros(N, T, dtype=torch.int64, device=dev) if next_state else None
        self._refs = torch.zeros(2, N, dtype=torch.int64, device=dev)
        self.t = 0

    def start(self, obs):
        """Pushes the observation after the env's reset (FrameStore.start)."""
        self.frames.start(obs)

    def push(self, obs, next_obs, done, auto_reset):
        """Pushes step t's frames (FrameStore.push), writes the reference of the stack acted on into column t and
        returns the next state's reference, for write_after_step()."""
        s, x = self.frames.push(obs, next_obs, done, auto_reset, out=self._refs)
        self.state_ref[:, self.t].copy_(s)
        if self.next_ref is not None:
            self.next_ref[:, self.t].copy_(x)
        return x

    def rows(self):
        """The N*T states, actor-major."""
        return FrameRows(self.frames, self.state_ref.view(-1))

    def last_rows(self):
        return FrameRows(self.frames, self.last_next_state)

    def next_rows(self):
        return None if self.next_ref is None else FrameRows(self.frames, self.next_ref.view(-1))
