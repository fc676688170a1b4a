"""Single-frame replay for Atari-shaped observations (csrc/frame_ring.cu).

A replay slot of the duplicated layout holds `state` and `next_state` as two uint8 [4,84,84] stacks: 56,448 B, with every
84x84 frame stored 8 times.  With a frame store attached, each batched env row (a lane) pushes every frame once into its
own ring of `F` frames, and the replay's `state` / `next_state` fields hold int64 frame references (8 B each).
`ReplayBuffer.gather_device` turns them back into the same [B,4,84,84] stacks, bit for bit, so sampling, learn() and the
PER tree do not change.

PPO's frame rollout (`FrameRollout`) keeps its states on a frame store too: `frames_per_rollout(T)` sizes the ring, and
`FrameRows` hands the CNN head a view of the referenced stacks whose conv1 im2col reads the ring directly.  MuZero's
windows reference their first stack: `frames_per_window` sizes the ring, and `FrameActionRows` adds the action planes.

This module owns the format: the sizing of the rings, the reference encoding ((lane << 40) | absolute frame position),
the push of one env step, the gather and conv1's im2col.  A reference whose frames have been overwritten is never
returned silently: the gather and im2col kernels set a status word and `check()` raises `FrameEvictedError`.
"""
import torch

from ..dev import C, ptr, stream_ptr

FRAME_BYTES = 84 * 84
STACK = 4
POS_BITS = 40
FRAME_KEYS = ("state", "next_state")


class FrameEvictedError(RuntimeError):
    """A replay slot referenced a frame that its lane's ring had already overwritten."""


def frames_per_lane(capacity, num_lanes, n_step, margin=None):
    """Ring length F per lane for a replay of `capacity` slots filled by `num_lanes` lanes.

    The ring holds ceil(C/N) transitions per lane, the n-step window emits a transition up to n_step env steps after its
    state, and the oldest stack reaches 3 frames further back (+ 4).  Episode resets push one extra frame each; the
    default margin of ceil(ceil(C/N)/16) frames covers a reset every 16 steps of every lane."""
    per_lane = -(-int(capacity) // int(num_lanes))
    if margin is None:
        margin = -(-per_lane // 16)
    return per_lane + int(n_step) + 4 + int(margin)


def frames_per_rollout(T):
    """Ring length F per lane for an on-policy rollout of T steps: max(2T + 4, 8).

    A rollout's first state is the newest frame pushed before it, at position h0 - 1 (h0: the lane's head when the
    rollout starts), and its stack reaches back to h0 - 4.  Each of the T steps pushes at most 2 frames (the newest
    frame, and the reset frame after an auto-reset), so when learn_rollout() reads the rollout the head is at most
    h0 + 2T, and every frame the rollout references lies in [h0 - 4, h0 + 2T): 2T + 4 frames, whatever the dones.  The
    next rollout's pushes start only after that read.  FrameStore (and jb_frame_push) need at least 8 frames."""
    return max(2 * int(T) + 4, 8)


def frames_per_window(capacity, num_lanes, window):
    """Ring length F per lane for a replay of `capacity` windows of `window` steps, each window referencing its first
    step's stack, one window per lane and step (MuZero): 2 (ceil(C/N) + window) + 2.

    A lane's live windows are its newest W = ceil(C/N).  The oldest starts at step t0 = T - window - (W - 1) (T: steps
    pushed so far); its stack is the frame at position h(t0) - 1 and reaches back to h(t0) - 4.  Each of the T - t0 =
    window + W - 1 steps since pushed at most 2 frames, so the head is at most h(t0) + 2 (window + W - 1) and every
    referenced frame lies in the last 2 (window + W) + 2 positions, whatever the dones."""
    return max(2 * (-(-int(capacity) // int(num_lanes)) + int(window)) + 2, 8)


def store_bytes(capacity, num_lanes, n_step, margin=None):
    """HBM taken by the frame rings (the replay adds 16 B of references per slot)."""
    return int(num_lanes) * frames_per_lane(capacity, num_lanes, n_step, margin) * FRAME_BYTES


def check_refs(transitions):
    """Raises ValueError unless every transition carries frame references (int64 [N]) under `state` / `next_state`."""
    for t in transitions:
        for k in FRAME_KEYS:
            v = t.get(k)
            if not (torch.is_tensor(v) and v.dtype == torch.int64 and v.dim() == 1):
                shape = tuple(v.shape) if hasattr(v, "shape") else type(v).__name__
                raise ValueError(
                    f"this replay keeps '{k}' as single-frame references (a frame store was attached when the Atari "
                    f"collector started), so it cannot store stacked observations (got {shape}); store them into a "
                    f"replay that no collector has attached a frame store to")


class FrameStore:
    def __init__(self, num_lanes, frames_per_lane, device):
        self.n, self.F = int(num_lanes), int(frames_per_lane)
        if self.F < 8:
            raise ValueError(f"frames_per_lane must be at least 8, got {self.F}")
        if self.n >= 1 << (63 - POS_BITS):
            raise ValueError(f"{self.n} lanes do not fit the frame reference encoding")
        self.device = device
        # only positions a push has written are ever read (the gather checks residency), so the frames start unset
        self.frames = torch.empty((self.n, self.F, FRAME_BYTES), dtype=torch.uint8, device=device)
        self.first = torch.zeros((self.n, self.F), dtype=torch.int64, device=device)
        self.head = torch.zeros(self.n, dtype=torch.int64, device=device)
        # written by the gather kernel only on an evicted reference; pinned host memory, so reading it after the
        # stream synchronisation that learn() already does costs no copy
        self.status = torch.zeros(1, dtype=torch.int32, pin_memory=True)
        self.started = False

    @classmethod
    def for_replay(cls, capacity, num_lanes, n_step, device, margin=None):
        return cls(num_lanes, frames_per_lane(capacity, num_lanes, n_step, margin), device)

    def start(self, obs):
        """Pushes obs[:,3] of every lane as an episode-first frame (obs: the [N,4,84,84] stacks after a reset)."""
        self._check_obs(obs)
        C.jb_frame_push(ptr(self.frames), ptr(self.first), ptr(self.head), self.F, ptr(obs), 0, 0, 0, 0, 0, self.n,
                        stream_ptr())
        self.started = True

    def push(self, obs, next_obs, done, auto_reset, out=None):
        """One env step: next_obs[:,3] continues each lane's episode; where done and the env auto-reset, obs[:,3] starts
        the next one.  Returns (state_ref, next_ref), int64 [N]: the stack acted on and the stack after the step, as
        the rows of `out` (int64 [2, N], contiguous) when given."""
        if not self.started:
            raise RuntimeError("FrameStore.start() must push the reset observation first")
        self._check_obs(obs)
        self._check_obs(next_obs)
        if out is not None and (out.dtype != torch.int64 or tuple(out.shape) != (2, self.n) or not out.is_contiguous()):
            raise ValueError(f"expected a contiguous int64 [2,{self.n}] reference buffer, got {out.dtype} {tuple(out.shape)}")
        refs = out if out is not None else torch.empty((2, self.n), dtype=torch.int64, device=self.device)
        C.jb_frame_push(ptr(self.frames), ptr(self.first), ptr(self.head), self.F, ptr(obs), ptr(next_obs),
                        ptr(done.contiguous()), int(bool(auto_reset)), ptr(refs[0]), ptr(refs[1]), self.n, stream_ptr())
        return refs[0], refs[1]

    def gather(self, state_refs, next_refs, idx=None):
        """Stacks [B,4,84,84] of state_refs[idx] and next_refs[idx] (idx None: all of them).  An evicted reference
        comes back zero-filled and makes the next check() raise."""
        B = int(idx.shape[0]) if idx is not None else int(state_refs.shape[0])
        state = torch.empty((B, STACK, 84, 84), dtype=torch.uint8, device=self.device)
        nxt = torch.empty_like(state)
        if B == 0:
            return state, nxt
        C.jb_frame_gather(ptr(self.frames), ptr(self.first), ptr(self.head), self.F, self.n, ptr(state_refs.contiguous()),
                          ptr(next_refs.contiguous()), ptr(idx), B, ptr(state), ptr(nxt), ptr(self.status), stream_ptr())
        return state, nxt

    def check(self):
        """Raises FrameEvictedError if a gather so far met a reference to an overwritten frame."""
        torch.cuda.current_stream(self.device).synchronize()
        if int(self.status[0]) != 0:
            raise FrameEvictedError(
                f"the replay sampled a frame that its lane's ring of {self.F} frames had already overwritten; the batch "
                f"gathered with it is invalid (more episode resets than the ring's margin covers)")

    def _check_obs(self, obs):
        if obs.dtype != torch.uint8 or tuple(obs.shape) != (self.n, STACK, 84, 84) or not obs.is_contiguous():
            raise ValueError(f"expected contiguous uint8 [{self.n},4,84,84] stacks, got {obs.dtype} {tuple(obs.shape)}")


class FrameRows:
    """The [M,4,84,84] stacks named by `refs` (int64 [M]) on `store`, as the CNN head's input: it has shape[0], row
    slices (inference chunks) and `im2col`, which writes conv1's column matrix straight from the ring.  data_ptr() is
    the refs tensor's, so a CUDA graph keyed on the input's pointer is replayed only over the same reference rows."""

    def __init__(self, store, refs):
        self.store, self.refs = store, refs

    @property
    def shape(self):
        return (int(self.refs.shape[0]), STACK, 84, 84)

    def __getitem__(self, rows):
        if not isinstance(rows, slice):
            raise TypeError("FrameRows supports row slices only")
        return FrameRows(self.store, self.refs[rows])

    def data_ptr(self):
        return self.refs.data_ptr()

    def im2col(self, idx, M, col):
        """col [M*400, 256] f32 <- conv1's im2col of the stacks refs[idx[i]] (idx int32 [M], None: rows 0..M-1), bit-equal
        to gather() + jb_im2col_u8.  An evicted reference gives zero rows and makes the next check() raise."""
        if idx is not None and (idx.dtype != torch.int32 or not idx.is_contiguous()):
            raise ValueError(f"expected contiguous int32 row indices, got {idx.dtype}")
        s = self.store
        C.jb_im2col_u8_frames(ptr(s.frames), ptr(s.first), ptr(s.head), s.F, s.n, ptr(self.refs), ptr(idx), M, ptr(col),
                              ptr(s.status), stream_ptr())
        return col


class FrameActionRows(FrameRows):
    """FrameRows plus MuZero's action planes: the [M,8,84,84] inputs named by `refs` and `actions` (int64 [M,4], the
    actions that produced each stack's four frames, oldest first; csrc/frame_ring.cu zeroes the planes of frames at or
    before an episode's first frame).  im2col writes conv1's 512-column matrix, planes as channels 4..7."""

    def __init__(self, store, refs, actions, num_actions):
        super().__init__(store, refs)
        self.actions, self.num_actions = actions, int(num_actions)

    @property
    def shape(self):
        return (int(self.refs.shape[0]), 2 * STACK, 84, 84)

    def __getitem__(self, rows):
        if not isinstance(rows, slice):
            raise TypeError("FrameActionRows supports row slices only")
        return FrameActionRows(self.store, self.refs[rows], self.actions[rows], self.num_actions)

    def im2col(self, idx, M, col):
        if idx is not None and (idx.dtype != torch.int32 or not idx.is_contiguous()):
            raise ValueError(f"expected contiguous int32 row indices, got {idx.dtype}")
        a = self.actions
        if a.dtype != torch.int64 or tuple(a.shape) != (int(self.refs.shape[0]), STACK) or not a.is_contiguous():
            raise ValueError(f"expected contiguous int64 [{int(self.refs.shape[0])},{STACK}] actions, got {a.dtype} "
                             f"{tuple(a.shape)}")
        s = self.store
        C.jb_im2col_u8_frames_actions(ptr(s.frames), ptr(s.first), ptr(s.head), s.F, s.n, ptr(self.refs), ptr(a),
                                      self.num_actions, ptr(idx), M, ptr(col), ptr(s.status), stream_ptr())
        return col


def attach(env, memory, n_step):
    """Gives `memory` a frame store sized for `env`'s lanes when the env produces frame stacks (`env.frame_stack`) and
    the memory is an empty replay ring; returns the store, or None (the memory keeps whole stacks)."""
    from .replay_buffer import ReplayBuffer
    if not getattr(env, "frame_stack", False) or not isinstance(memory, ReplayBuffer):
        return None
    if memory.fields is not None or memory.size > 0 or memory.frames is not None:
        return None
    store = FrameStore.for_replay(memory.buffer_size, env.num_envs, n_step, memory.device)
    memory.frames = store
    return store
