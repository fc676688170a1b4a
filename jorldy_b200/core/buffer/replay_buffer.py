"""HBM-resident replay ring (jorldy/core/buffer/replay_buffer.py:8-35).

The reference keeps a numpy array of python dicts and stacks B of them per sample; here every
transition field is one device tensor [capacity, ...] (structure of arrays, allocated on the
first store from the transition's own shapes), `store` is one host->device copy per field +
a row scatter into the ring and `sample` a row gather (csrc/replay.cu: jb_replay_store / jb_replay_gather).  Integer bookkeeping
(`buffer_index`, `buffer_counter`, `size`) matches the reference exactly and lives on the host.

dtypes in HBM: uint8 observations stay uint8 (the learner casts, base.py:61-73); float64 fields
are stored as float32 (the learner casts them to float32 anyway — same rounding, done once);
bool -> uint8; int64 kept.  `sample()` returns numpy arrays with the dtypes the reference's
`stack_transition` would have produced.

Atari-shaped collectors attach a single-frame store (frame_store.py): `state` / `next_state` then hold int64 frame
references, `gather_device` rebuilds the same uint8 stacks from them, and stacked stores are refused.
"""
import numpy as np
import torch

from ..dev import C, ptr, require_cuda, stream_ptr
from . import frame_store
from .base import BaseBuffer

_STORE_DTYPE = {np.dtype("float64"): torch.float32, np.dtype("float32"): torch.float32,
                np.dtype("uint8"): torch.uint8, np.dtype("bool"): torch.uint8,
                np.dtype("int64"): torch.int64, np.dtype("int32"): torch.int32}


def _np(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


class ReplayBuffer(BaseBuffer):
    def __init__(self, buffer_size, device=None):
        super().__init__()
        self.device = require_cuda(device)
        self.buffer_size = int(buffer_size)
        self.buffer_index = 0
        self.buffer_counter = 0
        self.fields = None          # key -> tensor | list[tensor]
        self._np_dtype = {}         # key / (key, i) -> numpy dtype the reference would return
        self.frames = None          # FrameStore (frame_store.py): `state` / `next_state` then hold frame references

    # ---- storage ------------------------------------------------------------------------------
    def _alloc_one(self, tag, sample):
        a = _np(sample) if not torch.is_tensor(sample) else sample
        if torch.is_tensor(a):
            dt, npdt = a.dtype, None
        else:
            npdt = a.dtype
            dt = _STORE_DTYPE.get(a.dtype)
            if dt is None:
                raise TypeError(f"unsupported transition dtype {a.dtype} for '{tag}'")
        self._np_dtype[tag] = npdt
        return torch.zeros((self.buffer_size,) + tuple(a.shape[1:]), dtype=dt, device=self.device)

    def _allocate(self, transition):
        self.fields = {}
        for key, val in transition.items():
            if isinstance(val, (list, tuple)):
                self.fields[key] = [self._alloc_one((key, i), v) for i, v in enumerate(val)]
            else:
                self.fields[key] = self._alloc_one(key, val)

    def _positions(self, n):
        pos = (self.buffer_index + np.arange(n)) % self.buffer_size
        return torch.as_tensor(pos, dtype=torch.int64, device=self.device)

    @staticmethod
    def _cat(vals, dtype, device):
        if torch.is_tensor(vals[0]):
            t = torch.cat([v.to(device) for v in vals], dim=0) if len(vals) > 1 else vals[0].to(device)
            return t.to(dtype)
        a = np.concatenate([np.asarray(v) for v in vals], axis=0) if len(vals) > 1 else np.asarray(vals[0])
        return torch.as_tensor(a, device=device).to(dtype)

    def _write(self, transitions):
        """Writes the stacked transitions into the ring; returns the number of rows written."""
        if self.frames is not None:
            frame_store.check_refs(transitions)
        if self.fields is None:
            self._allocate(transitions[0])
        n = sum(int(np.shape(t["reward"])[0]) if "reward" in t else 1 for t in transitions)
        pos = self._positions(n)
        if n > self.buffer_size:     # only the last `buffer_size` rows survive a wrap
            keep = slice(n - self.buffer_size, n)
        else:
            keep = slice(0, n)
        for key, dst in self.fields.items():
            if isinstance(dst, list):
                for i, d in enumerate(dst):
                    self._scatter(d, self._cat([t[key][i] for t in transitions], d.dtype, self.device)[keep], pos[keep])
            else:
                self._scatter(dst, self._cat([t[key] for t in transitions], dst.dtype, self.device)[keep], pos[keep])
        return n

    _MAX_ROWS = 32768          # rows per launch (grid.y)

    @staticmethod
    def _row_bytes(t):
        return t[0].numel() * t.element_size() if t.dim() > 1 else t.element_size()

    def _scatter(self, ring, rows, pos):
        rows = rows.contiguous().view(rows.shape[0], -1) if rows.dim() > 1 else rows.contiguous()
        assert rows.dtype == ring.dtype and self._row_bytes(rows) == self._row_bytes(ring), "transition field changed shape"
        rb, n = self._row_bytes(ring), rows.shape[0]
        for off in range(0, n, self._MAX_ROWS):
            m = min(self._MAX_ROWS, n - off)
            C.jb_replay_store(ptr(ring), ptr(rows[off:off + m]), ptr(pos[off:off + m]), m, rb, stream_ptr())

    def _gather(self, ring, idx):
        out = torch.empty((idx.shape[0],) + tuple(ring.shape[1:]), dtype=ring.dtype, device=ring.device)
        rb, n = self._row_bytes(ring), idx.shape[0]
        for off in range(0, n, self._MAX_ROWS):
            m = min(self._MAX_ROWS, n - off)
            C.jb_replay_gather(ptr(ring), ptr(idx[off:off + m]), m, rb, ptr(out[off:off + m]), stream_ptr())
        return out

    def store(self, transitions):
        if self.first_store:
            self.check_dim({k: ([_np(x) for x in v] if isinstance(v, (list, tuple)) else _np(v))
                            for k, v in transitions[0].items()})
        n = self._write(transitions)
        self.buffer_index = (self.buffer_index + n) % self.buffer_size
        self.buffer_counter = min(self.buffer_counter + n, self.buffer_size)

    # ---- sampling -----------------------------------------------------------------------------
    def gather_device(self, idx):
        """idx: int64 device tensor of ring positions -> dict of device tensors (stored dtypes)."""
        out = {}
        idx = idx.to(torch.int64).contiguous()
        stacks = {}
        if self.frames is not None:
            stacks = dict(zip(frame_store.FRAME_KEYS, self.frames.gather(self.fields["state"], self.fields["next_state"], idx)))
        for key, src in self.fields.items():
            if key in stacks:
                out[key] = stacks[key]
            else:
                out[key] = [self._gather(s, idx) for s in src] if isinstance(src, list) else self._gather(src, idx)
        return out

    def check_frames(self):
        """Raises if a gather so far handed out an evicted frame (no-op without a frame store).  Synchronises the stream."""
        if self.frames is not None:
            self.frames.check()

    def _to_numpy(self, dev_dict):
        out = {}
        for key, val in dev_dict.items():
            if isinstance(val, list):
                out[key] = [self._cast_np(v.cpu().numpy(), self._np_dtype[(key, i)]) for i, v in enumerate(val)]
            else:
                out[key] = self._cast_np(val.cpu().numpy(), self._np_dtype[key])
        self.check_frames()
        return out

    @staticmethod
    def _cast_np(a, npdt):
        return a if npdt is None or a.dtype == npdt else a.astype(npdt)

    def sample_indices(self, batch_size):
        """Uniform with replacement over the filled part (np.random.randint, replay_buffer.py:26)."""
        return np.random.randint(self.buffer_counter, size=batch_size)

    def sample(self, batch_size):
        idx = torch.as_tensor(self.sample_indices(batch_size), dtype=torch.int64, device=self.device)
        return self._to_numpy(self.gather_device(idx))

    def sample_device(self, batch_size, idx=None):
        if idx is None:
            idx = torch.randint(self.buffer_counter, (batch_size,), device=self.device)
        return self.gather_device(idx)

    @property
    def size(self):
        return self.buffer_counter
