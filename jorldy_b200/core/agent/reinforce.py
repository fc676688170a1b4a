"""REINFORCE agent (Williams, 1992) on whole episodes.

Mirror of jorldy/core/agent/reinforce.py (constructor :32-64, save / load :128-142): one policy network
(`discrete_policy` logits or `continuous_policy` raw [mu | log_std]), one optimiser, no critic.

  act      discrete a ~ Categorical(softmax(logits)) (argmax when not training) with jb_sacd_act; continuous
           a = tanh(z), z ~ Normal(clamp(mu, +-5), exp(tanh(log_std))) (tanh(mu) when not training) with
           jb_ppo_act_continuous
  process  stores the transitions; at an episode end learn() and, with lr_decay, learning_rate_decay(step)
  learn    the stored buffer as ONE episode (the reference's return loop has no reset at done flags)

learn() and the batched path share one learn over an EpisodeRing (buffer/rollout_buffer.py), `learn_episodes(ring)`:
  1. jb_episode_returns + jb_episode_rows: per completed episode the reference's discounted returns and standardisation,
     and the compact env-major, oldest-first row list (idx, ret) padded to a multiple of the chunk size C
  2. one device->host read of M, the number of rows (it decides the chunk count); M = 0 returns {} and touches nothing
  3. ceil(M / C) chunk steps: jb_take_minibatch -> forward_raw over the chunk's ring rows -> jb_reinforce_loss ->
     backward_raw -> jb_add_f32 into the summed gradient, captured once as a CUDA graph that takes its rows through the
     device cursor (use_cuda_graph=False: the same launches eagerly, bit-identical)
  4. one optimizer.step() on the summed gradient, with no clipping (the reference clips nothing)
  5. one device->host read of the result {"loss"}

The batched mapping: one env row plays one reference actor; a learn takes every episode that completed since the last
one, each with its own return statistics, and the loss is the mean over all their rows (DESIGN.md §5h).
"""
import numpy as np
import torch

from ..buffer import EpisodeRing, RolloutBuffer
from ..dev import C, capture_after_warmup, ptr, require_cuda, stream_ptr
from ..network import Network
from ..optimizer import Optimizer
from .base import BaseAgent
from .ppo import MAX_ACTION_SIZE

CHUNK_ROWS = 8192        # rows per chunk step: ~16 MB per activation at hidden_size 512; not tuned


class REINFORCE(BaseAgent):
    replicas_only = True          # parallel.attach: no data-parallel learner for REINFORCE
    FAMILY = "REINFORCE"
    LAUNCHES_PER_CHUNK = 12       # take + in_fwd + gemm + heads + loss + fold + 2 heads bwd + 3 gemm + add

    def __init__(self, state_size, action_size, hidden_size=512, network="discrete_policy", head="mlp",
                 optim_config={"name": "adam"}, gamma=0.99, use_standardization=False, run_step=1e6, lr_decay=True,
                 device=None, seed=0, use_cuda_graph=True, **kwargs):
        if head == "cnn":
            raise NotImplementedError("REINFORCE is built for the mlp head: an episode of Atari frames can outlive any "
                                      "episode ring a frame store could keep on the device")
        if network not in ("discrete_policy", "continuous_policy"):
            raise ValueError(f"REINFORCE network '{network}': use discrete_policy or continuous_policy")
        self.action_type = network.split("_")[0]
        max_a = MAX_ACTION_SIZE[self.action_type]
        if not 1 <= action_size <= max_a:
            raise ValueError(f"REINFORCE's {self.action_type} kernels take 1 to {max_a} actions, got {action_size}")
        if not isinstance(state_size, int):
            raise ValueError("REINFORCE takes an integer state_size (mlp head)")
        self.device = require_cuda(device)
        self.state_size, self.action_size = state_size, action_size
        self.network = Network(network, state_size, action_size, D_hidden=hidden_size, head=head, device=self.device)
        self.optimizer = Optimizer(**dict(optim_config), params=self.network.parameters())
        self.gamma = gamma
        self.use_standardization = use_standardization
        self.memory = RolloutBuffer()
        self.run_step = run_step
        self.lr_decay = lr_decay

        self.seed = int(seed)
        self.rng_stream_base = 0
        self._row_ctr = {}
        self.use_cuda_graph = use_cuda_graph
        self._graphs = {}
        self._work = {}
        self._single = None                 # learn()'s one-env ring
        dev = self.device
        self._acc = torch.zeros(2, dtype=torch.float32, device=dev)          # loss, chunks
        self._cursor = torch.zeros(1, dtype=torch.int64, device=dev)
        self._gsum = torch.zeros_like(self.network.grad)                     # chunk gradients summed in chunk order
        self.n_launches = 0                 # kernels launched by the last learn (throughput bookkeeping)
        self.last_M = 0                     # rows of the last learn

    @property
    def continuous(self):
        return self.action_type == "continuous"

    # ------------------------------------------------------------------------------------- act --
    def act_device(self, state, training=True, noise=None):
        """state [N, D] f32 device tensor -> action ([N] int64 / [N, A] f32).  noise: optional uniforms [N] / normals
        [N, A]."""
        net = self.network
        M, A = state.shape[0], self.action_size
        out = net._buf("act.out", (M, net.nout))
        net.forward_rows(state, out)
        row_ctr = self._row_counter(M)
        greedy = 0 if training else 1
        if self.continuous:
            action = net._buf("act.a", (M, A))
            C.jb_ppo_act_continuous(ptr(out), M, A, net.nout, ptr(noise), self.seed, self.rng_stream_base, 0,
                                    ptr(row_ctr), greedy, ptr(action), stream_ptr())
        else:
            action = net._buf("act.a", (M,), torch.int64)
            C.jb_sacd_act(ptr(out), M, A, ptr(noise), self.seed, self.rng_stream_base, ptr(row_ctr), greedy,
                          ptr(action), stream_ptr())
        return action

    @torch.no_grad()
    def act(self, state, training=True):
        self.network.train(training)
        s = self.as_tensor(state)
        a = self.act_device(s.view(s.shape[0], -1), training).cpu().numpy()
        return {"action": a.reshape(a.shape[0], -1)}

    # ----------------------------------------------------------------------------------- learn --
    def _chunk_rows(self, ring):
        return min(CHUNK_ROWS, -(-ring.N * ring.L // 256) * 256)

    def _workspace(self, ring):
        """Per-ring learn buffers: returns [N, L], counts, offsets, the padded row list and M."""
        key = (ring.state.data_ptr(), ring.N, ring.L)
        w = self._work.get(key)
        if w is None:
            N, L, dev = ring.N, ring.L, self.device
            Cr = self._chunk_rows(ring)
            n_rows = -(-N * L // Cr) * Cr
            w = {"C": Cr, "ret_ring": torch.zeros(N, L, device=dev), "count": torch.zeros(N, dtype=torch.int32, device=dev),
                 "offsets": torch.zeros(N, dtype=torch.int32, device=dev),
                 "idx": torch.zeros(n_rows, dtype=torch.int32, device=dev), "ret": torch.zeros(n_rows, device=dev),
                 "M": torch.zeros(1, dtype=torch.int32, device=dev)}
            self._work = {key: w}           # one ring at a time: a new ring retires the old workspace and graphs
            self._graphs = {}
        return w

    def _chunk_step(self, ring, w):
        """One chunk: the rows idx[k C:(k+1) C] with k the device cursor, then cursor += 1."""
        net, Cr, s = self.network, w["C"], stream_ptr()
        cur_idx = net._buf("ch.idx", (Cr,), torch.int32)
        C.jb_take_minibatch(ptr(w["idx"]), ptr(self._cursor), Cr, ptr(cur_idx), s)
        out = net.forward_raw(ring.state.view(ring.N * ring.L, -1), cur_idx, Cr, tag="ch.")
        dout = net._buf("ch.dout", (Cr, net.nout))
        partials = net._buf("ch.partials", (C.jb_reinforce_loss_partials(Cr),))
        C.jb_reinforce_loss(int(self.continuous), ptr(out), ptr(w["idx"]), ptr(w["ret"]), ptr(self._cursor), ptr(w["M"]),
                            Cr, ptr(ring.action), self.action_size, net.nout, ptr(dout), ptr(partials), ptr(self._acc), s)
        net.backward_raw(dout, Cr, tag="ch.")
        C.jb_add_f32(ptr(self._gsum), ptr(net.grad), net.num_flat, s)

    def _graph_for(self, ring, w):
        key = (w["C"], ring.state.data_ptr(), ring.action.data_ptr())
        g = self._graphs.get(key)
        if g is not None:
            return g
        # the warm-up restores every buffer a chunk step mutates
        g = capture_after_warmup(lambda: self._chunk_step(ring, w),
                                 restore=[self.network.grad, self._gsum, self._acc, self._cursor])
        self._graphs[key] = g
        return g

    def learn_episodes(self, ring):
        """One learn over every episode completed in `ring` since the last one; {} if none completed."""
        w = self._workspace(ring)
        N, L, Cr, s = ring.N, ring.L, w["C"], stream_ptr()
        C.jb_episode_returns(ptr(ring.reward), ptr(ring.done), N, L, ptr(ring.pos), ptr(ring.head), float(self.gamma),
                             int(bool(self.use_standardization)), ptr(w["ret_ring"]), ptr(w["count"]), s)
        C.jb_episode_rows(ptr(w["count"]), ptr(ring.head), ptr(w["ret_ring"]), N, L, Cr, ptr(w["offsets"]), ptr(w["idx"]),
                          ptr(w["ret"]), ptr(w["M"]), s)
        M = int(w["M"].item())                               # the one read that decides the chunk count
        self.last_M = M
        if M == 0:
            self.n_launches = 3
            return {}
        n_chunks = -(-M // Cr)
        self._acc.zero_()
        self._cursor.zero_()
        self._gsum.zero_()
        if self.use_cuda_graph:
            g = self._graph_for(ring, w)
            for _ in range(n_chunks):
                g.replay()
        else:
            for _ in range(n_chunks):
                self._chunk_step(ring, w)
        C.jb_copy_f32(ptr(self.network.grad), ptr(self._gsum), self.network.num_flat, s)
        self.optimizer.step()
        self.n_launches = 3 + n_chunks * self.LAUNCHES_PER_CHUNK + 3          # + copy, sumsq, adam
        return {"loss": float(self._acc[0].item())}

    def _single_ring(self, n, state_size):
        """learn()'s one-env ring, grown (to a multiple of 1024 steps) when an episode does not fit."""
        r = self._single
        if r is None or r.L < n:
            r = self._single = EpisodeRing(1, -(-n // 1024) * 1024, state_size, self.action_size, self.action_type,
                                           device=self.device)
        return r

    def learn(self):
        """The reference's learn(): the whole stored buffer is one episode."""
        tr = self.memory.sample()
        n = len(np.asarray(tr["reward"]).reshape(-1))
        state = torch.as_tensor(np.asarray(tr["state"]), dtype=torch.float32, device=self.device).reshape(n, -1)
        ring = self._single_ring(n, state.shape[1])
        ring.state[0, :n].copy_(state)
        a = np.asarray(tr["action"])
        if self.continuous:
            ring.action[0, :n].copy_(torch.as_tensor(a, dtype=torch.float32, device=self.device).reshape(n, -1))
        else:
            ring.action[0, :n].copy_(torch.as_tensor(a.reshape(-1), dtype=torch.int64, device=self.device))
        ring.reward[0, :n].copy_(torch.as_tensor(np.asarray(tr["reward"]).reshape(-1), dtype=torch.float32,
                                                 device=self.device))
        ring.done.zero_()
        ring.done[0, n - 1] = 1.0                            # no reset inside the buffer: one episode ending at its last row
        ring.pos.fill_(n)
        ring.head.zero_()
        return self.learn_episodes(ring)

    def process(self, transitions, step):
        result = {}
        self.memory.store(transitions)
        if np.asarray(transitions[0]["done"]).any():
            result = self.learn()
            if self.lr_decay:
                self.learning_rate_decay(step)
        return result
