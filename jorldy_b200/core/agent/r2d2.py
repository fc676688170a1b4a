"""R2D2 (Kapturowski, Ostrovski, Quan, Munos, Dabney, ICLR 2019): Ape-X's distributed prioritised double-Q learner with
a recurrent dueling Q-network trained on replayed sequences, with the actor's stored recurrent state and a burn-in.

Built on ApeX (per-lane epsilons through jb_q_act, PER sampling and priorities, _stamped_process, clip_grad_norm).  A
replay item is one sequence of L = n_burn_in + seq_len + n_step steps (core/collect.py SequenceAssembler) with the actor's
(h0, c0) from before its first step.  One learn():
  1. PERBuffer.sample_device: B sequences, IS weights (f64), tree indices, {sampled_p, mean_p};
  2. the online trunk (head + input projection) ONCE over the L distinct steps of each sequence, shared by the online
     passes on s and on s' (the same network on the same frames); the trained steps' rows keep their activations;
  3. from the stored (h0, c0): the online LSTM on s over steps 0 .. T_b+T-1 (the first T_b the burn-in, no gradient),
     the online LSTM on s' and the target network (its own trunk) on s', both over steps n .. n+T_b+T-1;
  4. jb_r2d2_loss (csrc/r2d2.cu): double-Q n-step targets under the value rescaling h, (1/(B T)) sum w_b td^2, and the
     sequence priorities (eta max_t |td| + (1 - eta) mean_t |td|)^alpha;
  5. backward over the T trained steps, Adam with clip_grad_norm, the allreduce hook; 6. update_priorities.
New sequences enter the tree at its max priority (no actor-side priorities).

Episode starts.  Sequences may straddle episode ends, as the n-step windows do.  The actor zeroes a lane's (h, c) and
uses no previous action (prev_action -1, an all-zero one-hot) at the first act of an episode; the stored `reset` marks
those steps and the learner's unroll zeroes the state at exactly the same steps.  This replaces the upstream
`zero_padding` (padding a sequence after its episode ends), which is accepted as a key but not implemented.

act(): each lane keeps (h, c) [N, H], its previous action and a reset flag on the device; end_step(done) after the env
step arms the reset.  The single-process driver goes through interact_callback, the batched collector through
`sequence_assembler` and attach_frames(); both use the same assembler.
"""
import numpy as np
import torch

from ..buffer import frame_store
from ..buffer.frame_store import FrameRows
from ..collect import SequenceAssembler
from ..dev import C, ptr, stream_ptr
from ..network import Network
from .dqn import ApeX


class R2D2(ApeX):
    def __init__(self, network="r2d2", seq_len=16, n_burn_in=8, eta=0.9, zero_padding=True, n_step=4, **kwargs):
        super().__init__(network=network, n_step=n_step, **kwargs)
        self.seq_len, self.n_burn_in, self.eta, self.zero_padding = int(seq_len), int(n_burn_in), float(eta), zero_padding
        self.L = self.n_burn_in + self.seq_len + self.n_step
        self.store_period = max(1, self.seq_len // 2)
        self.sequence_assembler = SequenceAssembler(self.n_burn_in, self.seq_len, self.n_step)
        self._frames = None
        self._lanes = None
        self.step_inputs = None
        self._scratch = torch.empty(2 * self.batch_size, dtype=torch.float64, device=self.device)

    def _build_networks(self, network, state_size, action_size, hidden_size, head, kwargs):
        mk = lambda: Network(network, state_size, action_size, D_hidden=hidden_size, head=head, device=self.device,
                             seed=self.seed)
        self.network, self.target_network = mk(), mk()

    # -------------------------------------------------------------------------------------- act --
    def _lane_state(self, M):
        if self._lanes is None or self._lanes["h"].shape[0] != M:
            H = self.network.D_hidden
            z = lambda: torch.zeros(M, H, dtype=torch.float32, device=self.device)
            self._lanes = {"h": z(), "h_alt": z(), "c": z(),
                           "prev": torch.full((M,), -1, dtype=torch.int64, device=self.device),
                           "reset": torch.ones(M, dtype=torch.float32, device=self.device)}
        return self._lanes

    def _q_values(self, state, training, tag="act."):
        """One recurrent step of every lane; records the step's inputs (and (h0, c0) when a window starts there)."""
        ln = self._lane_state(state.shape[0])
        self.step_inputs = {"prev_action": ln["prev"].clone(), "reset": ln["reset"].clone()}
        if self.sequence_assembler.starts_window():
            self.step_inputs.update(h0=ln["h"].clone(), c0=ln["c"].clone())
        q = self.network.step(state, ln["prev"], ln["reset"], ln["h"], ln["c"], ln["h_alt"], tag)
        ln["h"], ln["h_alt"] = ln["h_alt"], ln["h"]
        return q

    def act_device(self, state, training=True, noise=None):
        action, q_sel = super().act_device(state, training, noise)
        ln = self._lanes
        ln["prev"].copy_(action)
        ln["reset"].zero_()
        return action, q_sel

    def end_step(self, done):
        """done f32 [N] of the step just taken: the lanes that finished start their next episode with a zeroed state and
        no previous action."""
        ln = self._lanes
        ln["reset"].copy_(done)
        ln["prev"].masked_fill_(done > 0, -1)

    def interact_callback(self, transition):
        """Single-process driver: the step goes through the same sequence assembler with N = its rows."""
        done = torch.as_tensor(np.asarray(transition["done"], dtype=np.float32).reshape(-1), device=self.device)
        state = self._net_input(self._state_to_device(transition["state"]))
        action = torch.as_tensor(np.asarray(transition["action"]).reshape(-1), dtype=torch.int64, device=self.device)
        reward = torch.as_tensor(np.asarray(transition["reward"], dtype=np.float32).reshape(-1), device=self.device)
        tr = dict(self.step_inputs, state=state, action=action, reward=reward, done=done)
        self.end_step(done)
        return self.sequence_assembler.push(tr) or {}

    def attach_frames(self, env):
        """A single-frame store for `env`'s lanes when it produces Atari stacks: the replayed sequences then hold int64
        frame references, and the CNN head's conv1 im2col reads the ring.  None otherwise."""
        if not getattr(env, "frame_stack", False):
            return None
        F = frame_store.frames_per_lane(self.buffer_size * self.store_period, env.num_envs, self.L)
        self._frames = frame_store.FrameStore(env.num_envs, F, self.device)
        return self._frames

    # ------------------------------------------------------------------------------------ learn --
    def _learn_seq(self, batch, weights):
        B, L, Tb, T, n = batch["reward"].shape[0], self.L, self.n_burn_in, self.seq_len, self.n_step
        A, S = self.action_size, self.n_burn_in + self.seq_len
        tm = lambda t: t.transpose(0, 1).contiguous()
        state = batch["state"]
        if state.dtype == torch.int64:
            if self._frames is None:
                raise RuntimeError("these sequences hold frame references but no frame store is attached")
            x = FrameRows(self._frames, tm(state).view(-1))
        else:
            x = tm(state).view(L * B, *state.shape[2:])
            if x.dtype != torch.uint8:
                x = x.to(torch.float32).reshape(L * B, -1)
        prev = tm(batch["prev_action"].to(torch.int64)).view(-1)
        reset = tm(batch["reset"].to(torch.float32))
        h0, c0 = batch["h0"].contiguous(), batch["c0"].contiguous()
        net, tgt = self.network, self.target_network
        bm = lambda q: q.view(T, B, A).transpose(0, 1).contiguous()
        xg = net.encode(x, prev, L, B, Tb, S, "t.")
        q = bm(net.unroll(xg, 0, S, B, reset, h0, c0, Tb, "t."))
        q_next = bm(net.unroll(xg, n, S, B, reset, h0, c0, Tb, "n.", save=False))
        xg_t = tgt.encode(x[n * B:], prev[n * B:], S, B, 0, 0, "n.")
        qt_next = bm(tgt.unroll(xg_t, 0, S, B, reset[n:], h0, c0, Tb, "n.", save=False))
        action = batch["action"][:, Tb:S].to(torch.int64).contiguous()
        reward = batch["reward"][:, Tb:].to(torch.float32).contiguous()
        done = batch["done"][:, Tb:].to(torch.float32).contiguous()
        dq = net._buf("t.dq", (B, T, A))
        prio = net._buf("t.prio", (B,), torch.float64)
        if self._scratch.numel() < 2 * B:
            self._scratch = torch.empty(2 * B, dtype=torch.float64, device=self.device)
        C.jb_r2d2_loss(ptr(q), ptr(q_next), ptr(qt_next), ptr(action), ptr(reward), ptr(done), ptr(weights), B, T, A, n,
                       self.gamma, float(self.alpha), self.eta, ptr(dq), ptr(prio), ptr(self._stats), ptr(self._scratch),
                       stream_ptr())
        net.backward_tm(tm(dq).view(T * B, A), "t.")
        self._optimizer_step()
        return prio

    def learn(self):
        batch, weights, indices, stats_per = self._per_sample()
        prio = self._learn_seq(batch, weights)
        self.memory.update_priorities(indices, prio)
        loss, max_q, sampled_p, mean_p = self._per_result(stats_per)
        if self._frames is not None:
            self._frames.check()
        return {"loss": loss, "max_Q": max_q, "sampled_p": sampled_p, "mean_p": mean_p, "num_learn": self.num_learn,
                "num_transitions": self.num_transitions}
