"""Quantile-regression agents: QR-DQN (Dabney et al. 2017, arXiv:1710.10044) and IQN (Dabney et al. 2018,
arXiv:1806.06923), on DQN's replay, epsilon and target-update bookkeeping (process() is DQN's, unchanged).

One learn() = replay gather -> online forward on s and target forward on s' -> ONE quantile Huber loss launch pair
(csrc/quantile.cu jb_quantile_loss: a*, targets, loss, gradient, stats) -> backward -> Adam.  The loss is
(1/B) sum_b (1/N') sum_j sum_i |tau_i - 1{u_ij < 0}| smooth_l1(u_ij), u_ij = y_j - theta_i, kappa = 1.

QR-DQN: the `discrete_q_network` with A*K outputs viewed as [B, A, K] (C51's layout), fixed fractions
tau_i = (2i + 1) / (2K), a* = argmax of the TARGET net's mean on s', Q = mean_k theta_k.
IQN: the `iqn` network, N = N' = num_sample fractions drawn from U(0, 1) independently for the online pass on s and
the target pass on s' (a* = argmax of the target pass's own mean); act() averages num_sample draws from
U(sample_min, sample_max).  All draws come from one Philox stream per agent with a device counter (jb_iqn_tau).
"""
import numpy as np
import torch

from ..dev import C, ptr, stream_ptr
from ..network import Network
from .dqn import DQN, _action_kind

TAU_STREAM = 0x5141_4E00_0000_0000      # Philox stream id of IQN's fraction draws (q_act uses ids 0 .. lanes - 1)


class _Quantile:
    """The quantile loss launch shared by QRDQN and IQN."""

    def _quantile_step(self, batch, fwd, tau, tau_stride, layout, N):
        """fwd(net, x, tag) -> quantile output; layout = (sa, sq) of [B, A, K] or [B, N, A]."""
        B, state, next_state, reward, done, action = self._batch_tensors(batch, 1)
        A = self.action_size
        net, tgt = self.network, self.target_network
        theta = fwd(net, state, "t.", 0)
        theta_next = fwd(tgt, next_state, "n.", 1)
        dtheta = net._buf("t.dtheta", theta.shape)
        loss = net._buf("t.qloss", (B,))
        a_star = net._buf("t.astar", (B,), torch.int32)
        scratch = net._buf("t.qscratch", (2 * B,))
        sa, sq = layout
        C.jb_quantile_loss(ptr(theta), sa, sq, ptr(theta_next), sa, sq, ptr(tau), tau_stride, ptr(action),
                           _action_kind(action), ptr(reward), ptr(done), B, A, N, N, self.gamma, ptr(dtheta), ptr(loss),
                           ptr(a_star), ptr(self._stats), ptr(scratch), stream_ptr())
        self._backward(dtheta, B)
        self._optimizer_step()


class QRDQN(_Quantile, DQN):
    def __init__(self, state_size, action_size, num_support=200, **kwargs):
        self.num_support = num_support
        super().__init__(state_size, action_size * num_support, **kwargs)
        self.action_size = action_size
        K = num_support
        self.tau = torch.tensor((2 * np.arange(K) + 1) / (2.0 * K), dtype=torch.float32, device=self.device)

    def _q_values(self, state, training, tag="act."):
        M, A, K = state.shape[0], self.action_size, self.num_support
        theta = self.network._buf(tag + "theta", (M, A * K))
        self.network.forward_rows(state, theta)
        q = self.network._buf(tag + "q", (M, A))
        C.jb_quantile_mean(ptr(theta), K, 1, M, A, K, ptr(q), stream_ptr())
        return q

    def _backward(self, dtheta, B):
        self.network.backward(dtheta, B, tag="t.")

    def _learn_batch(self, batch, weights=None):
        self._quantile_step(batch, lambda net, x, tag, _: net.forward(x, tag=tag), self.tau, 0,
                            (self.num_support, 1), self.num_support)


class IQN(_Quantile, DQN):
    def __init__(self, state_size, action_size, network="iqn", num_sample=64, embedding_dim=64, sample_min=0.0,
                 sample_max=1.0, **kwargs):
        self.num_sample, self.embedding_dim = num_sample, embedding_dim
        self.sample_min, self.sample_max = sample_min, sample_max
        super().__init__(state_size, action_size, network=network, **kwargs)
        self._tau_ctr = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._inject_tau = None        # tests: [tau(s) [B,N], tau'(s') [B,N], tau(act) [M,N]] for the next learn / act

    def _build_networks(self, network, state_size, action_size, hidden_size, head, kwargs):
        mk = lambda: Network(network, state_size, action_size, D_em=self.embedding_dim, D_hidden=hidden_size, head=head,
                             device=self.device)
        self.network, self.target_network = mk(), mk()

    def _draw_tau(self, rows, lo, hi, tag, which):
        tau = self.network._buf(tag, (rows, self.num_sample))
        inj = self._inject_tau[which] if self._inject_tau is not None else None
        if inj is not None:
            tau.copy_(torch.as_tensor(np.asarray(inj), dtype=torch.float32).reshape(rows, self.num_sample))
        else:
            C.jb_iqn_tau(ptr(tau), rows, self.num_sample, float(lo), float(hi), self.seed, TAU_STREAM, ptr(self._tau_ctr),
                         stream_ptr())
        return tau

    def _q_values(self, state, training, tag="act."):
        M, A, N = state.shape[0], self.action_size, self.num_sample
        tau = self._draw_tau(M, self.sample_min, self.sample_max, tag + "tau", 2)
        theta = self.network._buf(tag + "theta", (M * N, A))
        self.network.forward_rows(state, tau, theta)
        q = self.network._buf(tag + "q", (M, A))
        C.jb_quantile_mean(ptr(theta), 1, A, M, A, N, ptr(q), stream_ptr())
        return q

    def _backward(self, dtheta, B):
        self.network.backward(dtheta, tag="t.")

    def _learn_batch(self, batch, weights=None):
        B = batch["reward"].shape[0]
        taus = [self._draw_tau(B, 0.0, 1.0, "t.tau", 0), self._draw_tau(B, 0.0, 1.0, "n.tau", 1)]
        self._quantile_step(batch, lambda net, x, tag, k: net.forward(x, taus[k], tag=tag), taus[0], self.num_sample,
                            (1, self.action_size), self.num_sample)
