"""Munchausen agents (Vieillard, Pietquin, Geist 2020, arXiv:2007.14430): M-DQN on DQN and M-IQN on IQN.

Both add the scaled, clipped log-policy of the taken action to the reward and bootstrap from the soft value of s', with
pi = softmax(q' / tau) of the TARGET network:
    y = r + alpha clip(tau logpi(a_t|s), l_0, 0) + ((1 - d) gamma) sum_a pi'(a) (q'(s', a) - tau logpi'(a|s'))
One learn() = replay gather -> online forward on s, target forwards on s' and on s (tag "m.") -> ONE Munchausen loss launch
pair (jb_mdqn_loss / jb_munchausen_quantile_loss, csrc/munchausen.cuh) -> backward -> Adam.  M-DQN's loss is DQN's
smooth_l1; M-IQN's is IQN's quantile Huber, with q'(s, .) and q'(s', .) the target network's per-action quantile means.
process(), act(), the replay, epsilon, target updates, save / load and learn()'s result keys are DQN's / IQN's.

The constructor keys alpha, tau and l_0 are stored as m_alpha, m_tau and m_l0: DQN keeps its PER exponent in self.alpha.
M-IQN draws three fraction sets per learn from IQN's Philox stream, in this order: tau(s) for the online pass on s,
tau'(s') for the target pass on s', tau''(s) for the target pass on s (tests inject them as _inject_tau[0], [1], [3];
[2] is act()'s).
"""
from ..dev import C, ptr, stream_ptr
from .dqn import DQN, _action_kind
from .quantile import IQN


class _Munchausen:
    def _set_munchausen(self, alpha, tau, l_0):
        if not tau > 0 or not l_0 <= 0:
            raise ValueError(f"Munchausen RL needs tau > 0 and l_0 <= 0 (got tau={tau}, l_0={l_0})")
        self.m_alpha, self.m_tau, self.m_l0 = float(alpha), float(tau), float(l_0)


class MDQN(_Munchausen, DQN):
    def __init__(self, state_size, action_size, alpha=0.9, tau=0.03, l_0=-1, **kwargs):
        super().__init__(state_size, action_size, **kwargs)
        self._set_munchausen(alpha, tau, l_0)

    def _learn_batch(self, batch, weights=None):
        B, state, next_state, reward, done, action = self._batch_tensors(batch, 1)
        A, net, tgt = self.action_size, self.network, self.target_network
        q = net.forward(state, tag="t.")
        qt_next = tgt.forward(next_state, tag="n.")
        qt_s = tgt.forward(state, tag="m.")
        dq = net._buf("t.dq", (B, A))
        scratch = net._buf("t.mscratch", (2 * B,))
        C.jb_mdqn_loss(ptr(q), ptr(qt_s), ptr(qt_next), ptr(action), _action_kind(action), ptr(reward), ptr(done), B, A,
                       self.gamma, self.m_alpha, self.m_tau, self.m_l0, ptr(dq), ptr(self._stats), ptr(scratch),
                       stream_ptr())
        net.backward(dq, B, tag="t.")
        self._optimizer_step()


class MIQN(_Munchausen, IQN):
    def __init__(self, state_size, action_size, alpha=0.9, tau=0.03, l_0=-1, **kwargs):
        super().__init__(state_size, action_size, **kwargs)
        self._set_munchausen(alpha, tau, l_0)

    def _learn_batch(self, batch, weights=None):
        B, state, next_state, reward, done, action = self._batch_tensors(batch, 1)
        A, N, net, tgt = self.action_size, self.num_sample, self.network, self.target_network
        tau = self._draw_tau(B, 0.0, 1.0, "t.tau", 0)
        tau_next = self._draw_tau(B, 0.0, 1.0, "n.tau", 1)
        tau_cur = self._draw_tau(B, 0.0, 1.0, "m.tau", 3)
        theta = net.forward(state, tau, tag="t.")
        theta_next = tgt.forward(next_state, tau_next, tag="n.")
        theta_cur = tgt.forward(state, tau_cur, tag="m.")
        dtheta = net._buf("t.dtheta", theta.shape)
        scratch = net._buf("t.qscratch", (2 * B,))
        C.jb_munchausen_quantile_loss(ptr(theta), ptr(theta_next), ptr(theta_cur), ptr(tau), N, ptr(action),
                                      _action_kind(action), ptr(reward), ptr(done), B, A, N, N, N, self.gamma,
                                      self.m_alpha, self.m_tau, self.m_l0, ptr(dtheta), ptr(self._stats), ptr(scratch),
                                      stream_ptr())
        self._backward(dtheta, B)
        self._optimizer_step()
