"""Rainbow-IQN (Toromanoff, Wirbel, Moutarde 2019, arXiv:1908.04683): IQN (arXiv:1806.06923) with Rainbow's
(arXiv:1710.02298) double-Q action choice, n-step targets, prioritised replay and noisy dueling network.

Built from PER (sampling, beta schedule, _stamped_process), Rainbow (act() gate, n-step windows through
interact_callback) and IQN (fractions from one Philox stream per agent with a device counter).  One learn():
  1. the PER sample: batch, IS weights w_b (f64, max-normalised), tree indices, {sampled_p, mean_p};
  2. three forwards of the `rainbow_iqn` network, each with its own fractions from U(0, 1) and its own fresh noise, drawn
     in this order: tau(s) then the online net on s; tau''(s') then the online net on s'; tau'(s') then the target net
     on s' (fractions before the forward's a1, v1, a2, v2 noise).  N = N' = N'' = num_sample;
  3. ONE loss launch pair (csrc/quantile.cu jb_rainbow_iqn_loss):
       a*  = argmax_a mean_j online(s')[b, j, a], first index on ties (double-Q);
       y_j = fold_{s = n-1 .. 0} (r_s + ((1 - d_s) gamma) y), from y = target(s')[b, j, a*];
       L_b = (1/N') sum_j sum_i |tau_i - 1{u_ij < 0}| smooth_l1(u_ij),  u_ij = y_j - theta_i(s, a_t),  kappa = 1;
       loss = (1/B) sum_b w_b L_b (each sample its own IS weight, as PER and Ape-X here and as the paper says; Rainbow's
       batch-mean weight, csrc/c51.cu, is a quirk of the upstream C51 loss not carried over without evidence);
       new priorities p_b = L_b^alpha from the unweighted per-sample loss;
  4. backward, Adam, the allreduce hook, num_learn += 1; the priorities go back through update_priorities.
act(): uniform random actions before max(batch_size, start_train_step) stored transitions, then the argmax of the quantile
means over num_sample fractions from U(sample_min, sample_max), no epsilon.  The noise is drawn once per act() call for all
rows; training=False uses the mu weights.  Tests inject _inject_u (PER uniforms), _inject_tau = [tau(s), tau''(s') online,
tau'(s') target, tau(act)] and _inject_noise = 3 x [(eps_i, eps_j)] x 4.
"""
from collections import deque

import torch

from ..dev import C, ptr, stream_ptr
from ..network import Network
from .dqn import PER, Rainbow, _action_kind
from .quantile import IQN


class RainbowIQN(PER):
    _decay_eps = False

    def __init__(self, state_size, action_size, hidden_size=512, network="rainbow_iqn", head="mlp",
                 optim_config={"name": "adam"}, gamma=0.99, buffer_size=50000, batch_size=64, start_train_step=2000,
                 target_update_period=500, run_step=1e6, lr_decay=True, n_step=4, alpha=0.6, beta=0.4, learn_period=4,
                 uniform_sample_prob=1e-3, noise_type="factorized", num_sample=64, embedding_dim=64, sample_min=0.0,
                 sample_max=1.0, device=None, seed=0, **kwargs):
        self._noise_type = noise_type
        self.num_sample, self.embedding_dim = num_sample, embedding_dim
        self.sample_min, self.sample_max = sample_min, sample_max
        super().__init__(alpha=alpha, beta=beta, learn_period=learn_period, uniform_sample_prob=uniform_sample_prob,
                         run_step=run_step, state_size=state_size, action_size=action_size, hidden_size=hidden_size,
                         network=network, head=head, optim_config=optim_config, gamma=gamma, buffer_size=buffer_size,
                         batch_size=batch_size, start_train_step=start_train_step,
                         target_update_period=target_update_period, lr_decay=lr_decay, device=device, seed=seed)
        self.n_step = n_step
        self.tmp_buffer = deque(maxlen=n_step)
        self._tau_ctr = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._inject_tau = None
        self._inject_noise = None

    def _build_networks(self, network, state_size, action_size, hidden_size, head, kwargs):
        mk = lambda s: Network(network, state_size, action_size, D_em=self.embedding_dim, noise_type=self._noise_type,
                               D_hidden=hidden_size, head=head, device=self.device, seed=s)
        self.network, self.target_network = mk(self.seed), mk(self.seed + 1)

    _draw_tau = IQN._draw_tau
    process = Rainbow.process
    learn = Rainbow.learn
    interact_callback = Rainbow.interact_callback

    def act_device(self, state, training=True, noise=None):
        """noise: injected draws [(eps_i, eps_j)] x 4 (a1, v1, a2, v2) for this call's single noisy forward."""
        M = state.shape[0]
        action = self._warmup_actions(M, training)
        if action is not None:
            return action, None
        A, N = self.action_size, self.num_sample
        tau = self._draw_tau(M, self.sample_min, self.sample_max, "act.tau", 3)
        theta = self.network._buf("act.theta", (M * N, A))
        self.network.forward_rows(state, tau, theta, is_train=training, noise=noise)
        q = self.network._buf("act.q", (M, A))
        C.jb_quantile_mean(ptr(theta), 1, A, M, A, N, ptr(q), stream_ptr())
        return torch.argmax(q, -1), None

    def _learn_batch(self, batch, weights=None):
        B, state, next_state, reward, done, action = self._batch_tensors(batch)
        A, N = self.action_size, self.num_sample
        net, tgt = self.network, self.target_network
        noise = self._inject_noise or [None, None, None]
        tau = self._draw_tau(B, 0.0, 1.0, "t.tau", 0)
        theta = net.forward(state, tau, True, "t.", noise[0])
        tau_online = self._draw_tau(B, 0.0, 1.0, "n.tau", 1)
        theta_online = net.forward(next_state, tau_online, True, "n.", noise[1])
        tau_target = self._draw_tau(B, 0.0, 1.0, "g.tau", 2)
        theta_target = tgt.forward(next_state, tau_target, True, "n.", noise[2])
        dtheta = net._buf("t.dtheta", theta.shape)
        loss = net._buf("t.qloss", (B,))
        prio = net._buf("t.prio", (B,), torch.float64)
        scratch = net._buf("t.riqn_scratch", (4 * B,))
        C.jb_rainbow_iqn_loss(ptr(theta), ptr(theta_online), ptr(theta_target), ptr(tau), ptr(action), _action_kind(action),
                              ptr(reward), ptr(done), ptr(weights), B, A, N, N, N, reward.shape[1], self.gamma,
                              float(self.alpha), ptr(dtheta), ptr(loss), ptr(prio), None, ptr(self._stats), ptr(scratch),
                              stream_ptr())
        net.backward(dtheta, tag="t.")
        self._optimizer_step()
        return prio
