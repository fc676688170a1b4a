"""Off-policy actor-critic agents on the GPU-resident pipeline: DDPG, TD3 and SAC (continuous actions), and the
discrete-action SAC (SACDiscrete, selected by SAC's `actor="discrete_policy"`).

Mirrors jorldy/core/agent/{ddpg,td3,sac}.py: same constructor kwargs, optimiser layout (one optimiser per network),
bookkeeping (soft target updates, TD3's delayed actor update, SAC's one-step-lagged alpha) and result keys.
One learn() = replay gather on the device -> target actor / target critics -> TD target + MSE gradient for the
critic(s) (csrc/actor_critic.cu) -> critic backward + Adam -> actor forward -> critic forward on the actor's action
-> d q / d action -> actor backward + Adam -> soft update.  All randomness (exploration, TD3 target smoothing, SAC's
reparameterisation noise) is Philox on the device, or injected by the parity tests.
"""
import os

import numpy as np
import torch

from ..buffer import ReplayBuffer
from ..dev import C, ptr, require_cuda, stream_ptr
from ..network import Network
from ..network.base import FlatNetwork
from ..optimizer import Optimizer
from .base import BaseAgent, cpu_optimizer_state, cpu_state_dict

_DEFAULT_OPTIM = {"actor": "adam", "critic": "adam", "actor_lr": 5e-4, "critic_lr": 1e-3}


class _Scalar(FlatNetwork):
    """Learnable scalars held like a network so that the flat Adam applies: SAC's log_alpha (sac.py:95-100), or V-MPO's
    [eta, alpha_mu, alpha_sigma] as one contiguous vector when `value` is a sequence."""

    def __init__(self, name, value, device):
        super().__init__(device)
        values = [float(v) for v in np.atleast_1d(value)]
        self._specs = [(name, (len(values),))]
        self._allocate()
        self.flat[:len(values)] = torch.tensor(values, dtype=torch.float32)


class _ActorCritic(BaseAgent):
    action_type = "continuous"
    _n_critics = 1
    _strict_gate = False        # learn once memory.size > batch_size (SAC) instead of >= batch_size (DDPG, TD3)
    _soft_in_process = True     # process() soft-updates the targets (TD3 does it inside its delayed learn() steps)

    def _common(self, state_size, action_size, hidden_size, actor, critic, head, optim_config, gamma, buffer_size, batch_size,
                start_train_step, tau, run_step, lr_decay, device, seed, target_actor, use_cuda_graph=True):
        self.device = require_cuda(device)
        self.use_cuda_graph = bool(use_cuda_graph)
        self._graphs, self._warm, self._idx_buf = {}, set(), None
        self.state_size, self.action_size = state_size, action_size
        self.seed = int(seed)
        mk = lambda name: Network(name, state_size, action_size, D_hidden=hidden_size, head=head, device=self.device)
        self.actor = mk(actor)
        self.actor_optimizer = Optimizer(optim_config["actor"], params=self.actor.parameters(), lr=optim_config["actor_lr"])
        if target_actor:
            self.target_actor = mk(actor)
            self.target_actor.copy_from(self.actor)
        self.critics, self.target_critics, self.critic_optimizers = [], [], []
        for _ in range(self._n_critics):
            c, t = mk(critic), mk(critic)
            t.copy_from(c)
            self.critics.append(c)
            self.target_critics.append(t)
            self.critic_optimizers.append(Optimizer(optim_config["critic"], params=c.parameters(), lr=optim_config["critic_lr"]))
        self.network = self.actor                       # sync_in / sync_out ship the actor (ddpg.py:199-210)
        self.gamma, self.tau = gamma, tau
        self.memory = ReplayBuffer(buffer_size, device=self.device)
        self.batch_size, self.start_train_step = batch_size, start_train_step
        self.run_step, self.lr_decay = run_step, lr_decay
        self.num_learn = 0
        self.n_step = 1
        self.rng_stream_base = 0
        self._stats = torch.zeros(16, dtype=torch.float32, device=self.device)
        self._fill_ctr = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._row_ctr = {}
        self._inject_idx = None         # tests: fixed replay indices for the next learn()
        self._inject_noise = None       # tests: dict of injected normal draws for the next learn()

    # ---- plumbing ----------------------------------------------------------------------------------------------------
    def _optimizers(self):
        return [self.actor_optimizer] + self.critic_optimizers

    def _all_optimizers(self):
        return self._optimizers()

    def _fill(self, key, shape, purpose, kind=0, lo=0.0, hi=1.0):
        """Standard normals (kind 0) / uniforms in [lo, hi) (kind 1) from the device Philox stream of this agent."""
        out = self.actor._buf("rng." + key, shape)
        C.jb_philox_fill(ptr(out), out.numel(), kind, lo, hi, self.seed, self.rng_stream_base + (purpose << 40), 0,
                         ptr(self._fill_ctr), stream_ptr())
        return out

    def _net_input(self, s):
        return s.to(torch.float32).reshape(s.shape[0], -1)

    def _sample(self):
        return self.memory.gather_device(self._replay_indices(self.device))

    def _unpack(self, batch):
        B = batch["reward"].shape[0]
        f = lambda k, w: batch[k].to(torch.float32).reshape(B, w).contiguous()
        return (B, f("state", -1), f("action", self.action_size), f("reward", 1).view(B), f("done", 1).view(B),
                f("next_state", -1))

    def _tanh(self, net, pre, key, noise=None, scale=0.0, noise_clip=0.0, out_clip=0.0):
        out = net._buf(key, tuple(pre.shape))
        C.jb_tanh_act(ptr(pre), ptr(noise), pre.numel(), scale, noise_clip, out_clip, ptr(out), stream_ptr())
        return out

    def _critic_step(self, i, dq, B):
        self.critics[i].backward(dq, B, tag="t.")
        self.critic_optimizers[i].step()

    def _soft(self, target, online):
        C.jb_soft_update(ptr(target.flat), ptr(online.flat), online.num_flat, float(self.tau), stream_ptr())

    def update_target_soft(self):
        for t, c in zip(self.target_critics, self.critics):
            self._soft(t, c)
        if hasattr(self, "target_actor"):
            self._soft(self.target_actor, self.actor)

    @torch.no_grad()
    def act(self, state, training=True):
        self.actor.train(training)
        action, _ = self.act_device(self._net_input(self._state_to_device(state)), training)
        return {"action": action.cpu().numpy()}

    def _learn_batch(self, batch):
        """One eager learn() on a device batch (the parity tests call this with injected draws)."""
        self._learn_core(batch)
        return self._finish()

    def _variant(self):
        """Host-side state that changes WHICH kernels a learn() launches (TD3's delayed actor / target updates)."""
        return 0

    def learn(self):
        """replay gather + _learn_core as ONE CUDA-graph replay (~90 launches otherwise).  The first learn of every variant runs
        eagerly (it allocates the workspaces and is a real learn), the second captures, later ones replay; the minibatch indices
        travel through a static device buffer, lr / Adam step / Philox counters live in device memory."""
        if not self.use_cuda_graph or self._inject_noise is not None:
            return self._learn_batch(self._sample())
        B = self.batch_size
        if self._idx_buf is None:
            self._idx_buf = torch.zeros(B, dtype=torch.int64, device=self.device)
        self._idx_buf.copy_(self._replay_indices())
        for opt in self._all_optimizers():
            opt._sync_lr()                       # graph replays do not pass through optimizer.step()'s host-side lr check
        key = self._variant()
        if key not in self._warm:
            self._warm.add(key)
            self._learn_core(self.memory.gather_device(self._idx_buf))
        else:
            g = self._graphs.get(key)
            if g is None:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):        # capture does not execute
                    self._learn_core(self.memory.gather_device(self._idx_buf))
                self._graphs[key] = g
            g.replay()
        return self._finish()

    def process(self, transitions, step):
        """ddpg.py / td3.py / sac.py process(): store; learn and decay the learning rates once the replay holds a batch and
        step >= start_train_step; then, once learning has started, soft-update the targets on every call."""
        result = {}
        self.memory.store(transitions)
        filled = self.memory.size > self.batch_size if self._strict_gate else self.memory.size >= self.batch_size
        if filled and step >= self.start_train_step:
            result = self.learn()
            if self.lr_decay:
                self.learning_rate_decay(step, self._optimizers())
        if self._soft_in_process and self.num_learn > 0:
            self.update_target_soft()
        return result

    # ---- checkpoints: the reference's key layout (ddpg.py:176-197, td3.py:222-246, sac.py:306-339) ---------------------
    def _ckpt(self):
        d = {"actor": cpu_state_dict(self.actor), "actor_optimizer": cpu_optimizer_state(self.actor_optimizer)}
        if self._n_critics == 1:
            d["critic"] = cpu_state_dict(self.critics[0])
            d["critic_optimizer"] = cpu_optimizer_state(self.critic_optimizers[0])
        else:
            for i in (0, 1):
                d[f"critic{i + 1}"] = cpu_state_dict(self.critics[i])
                d[f"critic_optimizer{i + 1}"] = cpu_optimizer_state(self.critic_optimizers[i])
        return d

    def save(self, path):
        print(f"...Save model to {path}...")
        torch.save(self._ckpt(), os.path.join(path, "ckpt"))

    def _load_common(self, ck):
        self.actor.load_state_dict(ck["actor"])
        self.actor_optimizer.load_state_dict(ck["actor_optimizer"])
        if self._n_critics == 1:
            self.critics[0].load_state_dict(ck["critic"])
            self.target_critics[0].copy_from(self.critics[0])
            self.critic_optimizers[0].load_state_dict(ck["critic_optimizer"])
        else:
            # td3.py:238-241 / sac.py:328-331 load checkpoint["critic2"] INTO critic1 (after critic1's own weights) and never
            # touch critic2; reproduced so that a resumed run continues from the same state as the reference's.
            self.critics[0].load_state_dict(ck["critic1"])
            self.critics[0].load_state_dict(ck["critic2"])
            self.target_critics[0].copy_from(self.critics[0])
            self.target_critics[1].copy_from(self.critics[1])
            self.critic_optimizers[0].load_state_dict(ck["critic_optimizer1"])
            self.critic_optimizers[1].load_state_dict(ck["critic_optimizer2"])

    def load(self, path):
        print(f"...Load model from {path}...")
        self._load_common(torch.load(os.path.join(path, "ckpt"), map_location="cpu", weights_only=False))


class DDPG(_ActorCritic):
    """jorldy/core/agent/ddpg.py:14-211."""

    def __init__(self, state_size, action_size, hidden_size=512, actor="deterministic_policy", critic="continuous_q_network",
                 head="mlp", optim_config=_DEFAULT_OPTIM, gamma=0.99, buffer_size=50000, batch_size=128,
                 start_train_step=2000, tau=1e-3, run_step=1e6, lr_decay=True, mu=0, theta=1e-3, sigma=2e-3, device=None,
                 seed=0, use_cuda_graph=True, **kwargs):
        self._common(state_size, action_size, hidden_size, actor, critic, head, optim_config, gamma, buffer_size, batch_size,
                     start_train_step, tau, run_step, lr_decay, device, seed, target_actor=True, use_cuda_graph=use_cuda_graph)
        self.ou_mu, self.ou_theta, self.ou_sigma = float(mu), float(theta), float(sigma)
        self._ou = {}                    # rows -> OU state X [rows, A] f64 (one process per batched env)

    def act_device(self, state, training=True, noise=None):
        """state [N, D] f32 -> action [N, A] f32: tanh(actor(s)) + clip(OU, -1, 1) when training (ddpg.py:113-118);
        noise: optional f64 [N] normals (one per env and step, utils.py:22)."""
        M, A = state.shape[0], self.action_size
        pre = self.actor._buf("act.pre", (M, A))
        self.actor.forward_rows(state, pre)
        if M not in self._ou:
            self._ou[M] = torch.full((M, A), self.ou_mu, dtype=torch.float64, device=self.device)
        row_ctr = self._row_counter(M)
        action = self.actor._buf("act.a", (M, A))
        C.jb_ou_act(ptr(pre), M, A, ptr(self._ou[M]), ptr(noise), self.seed, self.rng_stream_base, ptr(row_ctr),
                    self.ou_theta, self.ou_mu, self.ou_sigma, 0 if training else 1, ptr(action), stream_ptr())
        return action, None

    def _learn_core(self, batch):
        B, s, a, r, d, ns = self._unpack(batch)
        critic, tcritic = self.critics[0], self.target_critics[0]
        na = self._tanh(self.target_actor, self.target_actor.forward_raw(ns, tag="n.", save=False), "n.a")
        nq = tcritic.forward(ns, na, tag="n.")
        q = critic.forward(s, a, tag="t.")
        dq = critic._buf("t.dq", (B, 1))
        C.jb_ac_critic_loss(ptr(q), 0, ptr(nq), 0, 0, 0, ptr(r), ptr(d), B, self.gamma, ptr(dq), 0, ptr(self._stats),
                            stream_ptr())
        self._critic_step(0, dq, B)
        self._actor_step(s, B)

    def _finish(self):
        self.num_learn += 1
        st = self._stats[:5].cpu().numpy()
        return {"critic_loss": float(st[0]), "actor_loss": float(st[4]), "max_Q": float(st[2])}

    def _actor_step(self, s, B):
        """L = -mean(critic(s, actor(s))) through the UPDATED critic (ddpg.py:142-148, td3.py:175-181)."""
        critic = self.critics[0]
        ap = self._tanh(self.actor, self.actor.forward_raw(s, tag="t."), "t.a")
        qa = critic.forward(s, ap, tag="a.")
        dqa = critic._buf("a.dq", (B, 1))
        C.jb_ac_neg_mean(ptr(qa), B, ptr(dqa), self._stats.data_ptr() + 16, stream_ptr())
        da = critic.backward(dqa, B, tag="a.", params=False, want_dx2=True)
        dpre = self.actor._buf("t.dpre", (B, self.action_size))
        C.jb_tanh_bwd(ptr(da), ptr(ap), ap.numel(), ptr(dpre), stream_ptr())
        self.actor.backward_raw(dpre, B, tag="t.")
        self.actor_optimizer.step()


class TD3(DDPG):
    """jorldy/core/agent/td3.py:13-265: twin critics, clipped target-policy smoothing, delayed actor + target updates."""
    _n_critics = 2
    _soft_in_process = False

    def __init__(self, state_size, action_size, hidden_size=512, actor="deterministic_policy", critic="continuous_q_network",
                 head="mlp", optim_config=_DEFAULT_OPTIM, gamma=0.99, buffer_size=50000, batch_size=128,
                 start_train_step=2000, initial_random_step=0, tau=1e-3, update_delay=2, action_noise_std=0.1,
                 target_noise_std=0.2, target_noise_clip=0.5, run_step=1e6, lr_decay=True, device=None, seed=0,
                 use_cuda_graph=True, **kwargs):
        self._common(state_size, action_size, hidden_size, actor, critic, head, optim_config, gamma, buffer_size, batch_size,
                     start_train_step, tau, run_step, lr_decay, device, seed, target_actor=True, use_cuda_graph=use_cuda_graph)
        self.initial_random_step, self.num_random_step = initial_random_step, 0
        self.update_delay = update_delay
        self.action_noise_std, self.target_noise_std, self.target_noise_clip = action_noise_std, target_noise_std, target_noise_clip
        self.actor_loss = 0.0

    def act_device(self, state, training=True, noise=None):
        """td3.py:131-143: uniform(-1, 1) actions for the first initial_random_step calls, then
        clip(tanh(actor(s)) + N(0, action_noise_std), -1, 1); noise: optional f32 [N, A] standard normals."""
        M, A = state.shape[0], self.action_size
        if training and self.num_random_step < self.initial_random_step:
            self.num_random_step += 1
            return self._fill(f"act.u{M}", (M, A), 1, kind=1, lo=-1.0, hi=1.0), None
        pre = self.actor._buf("act.pre", (M, A))
        self.actor.forward_rows(state, pre)
        if not training:
            return self._tanh(self.actor, pre, "act.a"), None
        if noise is None:
            noise = self._fill(f"act.n{M}", (M, A), 1)
        return self._tanh(self.actor, pre, "act.a", noise, self.action_noise_std, 0.0, 1.0), None

    def _variant(self):
        upd = self.num_learn % self.update_delay == 0
        return (upd, upd and self.num_learn > 0)         # (actor step, soft target update) — td3.py:174-183

    def _learn_core(self, batch):
        B, s, a, r, d, ns = self._unpack(batch)
        inj = self._inject_noise or {}
        noise = inj.get("target")
        if noise is None:
            noise = self._fill("t.noise", (B, self.action_size), 2)
        na = self._tanh(self.target_actor, self.target_actor.forward_raw(ns, tag="n.", save=False), "n.a", noise,
                        self.target_noise_std, self.target_noise_clip, 1.0)
        nq1 = self.target_critics[0].forward(ns, na, tag="n.")
        nq2 = self.target_critics[1].forward(ns, na, tag="n.")
        q1 = self.critics[0].forward(s, a, tag="t.")
        q2 = self.critics[1].forward(s, a, tag="t.")
        dq1, dq2 = self.critics[0]._buf("t.dq", (B, 1)), self.critics[1]._buf("t.dq", (B, 1))
        C.jb_ac_critic_loss(ptr(q1), ptr(q2), ptr(nq1), ptr(nq2), 0, 0, ptr(r), ptr(d), B, self.gamma, ptr(dq1), ptr(dq2),
                            ptr(self._stats), stream_ptr())
        self._critic_step(0, dq1, B)
        self._critic_step(1, dq2, B)
        actor_updated, soft = self._variant()
        if actor_updated:
            self._actor_step(s, B)
            if soft:
                self.update_target_soft()

    def _finish(self):
        actor_updated = self.num_learn % self.update_delay == 0
        self.num_learn += 1
        st = self._stats[:5].cpu().numpy()
        if actor_updated:
            self.actor_loss = float(st[4])
        return {"critic_loss1": float(st[0]), "critic_loss2": float(st[1]), "actor_loss": self.actor_loss, "max_Q": float(st[2])}


class SAC(_ActorCritic):
    """jorldy/core/agent/sac.py:16-355, continuous actions (`actor="continuous_policy"`); `actor="discrete_policy"`
    constructs the discrete-action SAC (SACDiscrete below)."""
    _n_critics = 2
    _actor_kind = "continuous"
    _strict_gate = True

    def __new__(cls, *args, **kwargs):
        actor = kwargs.get("actor", args[3] if len(args) > 3 else "continuous_policy")
        if cls is SAC and actor.split("_")[0] == "discrete":
            cls = SACDiscrete
        return super().__new__(cls)

    def __init__(self, state_size, action_size, hidden_size=512, actor="continuous_policy", critic="continuous_q_network",
                 head="mlp", optim_config=dict(_DEFAULT_OPTIM, alpha="adam", alpha_lr=3e-4), use_dynamic_alpha=False,
                 gamma=0.99, tau=5e-3, buffer_size=50000, batch_size=64, start_train_step=2000, static_log_alpha=-2.0,
                 target_update_period=10000, run_step=1e6, lr_decay=True, device=None, seed=0, use_cuda_graph=True, **kwargs):
        # target_update_period is accepted because the reference's configs pass it; the targets follow the soft update
        if actor.split("_")[0] != self._actor_kind:
            raise NotImplementedError(f"actor '{actor}': SAC is built with continuous_policy and discrete_policy actors")
        self._common(state_size, action_size, hidden_size, actor, critic, head, optim_config, gamma, buffer_size, batch_size,
                     start_train_step, tau, run_step, lr_decay, device, seed, target_actor=False, use_cuda_graph=use_cuda_graph)
        self.use_dynamic_alpha = use_dynamic_alpha
        self.log_alpha = _Scalar("log_alpha", 0.0 if use_dynamic_alpha else float(np.float32(static_log_alpha)), self.device)
        self.alpha_optimizer = (Optimizer(optim_config["alpha"], params=self.log_alpha.parameters(), lr=optim_config["alpha_lr"])
                                if use_dynamic_alpha else None)
        self.alpha = self.log_alpha.flat[:1].exp()       # device scalar; refreshed inside learn() like sac.py:241
        self.target_entropy = -float(action_size)

    def act_device(self, state, training=True, noise=None):
        """sac.py:139-142: a = tanh(Normal(mu, std).sample()) when training, tanh(mu) otherwise."""
        M, A = state.shape[0], self.action_size
        raw = self.actor._buf("act.raw", (M, 2 * A))
        self.actor.forward_rows(state, raw)
        row_ctr = self._row_counter(M)
        action = self.actor._buf("act.a", (M, A))
        C.jb_ppo_act_continuous(ptr(raw), M, A, 2 * A, ptr(noise), self.seed, self.rng_stream_base, 0, ptr(row_ctr),
                                0 if training else 1, ptr(action), stream_ptr())
        return action, None

    def _sample_action(self, raw, eps, key, B):
        A = self.action_size
        action, logp = self.actor._buf(key + "a", (B, A)), self.actor._buf(key + "logp", (B,))
        C.jb_sac_sample(ptr(raw), 2 * A, ptr(eps), B, A, ptr(action), ptr(logp), stream_ptr())
        return action, logp

    def _all_optimizers(self):
        return self._optimizers() + ([self.alpha_optimizer] if self.use_dynamic_alpha else [])

    def _learn_core(self, batch):
        B, s, a, r, d, ns = self._unpack(batch)
        A, st, sp = self.action_size, self._stats, stream_ptr()
        inj = self._inject_noise or {}
        eps_n = inj.get("next") if inj.get("next") is not None else self._fill("n.eps", (B, A), 2)
        eps_a = inj.get("actor") if inj.get("actor") is not None else self._fill("t.eps", (B, A), 3)
        c1, c2 = self.critics
        q1, q2 = c1.forward(s, a, tag="t."), c2.forward(s, a, tag="t.")
        na, nlogp = self._sample_action(self.actor.forward_raw(ns, tag="n.", save=False), eps_n, "n.", B)
        nq1 = self.target_critics[0].forward(ns, na, tag="n.")
        nq2 = self.target_critics[1].forward(ns, na, tag="n.")
        dq1, dq2 = c1._buf("t.dq", (B, 1)), c2._buf("t.dq", (B, 1))
        C.jb_ac_critic_loss(ptr(q1), ptr(q2), ptr(nq1), ptr(nq2), ptr(self.alpha), ptr(nlogp), ptr(r), ptr(d), B, self.gamma,
                            ptr(dq1), ptr(dq2), ptr(st), sp)
        self._critic_step(0, dq1, B)
        self._critic_step(1, dq2, B)
        # actor: L = mean(alpha * logp - min(q1, q2)) through the updated critics (sac.py:222-236)
        raw = self.actor.forward_raw(s, tag="t.")
        ap, logp = self._sample_action(raw, eps_a, "t.", B)
        qa1, qa2 = c1.forward(s, ap, tag="a."), c2.forward(s, ap, tag="a.")
        dqa1, dqa2 = c1._buf("a.dq", (B, 1)), c2._buf("a.dq", (B, 1))
        C.jb_sac_minq(ptr(qa1), ptr(qa2), ptr(logp), ptr(self.alpha), self.target_entropy, B, ptr(dqa1), ptr(dqa2),
                      st.data_ptr() + 16, sp)
        da = c1.backward(dqa1, B, tag="a.", params=False, want_dx2=True)
        c2.backward(dqa2, B, tag="a.", params=False, want_dx2=True, dx2=da, accumulate=True)
        dout = self.actor._buf("t.dout", (B, 2 * A))
        C.jb_sac_actor_bwd(ptr(raw), 2 * A, ptr(eps_a), ptr(ap), ptr(da), ptr(self.alpha), B, A, ptr(dout), sp)
        self.actor.backward_raw(dout, B, tag="t.")
        self.actor_optimizer.step()
        # alpha: alpha_loss = log_alpha * mean(entropy - target_entropy); self.alpha = exp(log_alpha) BEFORE the step
        C.jb_sac_alpha(ptr(self.log_alpha.flat), st.data_ptr() + 16, ptr(self.alpha), ptr(self.log_alpha.grad),
                       st.data_ptr() + 32, sp)
        if self.use_dynamic_alpha:
            self.alpha_optimizer.step()

    def _finish(self):
        self.num_learn += 1
        h = torch.cat([self._stats[:9], self.alpha]).cpu().numpy()
        return {"critic_loss1": float(h[0]), "critic_loss2": float(h[1]), "actor_loss": float(h[4]), "alpha_loss": float(h[8]),
                "max_Q": float(h[2]), "mean_Q": float(h[5]), "alpha": float(h[9]), "entropy": float(h[6])}

    def _ckpt(self):
        d = super()._ckpt()
        if self.use_dynamic_alpha:
            d["log_alpha"] = self.log_alpha.flat[:1].detach().cpu().clone()
            d["alpha_optimizer"] = cpu_optimizer_state(self.alpha_optimizer)
        return d

    def load(self, path):
        print(f"...Load model from {path}...")
        ck = torch.load(os.path.join(path, "ckpt"), map_location="cpu", weights_only=False)
        self._load_common(ck)
        if self.use_dynamic_alpha and "log_alpha" in ck:
            self.log_alpha.flat[:1].copy_(torch.as_tensor(ck["log_alpha"]).detach().reshape(1).to(self.device))
            self.alpha_optimizer.load_state_dict(ck["alpha_optimizer"])


class SACDiscrete(SAC):
    """SAC with a categorical policy (`actor="discrete_policy"`, `critic="discrete_q_network"`): SAC-Discrete
    (Christodoulou 2019, arXiv:1910.07207) with the continuous SAC's bookkeeping: soft target update on every process()
    once learning has started, alpha from before the previous learn's log_alpha step, the checkpoint layout and its
    critic2 -> critic1 load.  The policy's expectations over the A actions are exact, so a learn() draws no noise:

        target   V' = sum_a pi'(a) [min(Q1', Q2')(s', a) - alpha logpi'(a)],  y = r + (1 - d) gamma V'
        critics  L_i = mean (Q_i(s)[a] - y)^2
        actor    L = mean_b sum_a pi(a) [alpha logpi(a) - min(Q1, Q2)(s, a)], through the updated critics
        alpha    alpha_loss = log_alpha * mean(H - target_entropy), H = -sum_a pi logpi, target_entropy = 0.98 ln A

    Actions are int64 [N, 1]; with the cnn head, states stay uint8 stacks (the head scales by 1/255)."""
    action_type = "discrete"
    _actor_kind = "discrete"

    def __init__(self, *args, **kwargs):
        if len(args) < 4:
            kwargs.setdefault("actor", "discrete_policy")
        if len(args) < 5:
            kwargs.setdefault("critic", "discrete_q_network")
        super().__init__(*args, **kwargs)
        self.target_entropy = 0.98 * float(np.log(self.action_size))

    def _net_input(self, s):
        return s if s.dtype == torch.uint8 else s.to(torch.float32).reshape(s.shape[0], -1)

    def _unpack(self, batch):
        B = batch["reward"].shape[0]
        f = lambda k: batch[k].to(torch.float32).reshape(B).contiguous()
        a = batch["action"].reshape(B).to(torch.int64).contiguous()
        return B, self._net_input(batch["state"]), a, f("reward"), f("done"), self._net_input(batch["next_state"])

    def act_device(self, state, training=True, noise=None):
        """a ~ Categorical(softmax(actor(s))) when training, argmax otherwise; noise: optional f32 [N] uniforms in [0, 1)."""
        M, A = state.shape[0], self.action_size
        logits = self.actor._buf("act.z", (M, A))
        self.actor.forward_rows(state, logits)
        row_ctr = self._row_counter(M)
        action = self.actor._buf("act.a", (M, 1), torch.int64)
        C.jb_sacd_act(ptr(logits), M, A, ptr(noise), self.seed, self.rng_stream_base, ptr(row_ctr),
                      0 if training else 1, ptr(action), stream_ptr())
        return action, None

    def _learn_core(self, batch):
        B, s, a, r, d, ns = self._unpack(batch)
        A, st, sp = self.action_size, self._stats, stream_ptr()
        c1, c2 = self.critics
        q1, q2 = c1.forward(s, tag="t."), c2.forward(s, tag="t.")
        nz = self.actor.forward_raw(ns, tag="n.", save=False)
        nq1 = self.target_critics[0].forward(ns, tag="n.", save=False)
        nq2 = self.target_critics[1].forward(ns, tag="n.", save=False)
        dq1, dq2 = c1._buf("t.dq", (B, A)), c2._buf("t.dq", (B, A))
        C.jb_sacd_critic_loss(ptr(q1), ptr(q2), ptr(nq1), ptr(nq2), ptr(nz), ptr(a), ptr(r), ptr(d), ptr(self.alpha), B, A,
                              self.gamma, ptr(dq1), ptr(dq2), ptr(st), sp)
        self._critic_step(0, dq1, B)
        self._critic_step(1, dq2, B)
        z = self.actor.forward_raw(s, tag="t.")
        qa1, qa2 = c1.forward(s, tag="a.", save=False), c2.forward(s, tag="a.", save=False)
        dz = self.actor._buf("t.dz", (B, A))
        C.jb_sacd_actor(ptr(z), ptr(qa1), ptr(qa2), ptr(self.alpha), self.target_entropy, B, A, ptr(dz), st.data_ptr() + 16, sp)
        self.actor.backward_raw(dz, B, tag="t.")
        self.actor_optimizer.step()
        C.jb_sac_alpha(ptr(self.log_alpha.flat), st.data_ptr() + 16, ptr(self.alpha), ptr(self.log_alpha.grad),
                       st.data_ptr() + 32, sp)
        if self.use_dynamic_alpha:
            self.alpha_optimizer.step()

    def _finish(self):
        result = super()._finish()
        self.memory.check_frames()
        return result
