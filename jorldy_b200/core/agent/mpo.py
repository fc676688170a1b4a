"""MPO agent (Abdolmaleki et al., arXiv:1806.06920) on the replay path, for discrete and continuous actions.

The replay holds n-step windows (collect.NStepAssembler's trajectory output): states s_0 .. s_n, and actions, rewards,
dones and the behaviour log mu_t = log pi_behaviour(a_t | s_t) taken at act time.  One learn() = one gradient step on
B = batch_size windows, as one CUDA-graph replay:

  1. target actor over the B (n+1) states; continuous: K = num_sample samples per state (jb_mpo_sample), so the target
     critic runs once over B (n+1) (K+1) rows (the K samples plus the taken action); discrete: all A values per state
  2. online critic over the B n steps -> jb_mpo_critic_target (Retrace, arXiv:1606.02647; "1step_TD": every c_t = 0)
     -> critic backward -> critic Adam
  3. actor over the B n states -> jb_mpo_policy_loss (E-step weights from the target actor and critic, L_eta, L_pi, the
     KL trust regions, arXiv:1812.02256 for the Gaussian split) -> actor backward -> actor Adam with clip_grad_norm on
     the actor only -> multiplier Adam -> jb_vmpo_clamp
  4. every target_update_period learns, a hard copy of both targets.

The multipliers [eta, alpha_mu, alpha_sigma] live in one device vector with their own flat Adam (same name, lr and
options as the actor's), which equals one torch Adam over actor.parameters() + the multipliers with clip_grad_norm_ on
the actor's parameters only; the checkpoint stores them in that layout, as V-MPO does.

Deviations from a literal restatement: log mu is stored, not a probability; the multipliers are clamped to their
minima after each step, not reparameterised; windows are not cut at episode ends (the (1 - d_t) masks carry the cut,
as for the other n-step agents).
"""
import os

import torch

from ..dev import C, ptr, stream_ptr
from ..optimizer import Optimizer
from .base import (_Scalar, cpu_optimizer_state, cpu_state_dict, joint_optimizer_state, load_joint_optimizer_state,
                   load_multipliers, multiplier_values)
from .ddpg import _ActorCritic
from .ppo import MAX_ACTION_SIZE

_PAIRS = {"discrete_policy": "discrete_q_network", "continuous_policy": "continuous_q_network"}
_CRITIC_LOSS = {"retrace": 1, "1step_TD": 0}
_SAMPLE_PURPOSE = 4          # Philox purpose id of the E-step normals (1: act, 2 / 3: the SAC / TD3 learn draws)


class MPO(_ActorCritic):
    FAMILY = "MPO"
    trajectory_windows = True     # ReplayCollector: store whole n-step windows with log mu
    _soft_in_process = False      # hard target copies inside learn()

    def __init__(self, state_size, action_size, hidden_size=512, actor="discrete_policy", critic="discrete_q_network",
                 head="mlp", optim_config={"name": "adam", "lr": 3e-4}, gamma=0.99, n_step=8, batch_size=64,
                 buffer_size=50000, start_train_step=2000, critic_loss_type="retrace", num_sample=30,
                 target_update_period=100, clip_grad_norm=1.0, min_eta=1e-8, min_alpha_mu=1e-8, min_alpha_sigma=1e-8,
                 eps_eta=0.01, eps_alpha_mu=0.01, eps_alpha_sigma=5e-5, eta=1.0, alpha_mu=1.0, alpha_sigma=1.0,
                 run_step=1e6, lr_decay=True, device=None, seed=0, use_cuda_graph=True, **kwargs):
        if head == "cnn":
            raise NotImplementedError("MPO is built for the mlp head; Atari frames in replayed windows are not implemented")
        if actor not in _PAIRS:
            raise ValueError(f"MPO actor '{actor}': use one of {list(_PAIRS)}")
        if critic != _PAIRS[actor]:
            raise ValueError(f"MPO actor '{actor}' takes the critic '{_PAIRS[actor]}', not '{critic}'")
        if critic_loss_type not in _CRITIC_LOSS:
            raise ValueError(f"critic_loss_type '{critic_loss_type}': use one of {list(_CRITIC_LOSS)}")
        if not 1 <= int(n_step) <= 32:
            raise ValueError(f"n_step {n_step}: MPO's windows take 1 <= n_step <= 32")
        self.action_type = actor.split("_")[0]
        self.continuous = self.action_type == "continuous"
        if self.continuous and not 1 <= int(num_sample) <= 64:
            raise ValueError(f"num_sample {num_sample}: continuous MPO takes 1 <= num_sample <= 64")
        if not isinstance(state_size, int):
            raise ValueError("MPO takes an integer state_size (mlp head)")
        if not 1 <= int(action_size) <= MAX_ACTION_SIZE[self.action_type]:
            raise ValueError(f"action_size {action_size}: {self.action_type} MPO takes at most "
                             f"{MAX_ACTION_SIZE[self.action_type]} actions")
        opt = dict(optim_config)
        name, lr = opt.pop("name"), opt.pop("lr")
        self._common(state_size, action_size, hidden_size, actor, critic, head,
                     {"actor": name, "critic": name, "actor_lr": lr, "critic_lr": lr}, gamma, buffer_size, batch_size,
                     start_train_step, 0.0, run_step, lr_decay, device, seed, target_actor=True,
                     use_cuda_graph=use_cuda_graph)
        if opt:                   # optimiser options besides the lr (betas, eps): the same for all three
            self.actor_optimizer = Optimizer(name, params=self.actor.parameters(), lr=lr, **opt)
            self.critic_optimizers = [Optimizer(name, params=self.critics[0].parameters(), lr=lr, **opt)]
        self.critic, self.target_critic = self.critics[0], self.target_critics[0]
        self.n_step, self.num_sample = int(n_step), int(num_sample)
        self.critic_loss_type, self._retrace = critic_loss_type, _CRITIC_LOSS[critic_loss_type]
        self.target_update_period, self.clip_grad_norm = int(target_update_period), clip_grad_norm
        self.min_eta, self.min_alpha_mu, self.min_alpha_sigma = float(min_eta), float(min_alpha_mu), float(min_alpha_sigma)
        self.eps_eta, self.eps_alpha_mu, self.eps_alpha_sigma = float(eps_eta), float(eps_alpha_mu), float(eps_alpha_sigma)
        self.mult = _Scalar("multipliers", [eta, alpha_mu, alpha_sigma], self.device)
        self.mult_optimizer = Optimizer(name, params=self.mult.parameters(), lr=lr, **opt)
        self._qret = None

    def _optimizers(self):
        return [self.actor_optimizer, self.critic_optimizers[0], self.mult_optimizer]

    # ---- act ---------------------------------------------------------------------------------------------------------
    def act_device(self, state, training=True, noise=None):
        """state [N, D] -> (action, log_mu [N]): discrete a ~ Categorical(softmax(logits)) (argmax when not training),
        int64 [N, 1]; continuous a = tanh(mu + sd eps) (tanh(mu) when not training), f32 [N, A].  log_mu is the
        log-probability of the returned action under the acting policy.  noise: optional uniforms [N] / normals [N, A]."""
        M, A = state.shape[0], self.action_size
        row_ctr = self._row_counter(M)
        logp = self.actor._buf("act.logp", (M,))
        if self.continuous:
            raw = self.actor._buf("act.raw", (M, 2 * A))
            self.actor.forward_rows(state, raw)
            action = self.actor._buf("act.a", (M, A))
            C.jb_ppo_act_continuous(ptr(raw), M, A, 2 * A, ptr(noise), self.seed, self.rng_stream_base, 0, ptr(row_ctr),
                                    0 if training else 1, ptr(action), stream_ptr())
            C.jb_mpo_logp(1, ptr(raw), 2 * A, ptr(action), M, A, ptr(logp), stream_ptr())
        else:
            raw = self.actor._buf("act.z", (M, A))
            self.actor.forward_rows(state, raw)
            action = self.actor._buf("act.a", (M, 1), torch.int64)
            C.jb_sacd_act(ptr(raw), M, A, ptr(noise), self.seed, self.rng_stream_base, ptr(row_ctr), 0 if training else 1,
                          ptr(action), stream_ptr())
            C.jb_mpo_logp(0, ptr(raw), A, ptr(action), M, A, ptr(logp), stream_ptr())
        return action, logp

    # ---- learn -------------------------------------------------------------------------------------------------------
    def _variant(self):
        """Whether this learn ends with the hard target copy."""
        return (self.num_learn + 1) % self.target_update_period == 0

    def _unpack(self, batch):
        B, n, A = batch["reward"].shape[0], self.n_step, self.action_size
        st = batch["state"].to(torch.float32).reshape(B, n + 1, -1)
        s_all = st.reshape(B * (n + 1), -1)
        s = st[:, :n].reshape(B * n, -1).contiguous()
        if self.continuous:
            a = batch["action"].to(torch.float32).reshape(B * n, A).contiguous()
        else:
            a = batch["action"].reshape(B * n).to(torch.int64).contiguous()
        f = lambda k: batch[k].to(torch.float32).reshape(B * n).contiguous()
        return B, s_all, s, a, f("reward"), f("done"), f("log_mu")

    def _learn_core(self, batch):
        B, s_all, s, a, r, d, log_mu = self._unpack(batch)
        n, A, K, sp = self.n_step, self.action_size, self.num_sample, stream_ptr()
        R, S, D = B * (n + 1), B * n, s_all.shape[1]
        actor, critic, tactor, tcritic = self.actor, self.critic, self.target_actor, self.target_critic
        tout = tactor.forward_raw(s_all, tag="n.", save=False)
        z = None
        if self.continuous:
            inj = self._inject_noise or {}
            eps = inj.get("sample") if inj.get("sample") is not None else self._fill("n.eps", (R, K, A), _SAMPLE_PURPOSE)
            z = tactor._buf("n.z", (R, K, A))
            xs, xa = tcritic._buf("n.xs", (R * (K + 1), D)), tcritic._buf("n.xa", (R * (K + 1), A))
            C.jb_mpo_sample(ptr(tout), ptr(eps), R, K, A, ptr(s_all), D, ptr(a), n, ptr(z), ptr(xs), ptr(xa), sp)
            tq = tcritic.forward(xs, xa, tag="n.")
            q = critic.forward(s, a, tag="t.")
            dq = critic._buf("t.dq", (S, 1))
        else:
            tq = tcritic.forward(s_all, tag="n.", save=False)
            q = critic.forward(s, tag="t.")
            dq = critic._buf("t.dq", (S, A))
        self._qret = critic._buf("t.qret", (S,))
        st = self._stats
        C.jb_mpo_critic_target(int(self.continuous), ptr(tq), ptr(tout), ptr(q), ptr(a), ptr(log_mu), ptr(r), ptr(d), B, n,
                               A, K, self.gamma, self._retrace, ptr(dq), ptr(self._qret), ptr(st), sp)
        critic.backward(dq, S, tag="t.")
        self.critic_optimizers[0].step()
        out = actor.forward_raw(s, tag="t.")
        dout = actor._buf("t.dout", (S, actor.nout))
        partials = actor._buf("t.partials", (C.jb_mpo_policy_partials(S),))
        C.jb_mpo_policy_loss(int(self.continuous), ptr(out), ptr(tout), ptr(tq), ptr(z), B, n, A, K, ptr(self.mult.flat),
                             self.eps_eta, self.eps_alpha_mu, self.eps_alpha_sigma, ptr(dout), ptr(self.mult.grad),
                             ptr(partials), st.data_ptr() + 8, sp)
        actor.backward_raw(dout, S, tag="t.")
        self.actor_optimizer.step(max_norm=self.clip_grad_norm)
        self.mult_optimizer.step()
        C.jb_vmpo_clamp(ptr(self.mult.flat), self.min_eta, self.min_alpha_mu, self.min_alpha_sigma, sp)
        if self._variant():
            tactor.copy_from(actor)
            tcritic.copy_from(critic)

    def _finish(self):
        self.num_learn += 1
        v = torch.cat([self._stats[:7], self.mult.flat[:3]]).cpu().numpy()      # ONE device->host read
        return {"actor_loss": float(v[2]), "critic_loss": float(v[0]), "eta_loss": float(v[3]), "alpha_loss": float(v[4]),
                "eta": float(v[7]), "alpha_mu": float(v[8]), "alpha_sigma": float(v[9]), "mean_Q": float(v[1])}

    # ---- checkpoint: actor, critic, one torch-Adam layout over actor + multipliers, critic_optimizer --------------------
    def _ckpt(self):
        d = {"actor": cpu_state_dict(self.actor), "critic": cpu_state_dict(self.critic),
             "actor_optimizer": joint_optimizer_state(self.actor_optimizer, self.mult_optimizer),
             "critic_optimizer": cpu_optimizer_state(self.critic_optimizers[0])}
        d.update(multiplier_values(self.mult))
        return d

    def load(self, path):
        print(f"...Load model from {path}...")
        ck = torch.load(os.path.join(path, "ckpt"), map_location="cpu", weights_only=False)
        self.actor.load_state_dict(ck["actor"])
        self.critic.load_state_dict(ck["critic"])
        self.target_actor.copy_from(self.actor)
        self.target_critic.copy_from(self.critic)
        load_joint_optimizer_state(ck["actor_optimizer"], self.actor_optimizer, self.mult_optimizer)
        self.critic_optimizers[0].load_state_dict(ck["critic_optimizer"])
        load_multipliers(ck, self.mult)
