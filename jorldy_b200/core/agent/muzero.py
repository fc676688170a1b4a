"""MuZero (Schrittwieser, Antonoglou, Hubert et al., arXiv:1911.08265) on flat observations and discrete actions.

act_device(state, training) for N envs, one tree per env (csrc/muzero.cu):
  1. initial inference: h over the N observations, then f over the root latents;
  2. jb_mcts_root: softmax priors (training: Dirichlet(0.25) noise at fraction 0.25), the tree reset;
  3. S simulations, each jb_mcts_select -> g -> f over the N leaf rows -> jb_mcts_expand_backup;
  4. jb_mcts_act: the root visit distribution, the search value and the action (training: sampled from N(a)^(1/T) with
     the visit temperature 1, 0.5, 0.25 after the temperature_learns thresholds of num_learn; eval: argmax N).
One CUDA graph per (row count, training) runs all of it (dev.capture_after_warmup); use_cuda_graph=False runs the same
launches eagerly, bit-identical.  step_inputs = {root_value, policy} is stored with the step.

Replay items are windows of L = K + n + 1 steps, one per env per step (SequenceAssembler with period 1), holding the first
step's observation and every step's action, reward, done, search value and visit distribution.  New windows enter the
PERBuffer at its max priority.  One learn():
  1. PERBuffer.sample_device: B windows, IS weights (f64), tree indices;
  2. h over the first observations, K dynamics steps with the stored actions, f over the K + 1 latents at once;
  3. jb_muzero_loss: n-step value targets from the stored search values, reward and policy targets, cross-entropies, the
     logit gradients and the priorities |v_0 - z_0|^alpha;
  4. the backward in reverse order, with the gradient into each dynamics step's latent input scaled by 0.5;
  5. Adam with clip_grad_norm, then update_priorities; one device->host read of the results.
"""
import numpy as np
import torch

from ..buffer import PERBuffer
from ..collect import SequenceAssembler
from ..dev import C, capture_after_warmup, ptr, require_cuda, stream_ptr
from ..network.muzero import MuZero as MuZeroNetwork
from ..optimizer import Optimizer
from .base import BaseAgent
from .ppo import MAX_ACTION_SIZE

WINDOW_FIELDS = ("action", "reward", "done", "root_value", "policy")
TEMPERATURES = (1.0, 0.5, 0.25)


class MuZero(BaseAgent):
    action_type = "discrete"
    replicas_only = True
    FAMILY = "MuZero"

    def __init__(self, state_size, action_size, hidden_size=128, latent_size=64, optim_config={"name": "adam"},
                 head="mlp", action_type="discrete", gamma=0.997, num_simulation=50, num_unroll=5, td_steps=10,
                 value_support=20, reward_support=1, value_loss_coef=0.25, alpha=1.0, beta=1.0,
                 uniform_sample_prob=1e-3, buffer_size=100000, batch_size=128, start_train_step=2000,
                 clip_grad_norm=5.0, root_dirichlet_alpha=0.25, root_exploration_fraction=0.25,
                 temperature_learns=(500000, 750000), run_step=1e6, lr_decay=True, num_workers=1, device=None,
                 seed=0, use_cuda_graph=True, **kwargs):
        if head != "mlp" or not isinstance(state_size, (int, np.integer)):
            raise NotImplementedError("MuZero runs on flat observations only: the CNN representation is not implemented")
        if action_type != "discrete":
            raise ValueError("MuZero plans over discrete actions only")
        if not 1 <= int(action_size) <= MAX_ACTION_SIZE["discrete"]:
            raise ValueError(f"action_size {action_size}: MuZero takes at most {MAX_ACTION_SIZE['discrete']} actions")
        for name, v in (("num_unroll", num_unroll), ("td_steps", td_steps), ("num_simulation", num_simulation)):
            if int(v) < 1:
                raise ValueError(f"{name} {v}: must be at least 1")
        self.device = require_cuda(device)
        self.state_size, self.action_size, self.seed = int(state_size), int(action_size), int(seed)
        self.gamma, self.S, self.K, self.n_step = float(gamma), int(num_simulation), int(num_unroll), int(td_steps)
        self.V, self.R, self.value_loss_coef = int(value_support), int(reward_support), float(value_loss_coef)
        self.alpha, self.beta, self.clip_grad_norm = float(alpha), float(beta), clip_grad_norm
        self.dir_alpha, self.dir_frac = float(root_dirichlet_alpha), float(root_exploration_fraction)
        self.temperature_learns = tuple(temperature_learns)
        self.batch_size, self.buffer_size, self.start_train_step = int(batch_size), int(buffer_size), start_train_step
        self.run_step, self.lr_decay, self.num_workers = run_step, lr_decay, num_workers
        self.use_cuda_graph = use_cuda_graph
        self.network = MuZeroNetwork(self.state_size, self.action_size, hidden_size, latent_size, self.V, self.R,
                                     device=self.device, seed=self.seed)
        self.optimizer = Optimizer(**dict(optim_config), params=self.network.parameters())
        self.memory = PERBuffer(self.buffer_size, uniform_sample_prob, device=self.device, seed=self.seed)
        self.L = self.K + self.n_step + 1
        self.sequence_assembler = SequenceAssembler(0, self.K + 1, self.n_step, fields=WINDOW_FIELDS, period=1,
                                                    snapshot=("state",))
        self.num_learn, self.time_t = 0, 0
        self.step_inputs = None
        self.world_size, self.allreduce = 1, None
        self._row_ctr = {}
        self._search, self._graphs = {}, {}
        self._temp = torch.ones(1, dtype=torch.float32, device=self.device)     # read by the act graphs
        self._temp_host = 1.0
        self._stats = torch.zeros(8, dtype=torch.float64, device=self.device)
        self._inject_gamma = self._inject_u = None     # tests: f64 [N, A] gamma draws / f64 [N] action uniforms
        self._inject_per_u = None                      # tests: (u_a, u_b) PER uniforms of the next learn

    # -------------------------------------------------------------------------------------- act --
    def temperature(self):
        k = sum(self.num_learn >= t for t in self.temperature_learns)
        return TEMPERATURES[min(k, len(TEMPERATURES) - 1)]

    def _net_input(self, s):
        return s.to(torch.float32).reshape(s.shape[0], -1)

    def _search_state(self, M):
        st = self._search.get(M)
        if st is None:
            A, S, H, Hs = self.action_size, self.S, self.network.D_hidden, self.network.Hs
            f = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=self.device)
            i = lambda *shape: torch.zeros(*shape, dtype=torch.int32, device=self.device)
            st = self._search[M] = {
                "x": f(M, self.state_size), "h1": f(M, H), "pre": f(M, Hs), "s": f(M, Hs), "hid": f(M, H),
                "pi": f(M, A), "v": f(M, 2 * self.V + 1), "r": f(M, 2 * self.R + 1), "z": f(M, Hs + A),
                "n": i(M, S + 1, A), "w": f(M, S + 1, A), "p": f(M, S + 1, A), "er": f(M, S + 1, A),
                "child": i(M, S + 1, A), "latent": f(M, S + 1, Hs), "count": i(M), "bounds": f(M, 2),
                "path": i(M, S + 1), "path_len": i(M), "leaf_node": i(M), "leaf_action": i(M),
                "action": torch.zeros(M, dtype=torch.int64, device=self.device), "policy": f(M, A),
                "root_value": f(M), "v0": f(M)}
        return st

    def _tree(self, st):
        return [ptr(st[k]) for k in ("n", "w", "p", "er", "child", "latent", "count", "bounds", "path", "path_len")]

    def _search_eager(self, M, training):
        st, net, s_ = self._search_state(M), self.network, stream_ptr()
        A, S, Hs, V, R, g = self.action_size, self.S, net.Hs, self.V, self.R, self.gamma
        ctr = self._row_counter(M)
        tree = self._tree(st)
        net.represent(st["x"], st["h1"], st["pre"], st["s"])
        net.predict(st["s"], st["hid"], st["pi"], st["v"])
        C.jb_mcts_root(ptr(st["pi"]), ptr(st["v"]), ptr(st["s"]), M, A, S, Hs, V, int(training), self.dir_alpha,
                       self.dir_frac, ptr(self._inject_gamma), self.seed, ptr(ctr), *tree, ptr(st["v0"]), s_)
        for _ in range(S):
            C.jb_mcts_select(M, A, S, Hs, g, *tree, ptr(st["leaf_node"]), ptr(st["leaf_action"]), ptr(st["z"]), s_)
            net.dynamics(st["z"], st["hid"], st["pre"], st["s"], st["r"])
            net.predict(st["s"], st["hid"], st["pi"], st["v"])
            C.jb_mcts_expand_backup(ptr(st["s"]), ptr(st["pi"]), ptr(st["v"]), ptr(st["r"]), M, A, S, Hs, V, R, g,
                                    ptr(st["leaf_node"]), ptr(st["leaf_action"]), *tree, s_)
        C.jb_mcts_act(M, A, S, g, int(training), ptr(self._temp), ptr(self._inject_u), self.seed + 1, ptr(ctr),
                      ptr(st["n"]), ptr(st["w"]), ptr(st["er"]), ptr(st["action"]), ptr(st["policy"]),
                      ptr(st["root_value"]), s_)

    def act_device(self, state, training=True):
        """state [N, D] device tensor -> (action int64 [N], search value f32 [N]); sets step_inputs."""
        M = state.shape[0]
        st = self._search_state(M)
        st["x"].copy_(state.reshape(M, -1))
        t = self.temperature()
        if t != self._temp_host:
            self._temp.fill_(t)
            self._temp_host = t
        injected = self._inject_gamma is not None or self._inject_u is not None
        if self.use_cuda_graph and not injected:
            key = (M, bool(training))
            graph = self._graphs.get(key)
            if graph is None:
                graph = self._graphs[key] = capture_after_warmup(lambda: self._search_eager(M, training),
                                                                 restore=[self._row_counter(M)])
            graph.replay()
        else:
            self._search_eager(M, training)
        self.step_inputs = {"root_value": st["root_value"], "policy": st["policy"]}
        return st["action"], st["root_value"]

    @torch.no_grad()
    def act(self, state, training=True):
        s = self._net_input(self._state_to_device(state))
        action, _ = self.act_device(s, training)
        return {"action": action.cpu().numpy().reshape(-1, 1)}

    def end_step(self, done):
        """The search keeps no state across steps."""

    def attach_frames(self, env):
        if getattr(env, "frame_stack", False):
            raise NotImplementedError("MuZero on frame-stack envs is not implemented")
        return None

    def interact_callback(self, transition):
        """Single-process driver: the step goes through the same window assembler with N = its rows."""
        dev = self.device
        tr = dict(self.step_inputs,
                  state=self._net_input(self._state_to_device(transition["state"])).clone(),
                  action=torch.as_tensor(np.asarray(transition["action"]).reshape(-1), dtype=torch.int64, device=dev),
                  reward=torch.as_tensor(np.asarray(transition["reward"], dtype=np.float32).reshape(-1), device=dev),
                  done=torch.as_tensor(np.asarray(transition["done"], dtype=np.float32).reshape(-1), device=dev))
        return self.sequence_assembler.push(tr) or {}

    # ------------------------------------------------------------------------------------ learn --
    def _unroll(self, x, action, B):
        """Forward of one learn: h, K dynamics steps, f over the K + 1 latents.  Returns the workspace dict."""
        net, K, A, H, Hs = self.network, self.K, self.action_size, self.network.D_hidden, self.network.Hs
        b = lambda name, *shape: net._buf("t." + name, shape)
        ws = {"x": x, "h1": b("h1", B, H), "pre": b("pre", (K + 1) * B, Hs), "s": b("s", (K + 1) * B, Hs),
              "z": b("z", K * B, Hs + A), "hidg": b("hidg", K * B, H), "r": b("r", K * B, 2 * self.R + 1),
              "hidf": b("hidf", (K + 1) * B, H), "pi": b("pi", (K + 1) * B, A), "v": b("v", (K + 1) * B, 2 * self.V + 1)}
        rows = lambda t, k: t[k * B:(k + 1) * B]
        net.represent(x, ws["h1"], rows(ws["pre"], 0), rows(ws["s"], 0), rows(ws["z"], 0)[:, :Hs])
        act32 = action.to(torch.int32).contiguous()
        idx = net._buf("t.rowidx", (B,), torch.int32)
        torch.mul(torch.arange(B, dtype=torch.int32, device=self.device), self.L, out=idx)
        for k in range(1, K + 1):
            z = rows(ws["z"], k - 1)
            C.jb_icm_action_rows(0, ptr(act32[:, k - 1]), ptr(idx), B, A, ptr(z[:, Hs:]), Hs + A, stream_ptr())
            nxt = rows(ws["z"], k)[:, :Hs] if k < K else None
            net.dynamics(z, rows(ws["hidg"], k - 1), rows(ws["pre"], k), rows(ws["s"], k), rows(ws["r"], k - 1), nxt)
        net.predict(ws["s"], ws["hidf"], ws["pi"], ws["v"])
        return ws

    def _backward(self, ws, d_pi, d_v, d_r, B):
        net, K, H, Hs, s_ = self.network, self.K, self.network.D_hidden, self.network.Hs, stream_ptr()
        b = lambda name, *shape: net._buf("t." + name, shape)
        rows = lambda t, k: t[k * B:(k + 1) * B]
        ds, dpre = b("ds", (K + 1) * B, Hs), b("dpre", (K + 1) * B, Hs)
        dhidg, ds_in = b("dhidg", K * B, H), b("ds_in", B, Hs)
        net.predict_bwd(ws["s"], ws["hidf"], d_pi, d_v, b("dhidf", (K + 1) * B, H), ds)
        for k in range(K, 0, -1):
            net.scale_bwd(rows(ws["pre"], k), rows(ds, k), rows(dpre, k))
            net.dynamics_bwd_step(rows(ws["hidg"], k - 1), rows(dpre, k), rows(d_r, k - 1), rows(dhidg, k - 1), ds_in)
            C.jb_scale_f32(ptr(ds_in), B * Hs, 0.5, s_)
            C.jb_add_f32(ptr(rows(ds, k - 1)), ptr(ds_in), B * Hs, s_)
        net.scale_bwd(rows(ws["pre"], 0), rows(ds, 0), rows(dpre, 0))
        net.dynamics_bwd_weights(ws["z"], ws["hidg"], dpre[B:], d_r, dhidg)
        net.represent_bwd(ws["x"], ws["h1"], rows(dpre, 0), b("dh1", B, H))

    def _learn_windows(self, batch, weights):
        """One unroll -> loss -> backward -> Adam on B windows; returns the priorities f64 [B]."""
        net, K, A, B = self.network, self.K, self.action_size, batch["reward"].shape[0]
        x = self._net_input(batch["state"]).contiguous()
        ws = self._unroll(x, batch["action"], B)
        w32 = {k: batch[k].to(torch.float32).contiguous() for k in ("reward", "done", "root_value", "policy")}
        d_pi, d_v, d_r = (net._buf("t.d" + k, tuple(ws[k].shape)) for k in ("pi", "v", "r"))
        prio = net._buf("t.prio", (B,), torch.float64)
        scratch = net._buf("t.lossscratch", (3 * B * (K + 1),), torch.float64)
        stats = net._buf("t.lossstats", (4,))
        C.jb_muzero_loss(ptr(ws["pi"]), ptr(ws["v"]), ptr(ws["r"]), ptr(w32["reward"]), ptr(w32["done"]),
                         ptr(w32["root_value"]), ptr(w32["policy"]), ptr(weights), B, K, self.n_step, A, self.V, self.R,
                         self.gamma, self.value_loss_coef, self.alpha, ptr(d_pi), ptr(d_v), ptr(d_r), ptr(prio),
                         ptr(stats), ptr(scratch), stream_ptr())
        self._backward(ws, d_pi, d_v, d_r, B)
        if self.allreduce is not None:
            self.allreduce(net.grad)
        self.optimizer.step(max_norm=self.clip_grad_norm)
        self.num_learn += 1
        self._stats[:4].copy_(stats)
        return prio

    def learn(self):
        u_a = u_b = None
        if self._inject_per_u is not None:
            u_a, u_b = (torch.as_tensor(np.asarray(u), dtype=torch.float64, device=self.device) for u in self._inject_per_u)
        batch, weights, indices, stats_per = self.memory.sample_device(self.beta, self.batch_size, u_a, u_b)
        prio = self._learn_windows(batch, weights)
        self.memory.update_priorities(indices, prio)
        self._stats[4:6].copy_(stats_per[:2])
        st = self._stats.cpu().numpy()
        return {"loss": float(st[0]), "value_loss": float(st[1]), "reward_loss": float(st[2]),
                "policy_loss": float(st[3]), "sampled_p": float(st[4]), "mean_p": float(st[5]),
                "num_learn": self.num_learn}

    def process(self, transitions, step):
        """Stores the windows at the tree's max priority; one learn per call once the replay holds a batch and step has
        reached start_train_step."""
        result = {}
        if transitions:
            self.memory.store(transitions)
        self.time_t = step
        if self.memory.size >= self.batch_size and self.time_t >= self.start_train_step:
            result = self.learn()
            if self.lr_decay:
                self.learning_rate_decay(step)
        return result
