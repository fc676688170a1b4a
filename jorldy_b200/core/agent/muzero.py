"""MuZero (Schrittwieser, Antonoglou, Hubert et al., arXiv:1911.08265) on flat observations or Atari frames, with
discrete actions.

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

Atari frames (head="cnn", state_size [4, 84, 84]), under the batched collector only: attach_frames() gives the agent a
single-frame store (buffer/frame_store.py) sized by frames_per_window, and a per-lane history of the last 4 actions.
h's input is the lane's newest stack plus 4 action planes (csrc/frame_ring.cu jb_im2col_u8_frames_actions, read
straight from the ring).  An act roots the search at each lane's newest stack (reference (lane << 40) | (head - 1))
with the history as it was before the act (step_inputs["prev_actions"]), then shifts the action into the history, all
inside the act graph.  A window keeps its first step's frame reference under `state` and that step's prev_actions; a
learn runs h through the same im2col over the B sampled windows and the trunk's backward after h's.

Board games (env.legal, e.g. TicTacToe): attach_legal(legal u8 [N, A]) masks the search root, as in the paper: the
root priors and noise cover the legal moves only and an illegal move is never selected at the root
(jb_mcts_root_legal / jb_mcts_select_legal); the act graph reads the mask in place.  Below the root every action stays
allowed.  Without a mask the search is unchanged.

Two-player zero-sum games (two_player=True, e.g. TicTacToe with opponent="self"): a step's reward and its stored search
value are the mover's, and the players alternate every step.  The negamax backup, where each ply's value is negated
to the parent's side, is then exactly the single-player backup with the discount negated, so the search and the loss
run the unchanged kernels at -gamma:
  - backup: q = r - gamma W / N, g <- r - gamma g (the pseudocode flips W to the parent's side at each ply instead);
  - root value (jb_mcts_act): sum(N r - gamma W) / sum N, the value for the side to move;
  - n-step value target (jb_muzero_loss): z = r_k - gamma r_{k+1} + ... + (-gamma)^n v_{k+n}, cut at the first done.
The reward and policy targets and the priorities do not change, nor do windows, replay, checkpoints or the masked root.
"""
import numpy as np
import torch

from ..buffer import PERBuffer, frame_store
from ..buffer.frame_store import STACK, FrameActionRows
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
                 seed=0, use_cuda_graph=True, two_player=False, **kwargs):
        frames = head == "cnn"
        if frames:
            shape = tuple(int(d) for d in np.atleast_1d(state_size))
            if len(shape) != 3:
                raise NotImplementedError(f"state_size {list(shape)}: MuZero's CNN representation takes frame stacks")
            if shape[1:] != (84, 84) or shape[0] != STACK:
                raise ValueError(f"state_size {list(shape)}: MuZero's CNN representation takes [{STACK}, 84, 84] frame "
                                 f"stacks (stack_frame {STACK})")
        elif head != "mlp" or not isinstance(state_size, (int, np.integer)):
            raise NotImplementedError("MuZero takes flat observations with head='mlp', or frame stacks with head='cnn'")
        if action_type != "discrete":
            raise ValueError("MuZero plans over discrete actions only")
        if not 1 <= int(action_size) <= MAX_ACTION_SIZE["discrete"]:
            raise ValueError(f"action_size {action_size}: MuZero takes at most {MAX_ACTION_SIZE['discrete']} actions")
        for name, v in (("num_unroll", num_unroll), ("td_steps", td_steps), ("num_simulation", num_simulation)):
            if int(v) < 1:
                raise ValueError(f"{name} {v}: must be at least 1")
        self.device = require_cuda(device)
        self.frames_input = frames
        self.state_size = shape if frames else int(state_size)
        self.action_size, self.seed = int(action_size), int(seed)
        self.gamma, self.S, self.K, self.n_step = float(gamma), int(num_simulation), int(num_unroll), int(td_steps)
        self.two_player = bool(two_player)
        self._discount = -self.gamma if self.two_player else self.gamma    # the search and loss kernels' gamma
        self.V, self.R, self.value_loss_coef = int(value_support), int(reward_support), float(value_loss_coef)
        self.alpha, self.beta, self.clip_grad_norm = float(alpha), float(beta), clip_grad_norm
        self.dir_alpha, self.dir_frac = float(root_dirichlet_alpha), float(root_exploration_fraction)
        self.temperature_learns = tuple(temperature_learns)
        self.batch_size, self.buffer_size, self.start_train_step = int(batch_size), int(buffer_size), start_train_step
        self.run_step, self.lr_decay, self.num_workers = run_step, lr_decay, num_workers
        self.use_cuda_graph = use_cuda_graph
        self.network = MuZeroNetwork(self.state_size, self.action_size, hidden_size, latent_size, self.V, self.R,
                                     head=head, device=self.device, seed=self.seed)
        self.optimizer = Optimizer(**dict(optim_config), params=self.network.parameters())
        self.memory = PERBuffer(self.buffer_size, uniform_sample_prob, device=self.device, seed=self.seed)
        self.L = self.K + self.n_step + 1
        self.sequence_assembler = SequenceAssembler(0, self.K + 1, self.n_step, fields=WINDOW_FIELDS, period=1,
                                                    snapshot=("state", "prev_actions") if frames else ("state",))
        self._frames = self._hist = None      # frames: the store and the lanes' last STACK actions (attach_frames)
        self._legal = None                    # board games: the env's legal moves u8 [N, A] (attach_legal)
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
        if self.frames_input:
            return s
        return s.to(torch.float32).reshape(s.shape[0], -1)

    def _search_state(self, M):
        st = self._search.get(M)
        if st is None:
            A, S, H, Hs = self.action_size, self.S, self.network.D_hidden, self.network.Hs
            f = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=self.device)
            i = lambda *shape: torch.zeros(*shape, dtype=torch.int32, device=self.device)
            i64 = lambda *shape: torch.zeros(*shape, dtype=torch.int64, device=self.device)
            if self.frames_input:
                x = {"refs": i64(M), "prev_actions": i64(M, STACK),
                     "lane_bits": torch.arange(M, dtype=torch.int64, device=self.device) << frame_store.POS_BITS}
            else:
                x = {"x": f(M, self.state_size)}
            st = self._search[M] = dict(x, **{
                "h1": f(M, self.network.D_repr), "pre": f(M, Hs), "s": f(M, Hs), "hid": f(M, H),
                "pi": f(M, A), "v": f(M, 2 * self.V + 1), "r": f(M, 2 * self.R + 1), "z": f(M, Hs + A),
                "n": i(M, S + 1, A), "w": f(M, S + 1, A), "p": f(M, S + 1, A), "er": f(M, S + 1, A),
                "child": i(M, S + 1, A), "latent": f(M, S + 1, Hs), "count": i(M), "bounds": f(M, 2),
                "path": i(M, S + 1), "path_len": i(M), "leaf_node": i(M), "leaf_action": i(M),
                "action": torch.zeros(M, dtype=torch.int64, device=self.device), "policy": f(M, A),
                "root_value": f(M), "v0": f(M)})
        return st

    def _tree(self, st):
        return [ptr(st[k]) for k in ("n", "w", "p", "er", "child", "latent", "count", "bounds", "path", "path_len")]

    def _search_eager(self, M, training):
        st, net, s_ = self._search_state(M), self.network, stream_ptr()
        A, S, Hs, V, R, g = self.action_size, self.S, net.Hs, self.V, self.R, self._discount
        ctr = self._row_counter(M)
        tree = self._tree(st)
        if self.frames_input:       # the roots: each lane's newest stack and its last STACK actions
            torch.add(st["lane_bits"], self._frames.head, out=st["refs"]).sub_(1)
            st["prev_actions"].copy_(self._hist)
            x = FrameActionRows(self._frames, st["refs"], st["prev_actions"], A)
        else:
            x = st["x"]
        net.represent(x, st["h1"], st["pre"], st["s"], tag="a.")
        net.predict(st["s"], st["hid"], st["pi"], st["v"])
        root_args = (ptr(st["pi"]), ptr(st["v"]), ptr(st["s"]), M, A, S, Hs, V, int(training), self.dir_alpha,
                     self.dir_frac, ptr(self._inject_gamma), self.seed, ptr(ctr), *tree, ptr(st["v0"]))
        select_args = (M, A, S, Hs, g, *tree, ptr(st["leaf_node"]), ptr(st["leaf_action"]), ptr(st["z"]))
        if self._legal is None:
            C.jb_mcts_root(*root_args, s_)
        else:
            C.jb_mcts_root_legal(*root_args, ptr(self._legal), s_)
        for _ in range(S):
            if self._legal is None:
                C.jb_mcts_select(*select_args, s_)
            else:
                C.jb_mcts_select_legal(*select_args, ptr(self._legal), s_)
            net.dynamics(st["z"], st["hid"], st["pre"], st["s"], st["r"])
            net.predict(st["s"], st["hid"], st["pi"], st["v"])
            C.jb_mcts_expand_backup(ptr(st["s"]), ptr(st["pi"]), ptr(st["v"]), ptr(st["r"]), M, A, S, Hs, V, R, g,
                                    ptr(st["leaf_node"]), ptr(st["leaf_action"]), *tree, s_)
        C.jb_mcts_act(M, A, S, g, int(training), ptr(self._temp), ptr(self._inject_u), self.seed + 1, ptr(ctr),
                      ptr(st["n"]), ptr(st["w"]), ptr(st["er"]), ptr(st["action"]), ptr(st["policy"]),
                      ptr(st["root_value"]), s_)
        if self.frames_input:
            self._hist[:, :-1].copy_(st["prev_actions"][:, 1:])
            self._hist[:, -1].copy_(st["action"])

    def act_device(self, state, training=True):
        """state [N, D] device tensor -> (action int64 [N], search value f32 [N]); sets step_inputs.  On frames, state
        is the collector's [N, 4, 84, 84] stacks, whose newest frames the attached store already holds: the roots are
        read from the store."""
        M = state.shape[0]
        st = self._search_state(M)
        if self.frames_input:
            if self._frames is None or M != self._frames.n:
                raise RuntimeError("MuZero on frames acts on the lanes of the frame store that attach_frames() made: "
                                   "run it under the batched collector (main --sync)")
        else:
            st["x"].copy_(state.reshape(M, -1))
        if self._legal is not None and M != self._legal.shape[0]:
            raise RuntimeError(f"MuZero acts on {M} rows but the attached legal-move mask has {self._legal.shape[0]}")
        t = self.temperature()
        if t != self._temp_host:
            self._temp.fill_(t)
            self._temp_host = t
        injected = self._inject_gamma is not None or self._inject_u is not None
        if self.use_cuda_graph and not injected:
            key = (M, bool(training))
            graph = self._graphs.get(key)
            if graph is None:
                restore = [self._row_counter(M)] + ([self._hist] if self.frames_input else [])
                graph = self._graphs[key] = capture_after_warmup(lambda: self._search_eager(M, training),
                                                                 restore=restore)
            graph.replay()
        else:
            self._search_eager(M, training)
        self.step_inputs = {"root_value": st["root_value"], "policy": st["policy"]}
        if self.frames_input:
            self.step_inputs["prev_actions"] = st["prev_actions"]
        return st["action"], st["root_value"]

    @torch.no_grad()
    def act(self, state, training=True):
        if self.frames_input:
            raise NotImplementedError("MuZero on frames runs under the batched collector (main --sync) only")
        s = self._net_input(self._state_to_device(state))
        action, _ = self.act_device(s, training)
        return {"action": action.cpu().numpy().reshape(-1, 1)}

    def end_step(self, done):
        """The search keeps no state across steps."""

    def attach_frames(self, env):
        """Frames: a single-frame store for `env`'s lanes, sized so that every frame a live window references stays
        resident (frame_store.frames_per_window), and a zeroed action history per lane.  None on flat observations."""
        stack = bool(getattr(env, "frame_stack", False))
        if stack != self.frames_input:
            raise ValueError("MuZero with head='cnn' needs a frame-stack env, and a frame-stack env needs head='cnn'")
        if not stack:
            return None
        F = frame_store.frames_per_window(self.buffer_size, env.num_envs, self.L)
        self._frames = frame_store.FrameStore(env.num_envs, F, self.device)
        self._hist = torch.zeros(env.num_envs, STACK, dtype=torch.int64, device=self.device)
        return self._frames

    def attach_legal(self, legal):
        """Board games: `legal` u8 [N, A] (the env's, updated in place) masks the root of every later search.  The act
        graphs captured before are dropped, so the next act captures one that reads this mask."""
        if legal.dtype != torch.uint8 or legal.dim() != 2 or legal.shape[1] != self.action_size or not legal.is_cuda \
                or not legal.is_contiguous():
            raise ValueError(f"legal {tuple(legal.shape)} {legal.dtype}: MuZero takes a u8 [N, {self.action_size}] "
                             "device mask")
        self._legal = legal
        self._graphs.clear()

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
        ws = {"x": x, "h1": b("h1", B, net.D_repr), "pre": b("pre", (K + 1) * B, Hs), "s": b("s", (K + 1) * B, Hs),
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
        net.represent_bwd(ws["x"], ws["h1"], rows(dpre, 0), b("dh1", B, net.D_repr))

    def _learn_windows(self, batch, weights):
        """One unroll -> loss -> backward -> Adam on B windows; returns the priorities f64 [B]."""
        net, K, A, B = self.network, self.K, self.action_size, batch["reward"].shape[0]
        if self.frames_input:
            if self._frames is None:
                raise RuntimeError("these windows hold frame references but no frame store is attached")
            x = FrameActionRows(self._frames, batch["state"].contiguous(), batch["prev_actions"].contiguous(),
                                self.action_size)
        else:
            x = self._net_input(batch["state"]).contiguous()
        ws = self._unroll(x, batch["action"], B)
        w32 = {k: batch[k].to(torch.float32).contiguous() for k in ("reward", "done", "root_value", "policy")}
        d_pi, d_v, d_r = (net._buf("t.d" + k, tuple(ws[k].shape)) for k in ("pi", "v", "r"))
        prio = net._buf("t.prio", (B,), torch.float64)
        scratch = net._buf("t.lossscratch", (3 * B * (K + 1),), torch.float64)
        stats = net._buf("t.lossstats", (4,))
        C.jb_muzero_loss(ptr(ws["pi"]), ptr(ws["v"]), ptr(ws["r"]), ptr(w32["reward"]), ptr(w32["done"]),
                         ptr(w32["root_value"]), ptr(w32["policy"]), ptr(weights), B, K, self.n_step, A, self.V, self.R,
                         self._discount, self.value_loss_coef, self.alpha, ptr(d_pi), ptr(d_v), ptr(d_r), ptr(prio),
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
        if self._frames is not None:
            self._frames.check()
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
