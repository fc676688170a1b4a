"""R2D2's recurrent dueling Q-network (Kapturowski et al., ICLR 2019): head -> [feat, onehot(prev_action)] ->
LSTM(F + A -> H) -> Dueling's l1_a / l1_v / l2_a / l2_v streams -> Q = V + A - mean A.

Parameters, in state_dict order: `head.*`, then torch.nn.LSTM's `lstm.weight_ih_l0 [4H, F+A]`, `lstm.weight_hh_l0 [4H, H]`,
`lstm.bias_ih_l0`, `lstm.bias_hh_l0` (gate order i, f, g, o; drawn from U(-1/sqrt(H), 1/sqrt(H)) as torch does), then the
dueling tensors.  prev_action -1 (no previous action: an episode's first step) gives an all-zero one-hot.

Sequences are laid out TIME-MAJOR inside the network: row s*B + b is step s of sequence b, so one time step is a
contiguous [B, .] block and the trained steps of a window are one contiguous block of rows.
  encode()       the head over every row and ONE jb_linear_fwd for the input projection of all steps,
                 xg = [feat, onehot] W_ih^T + b_ih + b_hh; the rows [lo*B, hi*B) keep their activations for backward_tm()
  unroll()       one jb_lstm_step_fwd per step from (h0, c0); the first grad_from steps are the burn-in and save nothing,
                 the rest save their gates / cells and go through the dueling streams
  backward_tm()  dueling backward, one jb_lstm_step_bwd per trained step (latest first; nothing flows into the burn-in),
                 then dW_hh, dW_ih with both biases, and d feat each as ONE GEMM over the stacked trained rows, then the
                 head backward over those rows only
forward_seq / backward_seq are the batch-major form of the same ([B, S] inputs, [B, T, A] outputs); step() is one act()
step for N lanes.
"""
import math

import torch

from ..dev import C, ptr, stream_ptr
from .base import FlatNetwork, init_gain, orthogonal_
from .dueling import streams_bwd, streams_fwd
from .head import make_head


class R2D2(FlatNetwork):
    def __init__(self, D_in, D_out, D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        self.D_in, self.D_out, self.D_hidden = D_in, D_out, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        F, H, A = self.head.D_head_out, D_hidden, D_out
        self.F, self.Z = F, F + A
        self._specs = self.head.specs() + [
            ("lstm.weight_ih_l0", (4 * H, F + A)), ("lstm.weight_hh_l0", (4 * H, H)),
            ("lstm.bias_ih_l0", (4 * H,)), ("lstm.bias_hh_l0", (4 * H,)),
            ("l1_a.weight", (H, H)), ("l1_a.bias", (H,)), ("l1_v.weight", (H, H)), ("l1_v.bias", (H,)),
            ("l2_a.weight", (A, H)), ("l2_a.bias", (A,)), ("l2_v.weight", (1, H)), ("l2_v.bias", (1,))]
        self._allocate()
        self.nout = A
        self._acts = torch.arange(A, dtype=torch.int64, device=self.device)
        self._enc, self._saved = {}, {}
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            k = 1.0 / math.sqrt(H)
            for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
                t = self.p[f"lstm.{n}"]
                t.copy_(torch.empty(tuple(t.shape)).uniform_(-k, k, generator=gen))
            for n in ("l1_a", "l1_v"):
                self.p[f"{n}.weight"].copy_(orthogonal_((H, H), init_gain("relu"), gen))
            self.p["l2_a.weight"].copy_(orthogonal_((A, H), init_gain("linear"), gen))
            self.p["l2_v.weight"].copy_(orthogonal_((1, H), init_gain("linear"), gen))

    # ------------------------------------------------------------------------------------ forward --
    def encode(self, x, prev_action, S, B, lo, hi, tag):
        """x: S*B time-major rows (a tensor or a frame-ring FrameRows), prev_action int64 [S*B] -> xg [S*B, 4H]."""
        M, F, Z, A, G = S * B, self.F, self.Z, self.D_out, 4 * self.D_hidden
        z = self._buf(tag + "lstm.z", (M, Z))
        if hi > lo:
            z[lo * B:hi * B, :F].copy_(self.head.forward(self, x[lo * B:hi * B], None, (hi - lo) * B, tag, True))
        step = self.head.max_rows
        for r0, r1 in ((0, lo * B), (hi * B, M)):
            for a in range(r0, r1, step):
                e = min(r1, a + step)
                z[a:e, :F].copy_(self.head.forward(self, x[a:e], None, e - a, f"inf{e - a}.", False))
        onehot = self._buf(tag + "lstm.onehot", (M, A), torch.bool)
        torch.eq(prev_action.reshape(M, 1), self._acts, out=onehot)
        z[:, F:].copy_(onehot)
        bias = torch.add(self.p["lstm.bias_ih_l0"], self.p["lstm.bias_hh_l0"], out=self._buf("lstm.bias", (G,)))
        xg = self._buf(tag + "lstm.xg", (M, G))
        C.jb_linear_fwd(ptr(z), ptr(self.p["lstm.weight_ih_l0"]), ptr(bias), ptr(xg), M, Z, G, 0, stream_ptr())
        self._enc[tag] = (lo, hi, B, z)
        return xg

    def unroll(self, xg, s0, S, B, reset, h0, c0, grad_from, tag, save=True):
        """Steps s0 .. s0+S-1 of xg (time-major) from (h0, c0) [B, H]; reset [steps, B] f32 (time-major, indexed like xg).
        The first grad_from steps are the burn-in.  Returns Q [(S - grad_from)*B, A] of the remaining steps."""
        H, A, G = self.D_hidden, self.D_out, 4 * self.D_hidden
        T, s, w = S - grad_from, stream_ptr(), ptr(self.p["lstm.weight_hh_l0"])
        hb = (self._buf(tag + "lstm.hb0", (B, H)), self._buf(tag + "lstm.hb1", (B, H)))
        c = self._buf(tag + "lstm.c", (B, H))
        c.copy_(c0)
        scratch = self._buf(tag + "lstm.gscratch", (B, G))
        h = h0
        for k in range(grad_from):
            st = s0 + k
            C.jb_lstm_step_fwd(ptr(xg[st * B:(st + 1) * B]), ptr(h), ptr(c), w, ptr(reset[st]), B, H, ptr(hb[k % 2]), ptr(c),
                               ptr(scratch), 0, s)
            h = hb[k % 2]
        hs = self._buf(tag + "lstm.hs", (T, B, H))
        if save:
            gates = self._buf(tag + "lstm.gates", (T, B, G))
            cs = self._buf(tag + "lstm.cs", (T + 1, B, H))
            hp = self._buf(tag + "lstm.hprev", (T, B, H))
            cs[0].copy_(c)
            self._saved[tag] = (reset, s0 + grad_from, T, B)
        for k in range(T):
            st = s0 + grad_from + k
            cin, cout = (cs[k], cs[k + 1]) if save else (c, c)
            C.jb_lstm_step_fwd(ptr(xg[st * B:(st + 1) * B]), ptr(h), ptr(cin), w, ptr(reset[st]), B, H, ptr(hs[k]), ptr(cout),
                               ptr(gates[k] if save else scratch), ptr(hp[k]) if save else 0, s)
            h = hs[k]
        return streams_fwd(self, hs.view(T * B, H), T * B, A, tag)

    def step(self, x, prev_action, reset, h, c, h_out, tag="act."):
        """One act() step for M lanes: Q [M, A]; h_out <- h_t (must not be h), c <- c_t in place.  reset f32 [M]."""
        M, H = x.shape[0], self.D_hidden
        xg = self.encode(x, prev_action, 1, M, 0, 0, tag)
        gates = self._buf(tag + "lstm.gscratch", (M, 4 * H))
        C.jb_lstm_step_fwd(ptr(xg), ptr(h), ptr(c), ptr(self.p["lstm.weight_hh_l0"]), ptr(reset), M, H, ptr(h_out), ptr(c),
                           ptr(gates), 0, stream_ptr())
        return streams_fwd(self, h_out, M, self.D_out, tag)

    # ----------------------------------------------------------------------------------- backward --
    def backward_tm(self, dq, tag="t."):
        """dq [T*B, A] (time-major) for the steps the last unroll(save=True) under `tag` trained; writes every gradient."""
        reset, st0, T, B = self._saved[tag]
        lo, hi, Be, z = self._enc[tag]
        assert Be == B and hi - lo == T, "backward_tm needs encode() to have saved exactly the trained rows"
        H, A, F, Z, G = self.D_hidden, self.D_out, self.F, self.Z, 4 * self.D_hidden
        M, s, p, g = T * B, stream_ptr(), self.p, self.g
        hs = self._buf(tag + "lstm.hs", (T, B, H))
        gates = self._buf(tag + "lstm.gates", (T, B, G))
        cs = self._buf(tag + "lstm.cs", (T + 1, B, H))
        hp = self._buf(tag + "lstm.hprev", (T, B, H))
        dh = streams_bwd(self, dq, hs.view(M, H), M, H, A, tag)
        dg = self._buf(tag + "lstm.dgates", (T, B, G))
        dc = self._buf(tag + "lstm.dc", (B, H))
        w = ptr(p["lstm.weight_hh_l0"])
        for k in reversed(range(T)):
            last = k == T - 1
            C.jb_lstm_step_bwd(ptr(dh[k * B:(k + 1) * B]), 0 if last else ptr(dg[k + 1]), w, ptr(gates[k]), ptr(cs[k]),
                               ptr(cs[k + 1]), 0 if last else ptr(dc), ptr(reset[st0 + k]), 0 if last else ptr(reset[st0 + k + 1]),
                               B, H, ptr(dg[k]), ptr(dc), s)
        C.jb_linear_bwd_dw(ptr(dg), ptr(hp), ptr(g["lstm.weight_hh_l0"]), 0, M, H, G, s)
        C.jb_linear_bwd_dw(ptr(dg), ptr(z[lo * B:hi * B]), ptr(g["lstm.weight_ih_l0"]), ptr(g["lstm.bias_ih_l0"]), M, Z, G, s)
        g["lstm.bias_hh_l0"].copy_(g["lstm.bias_ih_l0"])
        feat = self._buf(tag + "head.h", (M, F))
        dfeat = self._buf(tag + "lstm.dfeat", (M, F))
        # d feat = (dgates W_ih)[:, :F], masked by the head's ReLU output: the one-hot columns need no gradient
        C.jb_gemm(ptr(dg), G, 1, ptr(p["lstm.weight_ih_l0"]), Z, 0, ptr(dfeat), F, M, F, G, 0, 0, ptr(feat), F, 0, 0, s)
        self.head.backward(self, dfeat, M, tag)

    # ----------------------------------------------------------------------------- batch-major API --
    def forward_seq(self, x, prev_action, reset, h0, c0, grad_from=0, tag="t."):
        """x: B*S batch-major rows (tensor [B*S, ...] or FrameRows), prev_action int64 [B, S], reset [B, S], (h0, c0) [B, H].
        Steps before grad_from are the burn-in (no gradient).  Returns Q [B, S - grad_from, A]."""
        B, S = prev_action.shape
        T, A = S - grad_from, self.D_out
        x_tm = _time_major_rows(x, B, S)
        prev = prev_action.t().contiguous().reshape(-1)
        rs = reset.to(torch.float32).t().contiguous()
        xg = self.encode(x_tm, prev, S, B, grad_from, S, tag)
        q = self.unroll(xg, 0, S, B, rs, h0, c0, grad_from, tag)
        return q.view(T, B, A).transpose(0, 1).contiguous()

    def backward_seq(self, dq, tag="t."):
        """dq [B, T, A] for the trained steps of the last forward_seq."""
        B, T, A = dq.shape
        self.backward_tm(dq.transpose(0, 1).contiguous().view(T * B, A), tag)


def _time_major_rows(x, B, S):
    if torch.is_tensor(x):
        return x.reshape(B, S, *x.shape[1:]).transpose(0, 1).contiguous().reshape(B * S, *x.shape[1:])
    return type(x)(x.store, x.refs.view(B, S).t().contiguous().view(-1))
