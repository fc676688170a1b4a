"""MuZero's three networks (Schrittwieser et al., arXiv:1911.08265), H = D_hidden, Hs = latent_size:
  representation h:  x [D] -> H (ReLU) -> Hs, min-max scaled
                     (head="cnn", D_in = (4, 84, 84): the 4 frames + 4 action planes [8, 84, 84] -> the CNN head's trunk
                     (conv 8x8s4 -> 4x4s2 -> 3x3s1, ReLU each) -> 3136 -> Hs, min-max scaled)
  dynamics g:        [s, onehot(a)] [Hs + A] -> H (ReLU) -> next latent Hs (min-max scaled) and reward logits 2R + 1
  prediction f:      s [Hs] -> H (ReLU) -> policy logits A and value logits 2V + 1
Every latent is scaled per row to [0, 1] as (s - min) / max(max - min, 1e-5) (jb_muzero_scale_fwd).

Parameters, in state_dict order: `h.l1.weight [H, D]`, `h.l1.bias`, `h.l2.weight [Hs, H]`, `h.l2.bias`, `g.l1.weight
[H, Hs + A]`, `g.l1.bias`, `g.s.weight [Hs, H]`, `g.s.bias`, `g.r.weight [2R + 1, H]`, `g.r.bias`, `f.l1.weight [H, Hs]`,
`f.l1.bias`, `f.pi.weight [A, H]`, `f.pi.bias`, `f.v.weight [2V + 1, H]`, `f.v.bias`.  Weights are orthogonal (gain
sqrt(2) before a ReLU, 0.01 for the policy, 1 otherwise), biases zero.  With head="cnn", h's parameters are
`head.conv1.weight [32, 8, 8, 8]`, `head.conv1.bias`, `head.conv2.*`, `head.conv3.*` (the CNN head's names and init) and
`h.l.weight [Hs, 3136]`, `h.l.bias`, in place of h.l1 / h.l2.  D_repr is the width of h's hidden activation h1: H, or
the trunk's 3136 features.

The callers own the activation buffers: each method takes its inputs and outputs, so the learner can lay the K + 1 unroll
steps out as one time-major block ([k * B + b] is step k of window b) and run f over all of them at once.  The backward
methods overwrite the gradients they produce; each weight gradient is one product over all the rows that used it.
"""
import torch

from ..dev import C, ptr, stream_ptr
from . import layers as L
from .base import FlatNetwork, init_gain, orthogonal_
from .head import CNNHead

NARROW = 32         # heads of at most this many outputs use the row kernel (csrc/heads.cu); wider ones the GEMM


class MuZero(FlatNetwork):
    def __init__(self, D_in, D_out, D_hidden=128, latent_size=64, value_support=20, reward_support=1, head="mlp",
                 device=None, seed=None):
        super().__init__(device)
        A, H, Hs = int(D_out), int(D_hidden), int(latent_size)
        if head == "cnn":
            C_, Hh, Ww = (int(d) for d in D_in)
            self.trunk = CNNHead((2 * C_, Hh, Ww))        # frames + one action plane per frame
            D = (C_, Hh, Ww)
            self.D_repr = self.trunk.D_head_out
            h_specs = self.trunk.specs() + [("h.l.weight", (Hs, self.D_repr)), ("h.l.bias", (Hs,))]
        elif head == "mlp" and isinstance(D_in, int):
            self.trunk, D, self.D_repr = None, int(D_in), H
            h_specs = [("h.l1.weight", (H, D)), ("h.l1.bias", (H,)), ("h.l2.weight", (Hs, H)), ("h.l2.bias", (Hs,))]
        else:
            raise NotImplementedError("MuZero takes flat observations with head='mlp' or frame stacks with head='cnn'")
        self.D_in, self.D_out, self.D_hidden, self.Hs = D, A, H, Hs
        self.V, self.R = int(value_support), int(reward_support)
        nv, nr = 2 * self.V + 1, 2 * self.R + 1
        self._specs = h_specs + [
                       ("g.l1.weight", (H, Hs + A)), ("g.l1.bias", (H,)), ("g.s.weight", (Hs, H)), ("g.s.bias", (Hs,)),
                       ("g.r.weight", (nr, H)), ("g.r.bias", (nr,)), ("f.l1.weight", (H, Hs)), ("f.l1.bias", (H,)),
                       ("f.pi.weight", (A, H)), ("f.pi.bias", (A,)), ("f.v.weight", (nv, H)), ("f.v.bias", (nv,))]
        self._allocate()
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        h_gains = {"h.l": "linear"} if self.trunk is not None else {"h.l1": "relu", "h.l2": "linear"}
        gains = dict(h_gains, **{"g.l1": "relu", "g.s": "linear", "g.r": "linear", "f.l1": "relu", "f.pi": "policy",
                                 "f.v": "linear"})
        with torch.no_grad():
            if self.trunk is not None:
                self.trunk.init(self.p, gen)
            for name, gain in gains.items():
                w = self.p[f"{name}.weight"]
                w.copy_(orthogonal_(tuple(w.shape), init_gain(gain), gen))

    def _w(self, name):
        return self.p[f"{name}.weight"], self.p[f"{name}.bias"]

    def _head_fwd(self, h, name, out):
        w, b = self._w(name)
        if w.shape[0] <= NARROW:
            L.heads_fwd(h, [(w, b)], out)
        else:
            L.linear_fwd(h, w, b, out, relu=False)

    def _head_bwd(self, dout, h, name, dh, accumulate):
        """Weight gradients of one head and dh (+)= dout W masked by relu(h)."""
        L.linear_bwd_dw(dout, h, self.g[f"{name}.weight"], self.g[f"{name}.bias"])
        L.linear_bwd_dx(dout, self.p[f"{name}.weight"], dh, relu_act=h, accumulate=accumulate)

    # ------------------------------------------------------------------------------------ forward --
    def represent(self, x, h1, pre, s, s2=None, tag="t."):
        """x [M, D] -> h1 [M, D_repr], pre [M, Hs] (before scaling), s [M, Hs]; s2 (a column block with its own row
        stride, e.g. the first dynamics input) receives s too.  head="cnn": x is a FrameActionRows (buffer/frame_store.py)
        and the trunk keeps its column matrices under `tag` for represent_bwd."""
        if self.trunk is not None:
            self.trunk.forward(self, x, None, h1.shape[0], tag, True, out=h1)
            L.linear_fwd(h1, *self._w("h.l"), pre, relu=False)
        else:
            L.linear_fwd(x, *self._w("h.l1"), h1, relu=True)
            L.linear_fwd(h1, *self._w("h.l2"), pre, relu=False)
        self.scale(pre, s, s2)

    def dynamics(self, z, hid, pre, s, r_logits, s2=None):
        """z [M, Hs + A] = [s, onehot(a)] -> hid [M, H], pre [M, Hs], s [M, Hs] (and s2), r_logits [M, 2R + 1]."""
        L.linear_fwd(z, *self._w("g.l1"), hid, relu=True)
        L.linear_fwd(hid, *self._w("g.s"), pre, relu=False)
        self._head_fwd(hid, "g.r", r_logits)
        self.scale(pre, s, s2)

    def predict(self, s, hid, pi_logits, v_logits):
        """s [M, Hs] -> hid [M, H], pi_logits [M, A], v_logits [M, 2V + 1]."""
        L.linear_fwd(s, *self._w("f.l1"), hid, relu=True)
        self._head_fwd(hid, "f.pi", pi_logits)
        self._head_fwd(hid, "f.v", v_logits)

    def scale(self, pre, s, s2=None):
        M, Hs = pre.shape
        C.jb_muzero_scale_fwd(ptr(pre), M, Hs, ptr(s), ptr(s2), s2.stride(0) if s2 is not None else 0, stream_ptr())

    # ----------------------------------------------------------------------------------- backward --
    def predict_bwd(self, s, hid, d_pi, d_v, dhid, ds):
        """Gradients of f from d_pi, d_v over the rows of s; ds [M, Hs] = d loss / d s through f."""
        self._head_bwd(d_pi, hid, "f.pi", dhid, False)
        self._head_bwd(d_v, hid, "f.v", dhid, True)
        L.linear_bwd_dw(dhid, s, self.g["f.l1.weight"], self.g["f.l1.bias"])
        L.linear_bwd_dx(dhid, self.p["f.l1.weight"], ds)

    def scale_bwd(self, pre, ds, dpre):
        M, Hs = pre.shape
        C.jb_muzero_scale_bwd(ptr(pre), ptr(ds), M, Hs, ptr(dpre), stream_ptr())

    def dynamics_bwd_step(self, hid, dpre, d_r, dhid, ds_in):
        """One step: dhid = (dpre W_s + d_r W_r) masked by relu(hid); ds_in [M, Hs] = the gradient into the latent part of
        the dynamics input (dhid W_1[:, :Hs]).  The weight gradients come from dynamics_bwd_weights over all steps."""
        M, H = hid.shape
        Hs, A = self.Hs, self.D_out
        L.linear_bwd_dx(dpre, self.p["g.s.weight"], dhid, relu_act=hid)
        L.linear_bwd_dx(d_r, self.p["g.r.weight"], dhid, relu_act=hid, accumulate=True)
        C.jb_gemm(ptr(dhid), H, 1, ptr(self.p["g.l1.weight"]), Hs + A, 0, ptr(ds_in), Hs, M, Hs, H, 0, 0, 0, 0, 0, 0,
                  stream_ptr())

    def dynamics_bwd_weights(self, z, hid, dpre, d_r, dhid):
        """g's weight gradients over all the unrolled rows (z, hid, dpre, d_r, dhid stacked over the steps)."""
        L.linear_bwd_dw(dpre, hid, self.g["g.s.weight"], self.g["g.s.bias"])
        L.linear_bwd_dw(d_r, hid, self.g["g.r.weight"], self.g["g.r.bias"])
        L.linear_bwd_dw(dhid, z, self.g["g.l1.weight"], self.g["g.l1.bias"])

    def represent_bwd(self, x, h1, dpre, dh1, tag="t."):
        if self.trunk is not None:
            L.linear_bwd_dw(dpre, h1, self.g["h.l.weight"], self.g["h.l.bias"])
            L.linear_bwd_dx(dpre, self.p["h.l.weight"], dh1, relu_act=h1)
            self.trunk.backward(self, dh1, h1.shape[0], tag)
            return
        L.linear_bwd_dw(dpre, h1, self.g["h.l2.weight"], self.g["h.l2.bias"])
        L.linear_bwd_dx(dpre, self.p["h.l2.weight"], dh1, relu_act=h1)
        L.linear_bwd_dw(dh1, x, self.g["h.l1.weight"], self.g["h.l1.bias"])
