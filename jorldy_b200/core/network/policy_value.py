"""Trunk + narrow-heads networks: head -> l (Linear+ReLU) -> up to four narrow output heads.

Actor-critic (jorldy/core/network/policy_value.py:8-22 discrete, :38-57 continuous) and the plain
Q network (q_network.py:8-20) share this shape.  forward_raw returns the PRE-activation head
outputs; softmax / clamp / tanh-exp live in the fused agent kernels (csrc/ppo.cu)."""
import torch

from .base import FlatNetwork, init_gain, orthogonal_
from .head import make_head
from . import layers as L


class _PolicyValue(FlatNetwork):
    head_names = ()        # e.g. ("pi", "v"): (name, n_out, gain)

    def __init__(self, D_in, D_out, D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        self.D_in, self.D_out, self.D_hidden = D_in, D_out, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        self.out_heads = self._out_heads(D_out)
        self.nout = sum(n for _, n, _ in self.out_heads)
        self._wide = self.nout > 32
        assert not self._wide or len(self.out_heads) == 1
        specs = self.head.specs() + [("l.weight", (D_hidden, self.head.D_head_out)), ("l.bias", (D_hidden,))]
        for name, n, _ in self.out_heads:
            specs += [(f"{name}.weight", (n, D_hidden)), (f"{name}.bias", (n,))]
        self._specs = specs
        self._allocate()
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            self.p["l.weight"].copy_(orthogonal_((D_hidden, self.head.D_head_out), init_gain("relu"), gen))
            for name, n, gain in self.out_heads:
                self.p[f"{name}.weight"].copy_(orthogonal_((n, D_hidden), init_gain(gain), gen))

    def _heads_wb(self):
        return [(self.p[f"{n}.weight"], self.p[f"{n}.bias"]) for n, _, _ in self.out_heads]

    def _heads_grads(self):
        return [(self.g[f"{n}.weight"], self.g[f"{n}.bias"]) for n, _, _ in self.out_heads]

    def forward_raw(self, x, idx=None, M=None, out=None, tag="t.", save=True):
        """x [rows, D] f32 device tensor; returns out [M, nout] pre-activation head outputs."""
        M = M if M is not None else (idx.shape[0] if idx is not None else x.shape[0])
        h1 = self.head.forward(self, x, idx, M, tag, save)
        h2 = self._buf(tag + "h2", (M, self.D_hidden))
        L.linear_fwd(h1, self.p["l.weight"], self.p["l.bias"], h2, relu=True)
        if out is None:
            out = self._buf(tag + "out", (M, self.nout))
        if self._wide:      # a single wide head (e.g. C51's A*K logits): tiled GEMM instead of the row kernel
            w, b = self._heads_wb()[0]
            L.linear_fwd(h2, w, b, out, relu=False)
        else:
            L.heads_fwd(h2, self._heads_wb(), out)
        return out

    def forward_rows(self, x, out):
        """Inference over many rows in L2-sized chunks (act() on thousands of envs, PPO pre-pass)."""
        M = x.shape[0]
        for s in range(0, M, self.head.max_rows):
            e = min(M, s + self.head.max_rows)
            self.forward_raw(x[s:e], None, e - s, out[s:e], tag=f"inf{e - s}.", save=False)
        return out

    def backward_raw(self, dout, M, tag="t."):
        """dout [M, nout] = d loss / d forward_raw output; fills self.grad (overwrites)."""
        h1 = self._buf(tag + "head.h", (M, self.head.D_head_out))
        h2 = self._buf(tag + "h2", (M, self.D_hidden))
        dh2 = self._buf(tag + "dh2", (M, self.D_hidden))
        dh1 = self._buf(tag + "dh1", (M, self.head.D_head_out))
        if self._wide:
            (w, _), (dw, db) = self._heads_wb()[0], self._heads_grads()[0]
            L.linear_bwd_dw(dout, h2, dw, db)
            L.linear_bwd_dx(dout, w, dh2, relu_act=h2)
        else:
            L.heads_bwd_dw(dout, h2, self._heads_grads())
            L.heads_bwd_dx(dout, h2, self._heads_wb(), dh2)             # masked by relu(h2)
        L.linear_bwd_dw(dh2, h1, self.g["l.weight"], self.g["l.bias"])
        L.linear_bwd_dx(dh2, self.p["l.weight"], dh1, relu_act=h1)      # masked by relu(h1)
        self.head.backward(self, dh1, M, tag)


class DiscreteQ_Network(_PolicyValue):
    """q_network.py:8-20: head -> l -> q."""

    def _out_heads(self, D_out):
        return [("q", D_out, "linear")]

    def forward(self, x, *args, **kwargs):
        return self.forward_raw(x, *args, **kwargs)

    def backward(self, dq, M, tag="t."):
        return self.backward_raw(dq, M, tag=tag)


class DiscretePolicyValue(_PolicyValue):
    def _out_heads(self, D_out):
        return [("pi", D_out, "policy"), ("v", 1, "linear")]


class ContinuousPolicyValue(_PolicyValue):
    def _out_heads(self, D_out):
        return [("mu", D_out, "linear"), ("log_std", D_out, "tanh"), ("v", 1, "linear")]


class DiscretePolicyTwoValue(_PolicyValue):
    """RND-PPO's policy network: PPO's discrete heads and an intrinsic value head v_i, out = [pi | v | v_i]."""

    def _out_heads(self, D_out):
        return [("pi", D_out, "policy"), ("v", 1, "linear"), ("v_i", 1, "linear")]


class ContinuousPolicyTwoValue(_PolicyValue):
    """RND-PPO's policy network: PPO's continuous heads and v_i, out = [mu | log_std | v | v_i]."""

    def _out_heads(self, D_out):
        return [("mu", D_out, "linear"), ("log_std", D_out, "tanh"), ("v", 1, "linear"), ("v_i", 1, "linear")]
