"""Dueling Q network (jorldy/core/network/dueling.py:8-35): head -> {l1_a, l1_v} (Linear+ReLU) ->
{l2_a [A], l2_v [1]} -> Q = V + A - mean_a A."""
import torch

from ..dev import C, ptr, stream_ptr
from .base import FlatNetwork, init_gain, orthogonal_
from .head import make_head
from . import layers as L


class Dueling(FlatNetwork):
    def __init__(self, D_in, D_out, D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        self.D_in, self.D_out, self.D_hidden = D_in, D_out, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        F = self.head.D_head_out
        self._specs = self.head.specs() + [
            ("l1_a.weight", (D_hidden, F)), ("l1_a.bias", (D_hidden,)),
            ("l1_v.weight", (D_hidden, F)), ("l1_v.bias", (D_hidden,)),
            ("l2_a.weight", (D_out, D_hidden)), ("l2_a.bias", (D_out,)),
            ("l2_v.weight", (1, D_hidden)), ("l2_v.bias", (1,))]
        self._allocate()
        self.nout = D_out
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            for n in ("l1_a", "l1_v"):
                self.p[f"{n}.weight"].copy_(orthogonal_((D_hidden, F), init_gain("relu"), gen))
            self.p["l2_a.weight"].copy_(orthogonal_((D_out, D_hidden), init_gain("linear"), gen))
            self.p["l2_v.weight"].copy_(orthogonal_((1, D_hidden), init_gain("linear"), gen))

    def forward(self, x, idx=None, M=None, out=None, tag="t.", save=True):
        M = M if M is not None else (idx.shape[0] if idx is not None else x.shape[0])
        A = self.D_out
        feat = self.head.forward(self, x, idx, M, tag, save)
        return streams_fwd(self, feat, M, A, tag, out)

    def forward_rows(self, x, out):
        M = x.shape[0]
        for s in range(0, M, self.head.max_rows):
            e = min(M, s + self.head.max_rows)
            self.forward(x[s:e], None, e - s, out[s:e], tag=f"inf{e - s}.", save=False)
        return out

    def backward(self, dq, M, tag="t."):
        feat = self._buf(tag + "head.h", (M, self.head.D_head_out))
        dfeat = streams_bwd(self, dq, feat, M, self.D_hidden, self.D_out, tag, relu_act=feat)
        self.head.backward(self, dfeat, M, tag)


def streams_fwd(net, feat, M, A, tag, out=None):
    """Q [M, A] = V + A - mean A of the l1_a / l1_v / l2_a / l2_v streams on feat [M, F] (net's flat views)."""
    p, H = net.p, net.p["l1_a.weight"].shape[0]
    xa = net._buf(tag + "xa", (M, H)); xv = net._buf(tag + "xv", (M, H))
    L.linear_fwd(feat, p["l1_a.weight"], p["l1_a.bias"], xa, relu=True)
    L.linear_fwd(feat, p["l1_v.weight"], p["l1_v.bias"], xv, relu=True)
    a = net._buf(tag + "a", (M, A)); v = net._buf(tag + "v", (M, 1))
    L.heads_fwd(xa, [(p["l2_a.weight"], p["l2_a.bias"])], a)
    L.heads_fwd(xv, [(p["l2_v.weight"], p["l2_v.bias"])], v)
    if out is None:
        out = net._buf(tag + "q", (M, A))
    C.jb_dueling_fwd(ptr(a), ptr(v), M, A, 1, ptr(out), stream_ptr())
    return out


def streams_bwd(net, dq, feat, M, H, A, tag, relu_act=None):
    """Writes the four streams' gradients from dq [M, A] and returns d loss / d feat [M, F] (masked by relu_act when
    given), using the activations streams_fwd saved under `tag`."""
    p, g = net.p, net.g
    xa = net._buf(tag + "xa", (M, H)); xv = net._buf(tag + "xv", (M, H))
    da = net._buf(tag + "da", (M, A)); dv = net._buf(tag + "dv", (M, 1))
    C.jb_dueling_bwd(ptr(dq), M, A, 1, ptr(da), ptr(dv), stream_ptr())
    dxa = net._buf(tag + "dxa", (M, H)); dxv = net._buf(tag + "dxv", (M, H))
    L.heads_bwd_dw(da, xa, [(g["l2_a.weight"], g["l2_a.bias"])])
    L.heads_bwd_dx(da, xa, [(p["l2_a.weight"], None)], dxa)
    L.heads_bwd_dw(dv, xv, [(g["l2_v.weight"], g["l2_v.bias"])])
    L.heads_bwd_dx(dv, xv, [(p["l2_v.weight"], None)], dxv)
    L.linear_bwd_dw(dxa, feat, g["l1_a.weight"], g["l1_a.bias"])
    L.linear_bwd_dw(dxv, feat, g["l1_v.weight"], g["l1_v.bias"])
    dfeat = net._buf(tag + "dfeat", (M, feat.shape[1]))
    L.linear_bwd_dx(dxa, p["l1_a.weight"], dfeat, relu_act=relu_act)
    L.linear_bwd_dx(dxv, p["l1_v.weight"], dfeat, relu_act=relu_act, accumulate=True)
    return dfeat
