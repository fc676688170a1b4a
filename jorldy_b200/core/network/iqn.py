"""Implicit quantile network (Dabney et al. 2018, arXiv:1806.06923):

    psi = head(x)                                   [B, Dh]      (mlp: relu(Linear(D_in, H)); cnn: the conv trunk)
    phi = relu(sample_embed(cos(pi i tau)))         [B, N, Dh]   i = 0 .. D_em - 1, one row per sampled fraction tau
    q   = q(relu(l(psi (*) phi)))                   [B, N, A]

The cosine features c [B*N, D_em] are materialised (jb_iqn_cos) so that sample_embed runs on the dense GEMM tiles
forward and its weight gradient on jb_linear_bwd_dw; the product and its fused backward are csrc/quantile.cu.
"""
import torch

from ..dev import C, ptr, stream_ptr
from .base import FlatNetwork, init_gain, orthogonal_
from .head import make_head
from . import layers as L

ROW_BYTES_PER_PASS = 32 << 20      # act(): one [rows*N, Dh] activation chunk, sized like MAX_ROWS_PER_PASS rows at Dh=512


def rows_per_pass(head, N):
    """act()'s chunk of state rows: rows * N fraction rows of [Dh] activation fit in ROW_BYTES_PER_PASS (e.g. 41 lanes x
    64 samples at the CNN head's Dh = 3136)."""
    return max(1, min(head.max_rows, ROW_BYTES_PER_PASS // (4 * head.D_head_out * N)))


def embed_fwd(net, psi, tau, tag):
    """z [B*N, Dh] = psi (*) relu(sample_embed(cos(pi i tau))) from the head output psi [B, Dh] and the fractions tau
    [B, N], with net's sample_embed; the cosines and phi stay under `tag` for embed_bwd."""
    B, N = tau.shape
    p, Dh, s = net.p, net.head.D_head_out, stream_ptr()
    c = net._buf(tag + "cos", (B * N, net.D_em))
    C.jb_iqn_cos(ptr(tau), B * N, net.D_em, ptr(c), s)
    phi = net._buf(tag + "phi", (B * N, Dh))
    L.linear_fwd(c, p["sample_embed.weight"], p["sample_embed.bias"], phi, relu=True)
    z = net._buf(tag + "z", (B * N, Dh))
    C.jb_iqn_mul_fwd(ptr(psi), ptr(phi), B, N, Dh, ptr(z), s)
    return z


def embed_bwd(net, dz, B, N, tag):
    """From dz = d loss / d z: writes the sample_embed gradients and returns d loss / d psi [B, Dh] (masked by psi > 0)."""
    g, Dh = net.g, net.head.D_head_out
    psi = net._buf(tag + "head.h", (B, Dh))
    c = net._buf(tag + "cos", (B * N, net.D_em))
    phi = net._buf(tag + "phi", (B * N, Dh))
    dpsi = net._buf(tag + "dpsi", (B, Dh))
    dpre = net._buf(tag + "dpre", (B * N, Dh))
    C.jb_iqn_mul_bwd(ptr(dz), ptr(psi), ptr(phi), B, N, Dh, ptr(dpsi), ptr(dpre), stream_ptr())
    L.linear_bwd_dw(dpre, c, g["sample_embed.weight"], g["sample_embed.bias"])
    return dpsi


class IQN(FlatNetwork):
    def __init__(self, D_in, D_out, D_em=64, D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        self.D_in, self.D_out, self.D_em, self.D_hidden = D_in, D_out, D_em, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        Dh, H = self.head.D_head_out, D_hidden
        self._specs = self.head.specs() + [("sample_embed.weight", (Dh, D_em)), ("sample_embed.bias", (Dh,)),
                                           ("l.weight", (H, Dh)), ("l.bias", (H,)),
                                           ("q.weight", (D_out, H)), ("q.bias", (D_out,))]
        self._allocate()
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            self.p["sample_embed.weight"].copy_(orthogonal_((Dh, D_em), init_gain("relu"), gen))
            self.p["l.weight"].copy_(orthogonal_((H, Dh), init_gain("relu"), gen))
            self.p["q.weight"].copy_(orthogonal_((D_out, H), init_gain("linear"), gen))
        self._saved = {}

    def forward(self, x, tau, tag="t.", out=None, save=True):
        """x [B, ...] device rows, tau [B, N] f32 fractions -> out [B*N, A] (row b*N + n: sample n of state b)."""
        B, N = tau.shape
        p = self.p
        psi = self.head.forward(self, x, None, B, tag, save)
        z = embed_fwd(self, psi, tau, tag)
        h2 = self._buf(tag + "h2", (B * N, self.D_hidden))
        L.linear_fwd(z, p["l.weight"], p["l.bias"], h2, relu=True)
        if out is None:
            out = self._buf(tag + "out", (B * N, self.D_out))
        L.heads_fwd(h2, [(p["q.weight"], p["q.bias"])], out)
        self._saved[tag] = (B, N)
        return out

    def forward_rows(self, x, tau, out):
        """Inference over many rows (act() on thousands of lanes) in chunks of rows_per_pass rows."""
        M, N = tau.shape
        per = rows_per_pass(self.head, N)
        for s in range(0, M, per):
            e = min(M, s + per)
            self.forward(x[s:e], tau[s:e], tag=f"inf{e - s}.", out=out[s * N:e * N], save=False)
        return out

    def backward(self, dout, tag="t."):
        """dout [B*N, A] = d loss / d forward output; fills self.grad (overwrites)."""
        B, N = self._saved[tag]
        p, g, Dh, H = self.p, self.g, self.head.D_head_out, self.D_hidden
        z = self._buf(tag + "z", (B * N, Dh))
        h2 = self._buf(tag + "h2", (B * N, H))
        dh2 = self._buf(tag + "dh2", (B * N, H))
        dz = self._buf(tag + "dz", (B * N, Dh))
        L.heads_bwd_dw(dout, h2, [(g["q.weight"], g["q.bias"])])
        L.heads_bwd_dx(dout, h2, [(p["q.weight"], None)], dh2)                 # masked by relu(h2)
        L.linear_bwd_dw(dh2, z, g["l.weight"], g["l.bias"])
        L.linear_bwd_dx(dh2, p["l.weight"], dz)
        self.head.backward(self, embed_bwd(self, dz, B, N, tag), B, tag)
