"""Rainbow-IQN network (Toromanoff et al. 2019, arXiv:1908.04683): IQN's sampled-fraction embedding (iqn.py) feeding
Rainbow's noisy dueling streams (noisy.py), one output row per (state, fraction):

    psi = head(x)                                        [B, Dh]     (mlp: relu(Linear(D_in, H)); cnn: the conv trunk)
    phi = relu(sample_embed(cos(pi i tau)))              [B*N, Dh]   i = 0 .. D_em - 1
    f   = relu(l(psi (*) phi))                           [B*N, H]
    xa  = relu(noisy_a1(f)),  xv = relu(noisy_v1(f))     [B*N, H]
    out = v + (a - mean_a a),  a = noisy_a2(xa) [B*N, A],  v = noisy_v2(xv) [B*N, 1]

Built from existing pieces only: IQN's embedding (iqn.embed_fwd / embed_bwd), the dense GEMM layers and the Rainbow
network's noisy dueling streams (noisy.streams_fwd / streams_bwd with K = 1).  Parameters: the noisy tensors (a1, v1, a2,
v2 as in the Rainbow network), then the head, sample_embed and l; the four noisy layers draw from Philox streams 1..4.
A forward draws fresh noise for all four layers once; forward_rows (act()) draws it once per call and reuses it for every
chunk of rows.
"""
import torch

from .base import FlatNetwork, init_gain, orthogonal_
from .head import make_head
from .iqn import embed_bwd, embed_fwd, rows_per_pass
from .noisy import _NoisyMixin, dueling_layers, streams_bwd, streams_fwd
from . import layers as L


class RainbowIQN(FlatNetwork, _NoisyMixin):
    def __init__(self, D_in, D_out, D_em=64, noise_type="factorized", D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        self._noisy_setup(noise_type, seed)
        self.D_in, self.D_out, self.D_em, self.D_hidden = D_in, D_out, D_em, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        Dh, H = self.head.D_head_out, D_hidden
        self._noisy = dueling_layers(H, D_out, 1)
        self._specs = self._noisy_param_specs() + self.head.specs() + [
            ("sample_embed.weight", (Dh, D_em)), ("sample_embed.bias", (Dh,)), ("l.weight", (H, Dh)), ("l.bias", (H,))]
        self._allocate()
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            self.p["sample_embed.weight"].copy_(orthogonal_((Dh, D_em), init_gain("relu"), gen))
            self.p["l.weight"].copy_(orthogonal_((H, Dh), init_gain("relu"), gen))
            self._noisy_init_params(gen)
        self._saved = {}

    def _body(self, x, tau, wb, tag, out, save):
        B, N = tau.shape
        M, p, A = B * N, self.p, self.D_out
        psi = self.head.forward(self, x, None, B, tag, save)
        z = embed_fwd(self, psi, tau, tag)
        f = self._buf(tag + "f", (M, self.D_hidden))
        L.linear_fwd(z, p["l.weight"], p["l.bias"], f, relu=True)
        if out is None:
            out = self._buf(tag + "out", (M, A))
        streams_fwd(self, f, M, A, 1, wb, tag, out)
        self._saved[tag] = (B, N)
        return out

    def forward(self, x, tau, is_train=True, tag="t.", noise=None):
        """x [B, ...] device rows, tau [B, N] f32 fractions -> [B*N, A] (row b*N + n: fraction n of state b)."""
        return self._body(x, tau, self._make_noise(tag, is_train, noise), tag, None, True)

    def forward_rows(self, x, tau, out, is_train=True, noise=None):
        """Inference over many rows (act()): one noise draw for the whole call, then IQN's chunks of rows_per_pass rows,
        every chunk on the same effective weights."""
        M, N = tau.shape
        wb = self._make_noise("inf.", is_train, noise)
        per = rows_per_pass(self.head, N)
        for s in range(0, M, per):
            e = min(M, s + per)
            self._body(x[s:e], tau[s:e], wb, f"inf{e - s}.", out[s * N:e * N], False)
        return out

    def backward(self, dout, tag="t."):
        """dout [B*N, A] = d loss / d forward output; fills self.grad (overwrites)."""
        B, N = self._saved[tag]
        M, Dh = B * N, self.head.D_head_out
        z = self._buf(tag + "z", (M, Dh))
        f = self._buf(tag + "f", (M, self.D_hidden))
        df = streams_bwd(self, dout, f, M, self.D_out, 1, tag)
        L.linear_bwd_dw(df, z, self.g["l.weight"], self.g["l.bias"])
        dz = self._buf(tag + "dz", (M, Dh))
        L.linear_bwd_dx(df, self.p["l.weight"], dz)
        self.head.backward(self, embed_bwd(self, dz, B, N, tag), B, tag)
