"""Rainbow-IQN network (Toromanoff et al. 2019, arXiv:1908.04683): IQN's sampled-fraction embedding (iqn.py) feeding
Rainbow's noisy dueling streams (noisy.py), one output row per (state, fraction):

    psi = head(x)                                        [B, Dh]     (mlp: relu(Linear(D_in, H)); cnn: the conv trunk)
    phi = relu(sample_embed(cos(pi i tau)))              [B*N, Dh]   i = 0 .. D_em - 1
    f   = relu(l(psi (*) phi))                           [B*N, H]
    xa  = relu(noisy_a1(f)),  xv = relu(noisy_v1(f))     [B*N, H]
    out = v + (a - mean_a a),  a = noisy_a2(xa) [B*N, A],  v = noisy_v2(xv) [B*N, 1]

Built from existing kernels only: jb_iqn_cos / jb_iqn_mul_fwd / jb_iqn_mul_bwd, the dense GEMM layers, jb_noisy_make /
jb_noisy_grad and jb_dueling_fwd / bwd with K = 1.  Parameters: the noisy tensors (a1, v1, a2, v2 as in the Rainbow
network), then the head, sample_embed and l; the four noisy layers draw from Philox streams 1..4.  A forward draws fresh
noise for all four layers once; forward_rows (act()) draws it once per call and reuses it for every chunk of rows.
"""
import torch

from ..dev import C, ptr, stream_ptr
from .base import FlatNetwork, init_gain, orthogonal_
from .head import make_head
from .iqn import ROW_BYTES_PER_PASS
from .noisy import _NoisyMixin, _noisy_init, _noisy_specs
from . import layers as L

_LAYERS = (("_a1", 1), ("_v1", 2), ("_a2", 3), ("_v2", 4))      # call order of the noise draws, Philox stream ids


class RainbowIQN(FlatNetwork, _NoisyMixin):
    def __init__(self, D_in, D_out, D_em=64, noise_type="factorized", D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        self._noisy_setup(noise_type, seed)
        self.D_in, self.D_out, self.D_em, self.D_hidden = D_in, D_out, D_em, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        Dh, H = self.head.D_head_out, D_hidden
        self._dims = {"_a1": (H, H), "_v1": (H, H), "_a2": (H, D_out), "_v2": (H, 1)}
        self._specs = [s for lt, _ in _LAYERS for s in _noisy_specs(lt, *self._dims[lt])] + self.head.specs() + [
            ("sample_embed.weight", (Dh, D_em)), ("sample_embed.bias", (Dh,)), ("l.weight", (H, Dh)), ("l.bias", (H,))]
        self._allocate()
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            self.p["sample_embed.weight"].copy_(orthogonal_((Dh, D_em), init_gain("relu"), gen))
            self.p["l.weight"].copy_(orthogonal_((H, Dh), init_gain("relu"), gen))
            for lt, _ in _LAYERS:
                _noisy_init(self.p, lt, *self._dims[lt], noise_type, gen)
        self._saved = {}

    def _make_noise(self, tag, is_train, noise):
        """Effective (W, b) of the four noisy layers in call order a1, v1, a2, v2; noise: injected [(eps_i, eps_j)] x 4."""
        noise = noise if noise is not None else (None,) * 4
        return {lt: self._noisy_make(tag, lt, lid, *self._dims[lt], is_train, nz) for (lt, lid), nz in zip(_LAYERS, noise)}

    def _body(self, x, tau, wb, tag, out, save):
        B, N = tau.shape
        M, p, Dh, H, A, s = B * N, self.p, self.head.D_head_out, self.D_hidden, self.D_out, stream_ptr()
        psi = self.head.forward(self, x, None, B, tag, save)
        c = self._buf(tag + "cos", (M, self.D_em))
        C.jb_iqn_cos(ptr(tau), M, self.D_em, ptr(c), s)
        phi = self._buf(tag + "phi", (M, Dh))
        L.linear_fwd(c, p["sample_embed.weight"], p["sample_embed.bias"], phi, relu=True)
        z = self._buf(tag + "z", (M, Dh))
        C.jb_iqn_mul_fwd(ptr(psi), ptr(phi), B, N, Dh, ptr(z), s)
        f = self._buf(tag + "f", (M, H))
        L.linear_fwd(z, p["l.weight"], p["l.bias"], f, relu=True)
        xa = self._buf(tag + "xa", (M, H)); xv = self._buf(tag + "xv", (M, H))
        L.linear_io_fwd(f, *wb["_a1"], xa, relu=True)
        L.linear_io_fwd(f, *wb["_v1"], xv, relu=True)
        a = self._buf(tag + "a", (M, A)); v = self._buf(tag + "v", (M, 1))
        L.linear_io_fwd(xa, *wb["_a2"], a, relu=False)
        L.linear_io_fwd(xv, *wb["_v2"], v, relu=False)
        if out is None:
            out = self._buf(tag + "out", (M, A))
        C.jb_dueling_fwd(ptr(a), ptr(v), M, A, 1, ptr(out), s)
        self._saved[tag] = (B, N)
        return out

    def forward(self, x, tau, is_train=True, tag="t.", noise=None):
        """x [B, ...] device rows, tau [B, N] f32 fractions -> [B*N, A] (row b*N + n: fraction n of state b)."""
        return self._body(x, tau, self._make_noise(tag, is_train, noise), tag, None, True)

    def forward_rows(self, x, tau, out, is_train=True, noise=None):
        """Inference over many rows (act()): one noise draw for the whole call, then chunks of rows * N sized like IQN's
        (ROW_BYTES_PER_PASS of [rows*N, Dh] activation), every chunk on the same effective weights."""
        M, N = tau.shape
        wb = self._make_noise("inf.", is_train, noise)
        per = max(1, min(self.head.max_rows, ROW_BYTES_PER_PASS // (4 * self.head.D_head_out * N)))
        for s in range(0, M, per):
            e = min(M, s + per)
            self._body(x[s:e], tau[s:e], wb, f"inf{e - s}.", out[s * N:e * N], False)
        return out

    def backward(self, dout, tag="t."):
        """dout [B*N, A] = d loss / d forward output; fills self.grad (overwrites)."""
        B, N = self._saved[tag]
        M, p, g, Dh, H, A, s = B * N, self.p, self.g, self.head.D_head_out, self.D_hidden, self.D_out, stream_ptr()
        psi = self._buf(tag + "head.h", (B, Dh))
        c = self._buf(tag + "cos", (M, self.D_em))
        phi = self._buf(tag + "phi", (M, Dh))
        z = self._buf(tag + "z", (M, Dh))
        f = self._buf(tag + "f", (M, H))
        xa = self._buf(tag + "xa", (M, H)); xv = self._buf(tag + "xv", (M, H))
        da = self._buf(tag + "da", (M, A)); dv = self._buf(tag + "dv", (M, 1))
        C.jb_dueling_bwd(ptr(dout), M, A, 1, ptr(da), ptr(dv), s)
        dxa = self._buf(tag + "dxa", (M, H)); dxv = self._buf(tag + "dxv", (M, H))
        self._noisy_bwd(da, xa, tag, "_a2", H, A, dxa, xa)
        self._noisy_bwd(dv, xv, tag, "_v2", H, 1, dxv, xv)
        df = self._buf(tag + "df", (M, H)); df2 = self._buf(tag + "df2", (M, H))
        self._noisy_bwd(dxa, f, tag, "_a1", H, H, df, f)
        self._noisy_bwd(dxv, f, tag, "_v1", H, H, df2, f)
        df.add_(df2)
        L.linear_bwd_dw(df, z, g["l.weight"], g["l.bias"])
        dz = self._buf(tag + "dz", (M, Dh))
        L.linear_bwd_dx(df, p["l.weight"], dz)
        dpsi = self._buf(tag + "dpsi", (B, Dh)); dpre = self._buf(tag + "dpre", (M, Dh))
        C.jb_iqn_mul_bwd(ptr(dz), ptr(psi), ptr(phi), B, N, Dh, ptr(dpsi), ptr(dpre), s)
        L.linear_bwd_dw(dpre, c, g["sample_embed.weight"], g["sample_embed.bias"])
        self.head.backward(self, dpsi, B, tag)
