"""NoisyNet networks: `Noisy` (jorldy/core/network/noisy.py:8-50) and the Rainbow network
(jorldy/core/network/rainbow.py:8-94: head -> l -> noisy dueling streams over N_atom atoms).

Noisy tensors keep the reference layout (in, out) and parameter order (the direct nn.Parameters
precede the sub-modules in state_dict(), SURVEY.md Appendix B).  Every forward draws fresh factor
noise (utils.py:59-68) through jb_noisy_make — Philox stream = layer index, device-side draw
counter — or takes injected normals `noise=[(eps_i, eps_j), ...]` for parity tests.  forward_rows
(act()) draws once per call and runs every chunk of rows on those weights.
"""
import torch

from ..dev import C, ptr, stream_ptr
from .base import FlatNetwork, init_gain, orthogonal_
from .head import make_head
from . import layers as L


def _noisy_specs(tag, in_f, out_f):
    return [(f"mu_w{tag}", (in_f, out_f)), (f"sig_w{tag}", (in_f, out_f)), (f"mu_b{tag}", (out_f,)),
            (f"sig_b{tag}", (out_f,))]


def _noisy_init(p, tag, in_f, out_f, noise_type, gen):
    """utils.py:89-105 init_weights."""
    if noise_type == "factorized":
        mu_init, sig_init = 1.0 / (in_f ** 0.5), 0.5 / (in_f ** 0.5)
    else:
        mu_init, sig_init = (3.0 / in_f) ** 0.5, 0.017
    p[f"mu_w{tag}"].copy_((torch.rand((in_f, out_f), generator=gen) * 2 - 1) * mu_init)
    p[f"mu_b{tag}"].copy_((torch.rand((out_f,), generator=gen) * 2 - 1) * mu_init)
    p[f"sig_w{tag}"].fill_(sig_init)
    p[f"sig_b{tag}"].fill_(sig_init)


class _NoisyMixin:
    def _noisy_setup(self, noise_type, seed):
        if noise_type != "factorized":
            raise NotImplementedError("hot-path configs use factorized noise (config/noisy, config/rainbow)")
        self.noise_type = noise_type
        self.noise_seed = int(seed) if seed is not None else 0
        self._draw_ctr = torch.zeros(1, dtype=torch.int64, device=self.device)

    def _noisy_make(self, tag, lt, layer_id, in_f, out_f, is_train, noise):
        """Draws one layer's factors (or takes injected normals) and returns its effective (W, b), kept under `tag+lt`."""
        p = self.p
        fi = self._buf(tag + lt + ".fi", (in_f,)); fj = self._buf(tag + lt + ".fj", (out_f,))
        w = self._buf(tag + lt + ".w", (in_f, out_f)); b = self._buf(tag + lt + ".b", (out_f,))
        ei, ej = (noise if noise is not None else (None, None))
        C.jb_noisy_make(ptr(p[f"mu_w{lt}"]), ptr(p[f"sig_w{lt}"]), ptr(p[f"mu_b{lt}"]), ptr(p[f"sig_b{lt}"]), in_f, out_f,
                        ptr(ei), ptr(ej), self.noise_seed, layer_id, ptr(self._draw_ctr), int(is_train), ptr(fi), ptr(fj),
                        ptr(w), ptr(b), stream_ptr())
        return w, b

    def _noisy_bwd(self, dy, x, tag, lt, in_f, out_f, dx, relu_act):
        """Gradients of one noisy layer: fills g[mu/sig], returns dx (masked by relu_act>0) if dx given."""
        g = self.g
        w = self._buf(tag + lt + ".w", (in_f, out_f))
        fi = self._buf(tag + lt + ".fi", (in_f,)); fj = self._buf(tag + lt + ".fj", (out_f,))
        dw = self._buf(tag + lt + ".dw", (in_f, out_f)); db = self._buf(tag + lt + ".db", (out_f,))
        L.linear_io_bwd_dw(dy, x, dw, db)
        C.jb_noisy_grad(ptr(dw), ptr(db), ptr(fi), ptr(fj), in_f, out_f, ptr(g[f"mu_w{lt}"]), ptr(g[f"sig_w{lt}"]),
                        ptr(g[f"mu_b{lt}"]), ptr(g[f"sig_b{lt}"]), stream_ptr())
        if dx is not None:
            L.linear_io_bwd_dx(dy, w, dx, relu_act=relu_act)


class Noisy(FlatNetwork, _NoisyMixin):
    def __init__(self, D_in, D_out, noise_type="factorized", D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        assert noise_type in ["independent", "factorized"]
        self._noisy_setup(noise_type, seed)
        self.D_in, self.D_out, self.D_hidden = D_in, D_out, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        F = self.head.D_head_out
        self._specs = _noisy_specs("1", F, D_hidden) + _noisy_specs("2", D_hidden, D_out) + self.head.specs()
        self._allocate()
        self.nout = D_out
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            _noisy_init(self.p, "1", F, D_hidden, noise_type, gen)
            _noisy_init(self.p, "2", D_hidden, D_out, noise_type, gen)

    def _make_noise(self, tag, is_train, noise):
        """Effective (W, b) of the two noisy layers in call order; noise: injected [(eps_i, eps_j)] x 2."""
        F, H, A = self.head.D_head_out, self.D_hidden, self.D_out
        n1, n2 = noise if noise is not None else (None, None)
        return {"1": self._noisy_make(tag, "1", 1, F, H, is_train, n1), "2": self._noisy_make(tag, "2", 2, H, A, is_train, n2)}

    def _body(self, x, idx, M, wb, tag, out, save):
        feat = self.head.forward(self, x, idx, M, tag, save)
        h = self._buf(tag + "h", (M, self.D_hidden))
        L.linear_io_fwd(feat, *wb["1"], h, relu=True)
        if out is None:
            out = self._buf(tag + "q", (M, self.D_out))
        L.linear_io_fwd(h, *wb["2"], out, relu=False)
        return out

    def forward(self, x, is_train=True, idx=None, M=None, out=None, tag="t.", save=True, noise=None):
        M = M if M is not None else (idx.shape[0] if idx is not None else x.shape[0])
        return self._body(x, idx, M, self._make_noise(tag, is_train, noise), tag, out, save)

    def forward_rows(self, x, out, is_train=True, noise=None):
        """Chunked inference (act() over many env rows): one noise draw for the whole call, every chunk on the same
        effective weights, as the reference's act() draws once per call."""
        M = x.shape[0]
        wb = self._make_noise("inf.", is_train, noise)
        for s in range(0, M, self.head.max_rows):
            e = min(M, s + self.head.max_rows)
            self._body(x[s:e], None, e - s, wb, f"inf{e - s}.", out[s:e], False)
        return out

    def backward(self, dq, M, tag="t."):
        F, H, A = self.head.D_head_out, self.D_hidden, self.D_out
        feat = self._buf(tag + "head.h", (M, F)); h = self._buf(tag + "h", (M, H))
        dh = self._buf(tag + "dh", (M, H)); dfeat = self._buf(tag + "dfeat", (M, F))
        self._noisy_bwd(dq, h, tag, "2", H, A, dh, h)
        self._noisy_bwd(dh, feat, tag, "1", F, H, dfeat, feat)
        self.head.backward(self, dfeat, M, tag)

    def get_sig_w_mean(self):
        return torch.abs(self.p["sig_w1"]).mean(), torch.abs(self.p["sig_w2"]).mean()


class Rainbow(FlatNetwork, _NoisyMixin):
    def __init__(self, D_in, D_out, N_atom, noise_type="factorized", D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        self._noisy_setup(noise_type, seed)
        self.D_in, self.D_out, self.N_atom, self.D_hidden = D_in, D_out, N_atom, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        F, H = self.head.D_head_out, D_hidden
        self._specs = (_noisy_specs("_a1", H, H) + _noisy_specs("_v1", H, H) + _noisy_specs("_a2", H, N_atom * D_out)
                       + _noisy_specs("_v2", H, N_atom) + self.head.specs() + [("l.weight", (H, F)), ("l.bias", (H,))])
        self._allocate()
        self.nout = D_out * N_atom
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            self.p["l.weight"].copy_(orthogonal_((H, F), init_gain("relu"), gen))
            _noisy_init(self.p, "_a1", H, H, noise_type, gen)
            _noisy_init(self.p, "_v1", H, H, noise_type, gen)
            _noisy_init(self.p, "_a2", H, N_atom * D_out, noise_type, gen)
            _noisy_init(self.p, "_v2", H, N_atom, noise_type, gen)

    def _make_noise(self, tag, is_train, noise):
        """Effective (W, b) of the four noisy layers in the reference's call order a1, v1, a2, v2 (Philox streams 1..4);
        noise: injected [(eps_i, eps_j)] x 4."""
        H, AK, K = self.D_hidden, self.D_out * self.N_atom, self.N_atom
        dims = (("_a1", 1, H, H), ("_v1", 2, H, H), ("_a2", 3, H, AK), ("_v2", 4, H, K))
        noise = noise if noise is not None else (None,) * 4
        return {lt: self._noisy_make(tag, lt, lid, i, o, is_train, nz) for (lt, lid, i, o), nz in zip(dims, noise)}

    def _body(self, x, idx, M, wb, tag, out, save):
        H, A, K = self.D_hidden, self.D_out, self.N_atom
        feat = self.head.forward(self, x, idx, M, tag, save)
        f = self._buf(tag + "f", (M, H))
        L.linear_fwd(feat, self.p["l.weight"], self.p["l.bias"], f, relu=True)
        xa = self._buf(tag + "xa", (M, H)); xv = self._buf(tag + "xv", (M, H))
        L.linear_io_fwd(f, *wb["_a1"], xa, relu=True)
        L.linear_io_fwd(f, *wb["_v1"], xv, relu=True)
        a = self._buf(tag + "a", (M, A * K)); v = self._buf(tag + "v", (M, K))
        L.linear_io_fwd(xa, *wb["_a2"], a, relu=False)
        L.linear_io_fwd(xv, *wb["_v2"], v, relu=False)
        if out is None:
            out = self._buf(tag + "logits", (M, A, K))
        C.jb_dueling_fwd(ptr(a), ptr(v), M, A, K, ptr(out), stream_ptr())
        return out

    def forward(self, x, is_train=True, idx=None, M=None, out=None, tag="t.", save=True, noise=None):
        """Returns logits [M, A, K].  noise order = the reference's call order: a1, v1, a2, v2."""
        M = M if M is not None else (idx.shape[0] if idx is not None else x.shape[0])
        return self._body(x, idx, M, self._make_noise(tag, is_train, noise), tag, out, save)

    def forward_rows(self, x, out, is_train=True, noise=None):
        """Chunked inference (act() over many env rows); out [M, A, K].  One noise draw for the whole call, every chunk
        on the same effective weights (the reference's act() draws once per call).  noise: injected draws (parity tests)."""
        M = x.shape[0]
        wb = self._make_noise("inf.", is_train, noise)
        for s in range(0, M, self.head.max_rows):
            e = min(M, s + self.head.max_rows)
            self._body(x[s:e], None, e - s, wb, f"inf{e - s}.", out[s:e], False)
        return out

    def backward(self, dlogits, M, tag="t."):
        H, A, K = self.D_hidden, self.D_out, self.N_atom
        F = self.head.D_head_out
        feat = self._buf(tag + "head.h", (M, F)); f = self._buf(tag + "f", (M, H))
        xa = self._buf(tag + "xa", (M, H)); xv = self._buf(tag + "xv", (M, H))
        da = self._buf(tag + "da", (M, A * K)); dv = self._buf(tag + "dv", (M, K))
        C.jb_dueling_bwd(ptr(dlogits), M, A, K, ptr(da), ptr(dv), stream_ptr())
        dxa = self._buf(tag + "dxa", (M, H)); dxv = self._buf(tag + "dxv", (M, H))
        self._noisy_bwd(da, xa, tag, "_a2", H, A * K, dxa, xa)
        self._noisy_bwd(dv, xv, tag, "_v2", H, K, dxv, xv)
        df = self._buf(tag + "df", (M, H)); df2 = self._buf(tag + "df2", (M, H))
        self._noisy_bwd(dxa, f, tag, "_a1", H, H, df, f)
        self._noisy_bwd(dxv, f, tag, "_v1", H, H, df2, f)
        df.add_(df2)
        L.linear_bwd_dw(df, feat, self.g["l.weight"], self.g["l.bias"])
        dfeat = self._buf(tag + "dfeat", (M, F))
        L.linear_bwd_dx(df, self.p["l.weight"], dfeat, relu_act=feat)
        self.head.backward(self, dfeat, M, tag)
