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


def dueling_layers(H, A, K):
    """The noisy dueling streams' layer table: a1, v1 [H -> H], a2 [H -> A*K], v2 [H -> K] in the reference's call order,
    on Philox streams 1..4."""
    return (("_a1", 1, H, H), ("_v1", 2, H, H), ("_a2", 3, H, A * K), ("_v2", 4, H, K))


class _NoisyMixin:
    """A network's noisy layers, listed once in self._noisy as (tag, Philox stream, in, out) in the order the reference
    calls them.  That table gives their parameter specs (first in state_dict), their init (the generator's last draws)
    and their noise draws; forward / forward_rows run the network's _body on the effective weights of one draw."""

    def _noisy_setup(self, noise_type, seed):
        if noise_type != "factorized":
            raise NotImplementedError("hot-path configs use factorized noise (config/noisy, config/rainbow)")
        self.noise_type = noise_type
        self.noise_seed = int(seed) if seed is not None else 0
        self._draw_ctr = torch.zeros(1, dtype=torch.int64, device=self.device)

    def _noisy_param_specs(self):
        return [spec for lt, _, i, o in self._noisy for spec in _noisy_specs(lt, i, o)]

    def _noisy_init_params(self, gen):
        for lt, _, i, o in self._noisy:
            _noisy_init(self.p, lt, i, o, self.noise_type, gen)

    def _make_noise(self, tag, is_train, noise):
        """Effective (W, b) of every noisy layer, drawn in table order; noise: injected [(eps_i, eps_j)] per layer."""
        noise = noise if noise is not None else (None,) * len(self._noisy)
        return {lt: self._noisy_make(tag, lt, lid, i, o, is_train, nz) for (lt, lid, i, o), nz in zip(self._noisy, noise)}

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


def streams_fwd(net, f, M, A, K, wb, tag, out):
    """out [M, A, K] = v + a - mean_a a of the noisy dueling streams on f [M, H] (K = 1: one Q per action), with the
    effective weights wb; the activations stay under `tag` for streams_bwd."""
    H = net.D_hidden
    xa = net._buf(tag + "xa", (M, H)); xv = net._buf(tag + "xv", (M, H))
    L.linear_io_fwd(f, *wb["_a1"], xa, relu=True)
    L.linear_io_fwd(f, *wb["_v1"], xv, relu=True)
    a = net._buf(tag + "a", (M, A * K)); v = net._buf(tag + "v", (M, K))
    L.linear_io_fwd(xa, *wb["_a2"], a, relu=False)
    L.linear_io_fwd(xv, *wb["_v2"], v, relu=False)
    C.jb_dueling_fwd(ptr(a), ptr(v), M, A, K, ptr(out), stream_ptr())
    return out


def streams_bwd(net, dout, f, M, A, K, tag):
    """Writes the four noisy layers' gradients from dout [M, A, K] and returns d loss / d f [M, H] (masked by f > 0)."""
    H = net.D_hidden
    xa = net._buf(tag + "xa", (M, H)); xv = net._buf(tag + "xv", (M, H))
    da = net._buf(tag + "da", (M, A * K)); dv = net._buf(tag + "dv", (M, K))
    C.jb_dueling_bwd(ptr(dout), M, A, K, ptr(da), ptr(dv), stream_ptr())
    dxa = net._buf(tag + "dxa", (M, H)); dxv = net._buf(tag + "dxv", (M, H))
    net._noisy_bwd(da, xa, tag, "_a2", H, A * K, dxa, xa)
    net._noisy_bwd(dv, xv, tag, "_v2", H, K, dxv, xv)
    df = net._buf(tag + "df", (M, H)); df2 = net._buf(tag + "df2", (M, H))
    net._noisy_bwd(dxa, f, tag, "_a1", H, H, df, f)
    net._noisy_bwd(dxv, f, tag, "_v1", H, H, df2, f)
    df.add_(df2)
    return df


class Noisy(FlatNetwork, _NoisyMixin):
    def __init__(self, D_in, D_out, noise_type="factorized", D_hidden=512, head="mlp", device=None, seed=None):
        super().__init__(device)
        assert noise_type in ["independent", "factorized"]
        self._noisy_setup(noise_type, seed)
        self.D_in, self.D_out, self.D_hidden = D_in, D_out, D_hidden
        self.head = make_head(head, D_in, D_hidden)
        self._noisy = (("1", 1, self.head.D_head_out, D_hidden), ("2", 2, D_hidden, D_out))
        self._specs = self._noisy_param_specs() + self.head.specs()
        self._allocate()
        self.nout = D_out
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            self._noisy_init_params(gen)

    def _body(self, x, idx, M, wb, tag, out, save):
        feat = self.head.forward(self, x, idx, M, tag, save)
        h = self._buf(tag + "h", (M, self.D_hidden))
        L.linear_io_fwd(feat, *wb["1"], h, relu=True)
        if out is None:
            out = self._buf(tag + "q", (M, self.D_out))
        L.linear_io_fwd(h, *wb["2"], out, relu=False)
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
        self._noisy = dueling_layers(H, D_out, N_atom)
        self._specs = self._noisy_param_specs() + self.head.specs() + [("l.weight", (H, F)), ("l.bias", (H,))]
        self._allocate()
        self.nout = D_out * N_atom
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            self.head.init(self.p, gen)
            self.p["l.weight"].copy_(orthogonal_((H, F), init_gain("relu"), gen))
            self._noisy_init_params(gen)

    def _body(self, x, idx, M, wb, tag, out, save):
        """logits [M, A, K]"""
        H, A, K = self.D_hidden, self.D_out, self.N_atom
        feat = self.head.forward(self, x, idx, M, tag, save)
        f = self._buf(tag + "f", (M, H))
        L.linear_fwd(feat, self.p["l.weight"], self.p["l.bias"], f, relu=True)
        if out is None:
            out = self._buf(tag + "logits", (M, A, K))
        return streams_fwd(self, f, M, A, K, wb, tag, out)

    def backward(self, dlogits, M, tag="t."):
        F = self.head.D_head_out
        feat = self._buf(tag + "head.h", (M, F)); f = self._buf(tag + "f", (M, self.D_hidden))
        df = streams_bwd(self, dlogits, f, M, self.D_out, self.N_atom, tag)
        L.linear_bwd_dw(df, feat, self.g["l.weight"], self.g["l.bias"])
        dfeat = self._buf(tag + "dfeat", (M, F))
        L.linear_bwd_dx(df, self.p["l.weight"], dfeat, relu_act=feat)
        self.head.backward(self, dfeat, M, tag)
