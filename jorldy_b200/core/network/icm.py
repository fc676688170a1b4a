"""ICM network (Pathak et al., ICML 2017) for ICM-PPO: an encoder phi, a forward model and an inverse model.

    phi(x) = elu(fc2(elu(BN(fc1(norm(x))))))         fc1 / fc2 shared by s and s'; BN = bn1 on s, bn1_next on s'
    f      = fc_f2([relu(fc_f1([phi(s), a])), a])    a: one-hot (discrete) or the raw action (continuous)
    g      = pi(relu(inv([phi(s), phi(s')])))

`icm_cnn` puts the CNN head's trunk (head.py CNNHead: /255, three ReLU convolutions, conv1's im2col read straight from
the frame ring for frame-reference rows) in front of fc1 in place of norm(x); the rest is the same.

Both BatchNorm1d layers always run in training mode (batch statistics, running buffers updated), as the reference's
module is never put in eval mode; batch_norm=False drops them.  norm(x) is the observation RunningMeanStd's clipped
standardisation (agent-owned state), or the identity.

Layout: the s and s' rows are stacked [s; s'] through fc1 and fc2 (one GEMM each, so the shared weights' gradients are
one product); BatchNorm and the ELUs run per half.  phi(s) and phi(s') are written side by side into `pp` [M, 2F] (the
inverse model's input) and phi(s) also into the first F columns of `fa` [M, F + A] (the forward model's input), whose
last A columns hold the action rows; `ha` [M, H + A] holds [relu(fc_f1(fa)), a].  The concatenations are never copied.
"""
import math
from collections import OrderedDict

import torch

from ..dev import C, ptr, stream_ptr
from . import layers as L
from .base import FlatNetwork
from .head import CNNHead

FEATURE = 256      # F, csrc/icm.cu ICM_F
HIDDEN = 256
BN_EPS, BN_MOMENTUM = 1e-5, 0.1
OBS_CLIP = 5.0


class BatchNormNetwork(FlatNetwork):
    """A flat network with training-mode BatchNorm1d layers (csrc/icm.cu jb_bn_elu_fwd / _bwd, width HIDDEN): their
    running buffers live in `self.buffers`, and state_dict puts each layer's buffers after its bias, in torch's module
    order.  Shared by the ICM and the RND predictor."""

    def state_dict(self):
        out = OrderedDict()
        for k, v in self.p.items():
            out[k] = v.detach().clone()
            if k.startswith("bn") and k.endswith(".bias"):
                bn = k[:-len(".bias")]
                for b in ("running_mean", "running_var", "num_batches_tracked"):
                    out[f"{bn}.{b}"] = self.buffers[f"{bn}.{b}"].clone()
        return out

    def load_state_dict(self, sd):
        sd = dict(sd)
        bufs = {k: sd.pop(k) for k in list(sd) if k in self.buffers}
        missing = [k for k in self.buffers if k not in bufs]
        if missing:
            raise KeyError(f"state_dict mismatch: missing {missing}")
        super().load_state_dict(sd)
        for k, v in bufs.items():
            self.buffers[k].copy_(torch.as_tensor(v).to(self.buffers[k].dtype).reshape(self.buffers[k].shape))

    def buffer_tensors(self):
        return list(self.buffers.values())

    def _bn_args(self, bn, M, tag):
        if not self.batch_norm:
            return [0] * 9
        H = HIDDEN
        b = self.buffers
        return [ptr(self.p[f"{bn}.weight"]), ptr(self.p[f"{bn}.bias"]), ptr(b[f"{bn}.running_mean"]),
                ptr(b[f"{bn}.running_var"]), ptr(b[f"{bn}.num_batches_tracked"]), BN_MOMENTUM, BN_EPS,
                ptr(self._buf(tag + bn + ".mean", (H,))), ptr(self._buf(tag + bn + ".invstd", (H,)))]

    def _partials(self, M, N, tag):
        return self._buf(tag + "partials", (C.jb_col_partials_doubles(M, N),), torch.float64)


class ICM_MLP(BatchNormNetwork):
    """`cnn` = True: D_in is the frame stack's [C, H, W] and the CNN trunk feeds fc1 (icm_cnn)."""

    def __init__(self, D_in, D_out, action_type, batch_norm=True, device=None, seed=None, cnn=False):
        super().__init__(device)
        self.head = CNNHead(tuple(D_in)) if cnn else None
        self.D_in = self.head.D_head_out if cnn else int(D_in)      # fc1's input width
        self.A, self.continuous, self.batch_norm = int(D_out), action_type == "continuous", batch_norm
        F, H, A = FEATURE, HIDDEN, self.A
        self._linears = [("fc1", H, self.D_in), ("fc2", F, H), ("fc_f1", H, F + A), ("fc_f2", F, H + A),
                         ("inv", H, 2 * F), ("pi", A, H)]
        specs = (self.head.specs() if cnn else []) + [("fc1.weight", (H, self.D_in)), ("fc1.bias", (H,))]
        if batch_norm:
            specs += [("bn1.weight", (H,)), ("bn1.bias", (H,)), ("bn1_next.weight", (H,)), ("bn1_next.bias", (H,))]
        for name, o, i in self._linears[1:]:
            specs += [(f"{name}.weight", (o, i)), (f"{name}.bias", (o,))]
        self._specs = specs
        self._allocate()
        # torch.nn.Linear's default init (kaiming_uniform_(a=sqrt(5)) = U(+-1/sqrt(fan_in)), bias the same), BN (1, 0)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        with torch.no_grad():
            if cnn:
                self.head.init(self.p, gen)
            for name, o, i in self._linears:
                bound = 1.0 / math.sqrt(i)
                for suffix, shape in (("weight", (o, i)), ("bias", (o,))):
                    self.p[f"{name}.{suffix}"].copy_(torch.rand(shape, generator=gen) * (2 * bound) - bound)
            if batch_norm:
                for bn in ("bn1", "bn1_next"):
                    self.p[f"{bn}.weight"].fill_(1.0)
        self.buffers = OrderedDict()
        if batch_norm:
            for bn in ("bn1", "bn1_next"):
                self.buffers[f"{bn}.running_mean"] = torch.zeros(H, device=self.device)
                self.buffers[f"{bn}.running_var"] = torch.ones(H, device=self.device)
                self.buffers[f"{bn}.num_batches_tracked"] = torch.zeros((), dtype=torch.int64, device=self.device)

    def _stacked_rows(self, s, s_next, idx, M, tag):
        """The CNN trunk's input: the rows idx of s, then those of s_next, as one row source of 2M stacks (frame
        references when s / s_next are FrameRows on one ring, uint8 stacks otherwise)."""
        if torch.is_tensor(s):
            x = self._buf(tag + "stack", (2 * M,) + tuple(self.head.D_in), torch.uint8)
            for h, src in enumerate((s, s_next)):
                src = src.view(src.shape[0], *self.head.D_in)
                x[h * M:(h + 1) * M].copy_(src[:M] if idx is None else src.index_select(0, idx.to(torch.int64)))
            return x
        if s.store is not s_next.store:
            raise ValueError("the states and next states must reference the same frame ring")
        refs = self._buf(tag + "refs", (2 * M,), torch.int64)
        for h, src in enumerate((s, s_next)):
            if idx is None:
                refs[h * M:(h + 1) * M].copy_(src.refs[:M])
            else:
                torch.index_select(src.refs, 0, idx, out=refs[h * M:(h + 1) * M])
        return type(s)(s.store, refs)

    def forward(self, s, s_next, action, idx, M, rms=None, inverse=True, tag="icm.", chunk_rows=None):
        """s / s_next: [rows, D] f32 device tensors (icm_cnn: uint8 stacks or FrameRows), rows idx[M] (idx None: the
        first M rows); rms = (mean, var) float64 observation statistics or None (icm_mlp only).  chunk_rows: run the CNN
        trunk in chunks of that many rows (no backward then).  Returns (f [M, F], phi(s') as a strided [M, F] view,
        g [M, A] or None)."""
        F, H, A, D = FEATURE, HIDDEN, self.A, self.D_in
        s_ = stream_ptr()
        X = self._buf(tag + "x", (2 * M, D))
        if self.head is not None:
            rows = self._stacked_rows(s, s_next, idx, M, tag)
            step = chunk_rows or 2 * M
            for a in range(0, 2 * M, step):
                b = min(2 * M, a + step)
                self.head.forward(self, rows[a:b], None, b - a, tag if step == 2 * M else f"{tag}c{b - a}.", step == 2 * M,
                                  out=X[a:b])
        else:
            mean, var = (ptr(rms[0]), ptr(rms[1])) if rms is not None else (0, 0)
            for h, src in enumerate((s, s_next)):
                C.jb_rms_normalize(ptr(src), ptr(idx), M, D, mean, var, OBS_CLIP, ptr(X[h * M:]), s_)
        z1 = self._buf(tag + "z1", (2 * M, H))
        L.linear_fwd(X, self.p["fc1.weight"], self.p["fc1.bias"], z1, relu=False)
        a1 = self._buf(tag + "a1", (2 * M, H))
        if self.batch_norm:
            part = self._partials(M, H, tag)
            for h, bn in enumerate(("bn1", "bn1_next")):
                C.jb_bn_elu_fwd(ptr(z1[h * M:]), M, H, *self._bn_args(bn, M, tag), ptr(part), ptr(a1[h * M:]), H, 0, 0, s_)
        else:
            C.jb_bn_elu_fwd(ptr(z1), 2 * M, H, *self._bn_args(None, M, tag), 0, ptr(a1), H, 0, 0, s_)
        z2 = self._buf(tag + "z2", (2 * M, F))
        L.linear_fwd(a1, self.p["fc2.weight"], self.p["fc2.bias"], z2, relu=False)
        pp = self._buf(tag + "pp", (M, 2 * F))
        fa = self._buf(tag + "fa", (M, F + A))
        ha = self._buf(tag + "ha", (M, H + A))
        none = [0] * 9
        C.jb_bn_elu_fwd(ptr(z2), M, F, *none, 0, ptr(pp), 2 * F, ptr(fa), F + A, s_)
        C.jb_bn_elu_fwd(ptr(z2[M:]), M, F, *none, 0, ptr(pp[:, F:]), 2 * F, 0, 0, s_)
        C.jb_icm_action_rows(int(self.continuous), ptr(action), ptr(idx), M, A, ptr(fa[:, F:]), F + A, s_)
        C.jb_icm_action_rows(int(self.continuous), ptr(action), ptr(idx), M, A, ptr(ha[:, H:]), H + A, s_)
        C.jb_gemm(ptr(fa), F + A, 1, ptr(self.p["fc_f1.weight"]), F + A, 1, ptr(ha), H + A, M, H, F + A,
                  ptr(self.p["fc_f1.bias"]), 1, 0, 0, 0, 0, s_)
        f = self._buf(tag + "f", (M, F))
        L.linear_fwd(ha, self.p["fc_f2.weight"], self.p["fc_f2.bias"], f, relu=False)
        g = None
        if inverse:
            hi = self._buf(tag + "hi", (M, H))
            L.linear_fwd(pp, self.p["inv.weight"], self.p["inv.bias"], hi, relu=True)
            g = self._buf(tag + "g", (M, A))
            L.linear_fwd(hi, self.p["pi.weight"], self.p["pi.bias"], g, relu=False)
        return f, pp[:, F:], g

    def backward(self, df, dg, M, tag="icm."):
        """df [M, F] = d loss / d f, dg [M, A] = d loss / d g of the last forward(tag); fills self.grad (overwrites)."""
        F, H, A = FEATURE, HIDDEN, self.A
        s_ = stream_ptr()
        p, gr = self.p, self.g
        X, z1, a1 = self._buf(tag + "x", (2 * M, self.D_in)), self._buf(tag + "z1", (2 * M, H)), self._buf(tag + "a1", (2 * M, H))
        pp, fa, ha = self._buf(tag + "pp", (M, 2 * F)), self._buf(tag + "fa", (M, F + A)), self._buf(tag + "ha", (M, H + A))
        hi = self._buf(tag + "hi", (M, H))
        # inverse model
        dhi = self._buf(tag + "dhi", (M, H))
        L.linear_bwd_dw(dg, hi, gr["pi.weight"], gr["pi.bias"])
        L.linear_bwd_dx(dg, p["pi.weight"], dhi, relu_act=hi)
        L.linear_bwd_dw(dhi, pp, gr["inv.weight"], gr["inv.bias"])
        dpp = self._buf(tag + "dpp", (M, 2 * F))
        L.linear_bwd_dx(dhi, p["inv.weight"], dpp)
        # forward model: d relu(fc_f1) from fc_f2's first H input columns, then d phi(s) added into dpp[:, :F]
        L.linear_bwd_dw(df, ha, gr["fc_f2.weight"], gr["fc_f2.bias"])
        dh = self._buf(tag + "dh", (M, H))
        C.jb_gemm(ptr(df), F, 1, ptr(p["fc_f2.weight"]), H + A, 0, ptr(dh), H, M, H, F, 0, 0, ptr(ha), H + A, 0, 0, s_)
        L.linear_bwd_dw(dh, fa, gr["fc_f1.weight"], gr["fc_f1.bias"])
        C.jb_gemm(ptr(dh), H, 1, ptr(p["fc_f1.weight"]), F + A, 0, ptr(dpp), 2 * F, M, F, H, 0, 0, 0, 0, 0, 1, s_)
        # encoder
        dz2 = self._buf(tag + "dz2", (2 * M, F))
        for h in range(2):
            C.jb_bn_elu_bwd(ptr(dpp[:, h * F:]), 2 * F, ptr(pp[:, h * F:]), 2 * F, 0, M, F, 0, 0, 0, 0, 0,
                            ptr(dz2[h * M:]), 0, 0, s_)
        L.linear_bwd_dw(dz2, a1, gr["fc2.weight"], gr["fc2.bias"])
        da1 = self._buf(tag + "da1", (2 * M, H))
        L.linear_bwd_dx(dz2, p["fc2.weight"], da1)
        dz1 = self._buf(tag + "dz1", (2 * M, H))
        if self.batch_norm:
            part = self._partials(M, H, tag)
            xhat = self._buf(tag + "xhat", (M, H))
            for h, bn in enumerate(("bn1", "bn1_next")):
                C.jb_bn_elu_bwd(ptr(da1[h * M:]), H, ptr(a1[h * M:]), H, ptr(z1[h * M:]), M, H, ptr(p[f"{bn}.weight"]),
                                ptr(self._buf(tag + bn + ".mean", (H,))), ptr(self._buf(tag + bn + ".invstd", (H,))),
                                ptr(xhat), ptr(part), ptr(dz1[h * M:]), ptr(gr[f"{bn}.weight"]), ptr(gr[f"{bn}.bias"]), s_)
        else:
            C.jb_bn_elu_bwd(ptr(da1), H, ptr(a1), H, 0, 2 * M, H, 0, 0, 0, 0, 0, ptr(dz1), 0, 0, s_)
        L.linear_bwd_dw(dz1, X, gr["fc1.weight"], gr["fc1.bias"])
        if self.head is not None:
            dX = self._buf(tag + "dx", (2 * M, self.D_in))
            L.linear_bwd_dx(dz1, p["fc1.weight"], dX, relu_act=X)         # X is the trunk's ReLU output
            self.head.backward(self, dX, 2 * M, tag)
