"""RND networks (Burda et al., 2018, arXiv:1810.12894) for RND-PPO: a frozen random target and a trained predictor, both
reading the next state s'.

    x' = clip((s' - mean) / sqrt(var), +-5)           (obs_normalize; else x' = s')
    t  = fc2(elu(fc1(x')))                            target: never updated, no optimiser state
    p  = fc3(elu(fc2(elu(BN(fc1(x'))))))              predictor: BN = BatchNorm1d, always in training mode (batch
                                                      statistics, running buffers updated); batch_norm=False drops it

`rnd_cnn` gives each network its own CNN trunk (head.py CNNHead: /255, three ReLU convolutions, conv1's im2col read
straight from the frame ring for frame-reference rows) in place of x'.  Linear layers take torch.nn.Linear's default
init, as the ICM's do.  Each network is one flat buffer; `RND.state_dict()` lists the target's parameters under
`target.` and the predictor's (with the BatchNorm buffers) under `predictor.`, in torch's module order.
"""
import math
from collections import OrderedDict

import torch

from ..dev import C, ptr, stream_ptr
from . import layers as L
from .head import CNNHead
from .icm import BatchNormNetwork, HIDDEN, OBS_CLIP

FEATURE = 256      # F, csrc/rnd.cu RND_F
_NO_BN = [0] * 9


class _Branch(BatchNormNetwork):
    """One RND network: [CNN trunk] then the linear layers `linears` [(name, out, in)], BatchNorm after fc1 if bn."""

    def __init__(self, D_in, linears, bn, cnn, device, gen):
        super().__init__(device)
        self.head = CNNHead(tuple(D_in)) if cnn else None
        self.D_in = self.head.D_head_out if cnn else int(D_in)
        self.batch_norm = bn
        self._linears = [(name, o, self.D_in if name == "fc1" else i) for name, o, i in linears]
        specs = self.head.specs() if cnn else []
        for name, o, i in self._linears:
            specs += [(f"{name}.weight", (o, i)), (f"{name}.bias", (o,))]
            if name == "fc1" and bn:
                specs += [("bn1.weight", (o,)), ("bn1.bias", (o,))]
        self._specs = specs
        self._allocate()
        with torch.no_grad():
            if cnn:
                self.head.init(self.p, gen)
            for name, o, i in self._linears:
                bound = 1.0 / math.sqrt(i)
                for suffix, shape in (("weight", (o, i)), ("bias", (o,))):
                    self.p[f"{name}.{suffix}"].copy_(torch.rand(shape, generator=gen) * (2 * bound) - bound)
            if bn:
                self.p["bn1.weight"].fill_(1.0)
        self.buffers = OrderedDict()
        if bn:
            self.buffers["bn1.running_mean"] = torch.zeros(HIDDEN, device=self.device)
            self.buffers["bn1.running_var"] = torch.ones(HIDDEN, device=self.device)
            self.buffers["bn1.num_batches_tracked"] = torch.zeros((), dtype=torch.int64, device=self.device)

    def inputs(self, src, idx, M, rms, tag, chunk_rows=None):
        """x' of the rows idx[M] of src (idx None: the first M rows) into the tag's [M, D_in] workspace.  src: [rows, D]
        f32 (rnd_mlp), uint8 stacks or FrameRows (rnd_cnn).  chunk_rows: run the CNN trunk in chunks (no backward)."""
        X = self._buf(tag + "x", (M, self.D_in))
        if self.head is None:
            mean, var = (ptr(rms[0]), ptr(rms[1])) if rms is not None else (0, 0)
            C.jb_rms_normalize(ptr(src), ptr(idx), M, self.D_in, mean, var, OBS_CLIP, ptr(X), stream_ptr())
            return X
        if torch.is_tensor(src):
            src = src.view(src.shape[0], *self.head.D_in)
        step = chunk_rows or M
        for a in range(0, M, step):
            b = min(M, a + step)
            whole = step == M
            self.head.forward(self, src if whole else src[a:b], idx, b - a, tag if whole else f"{tag}c{b - a}.", whole,
                              out=X[a:b])
        return X

    def forward(self, X, M, tag, out=None):
        """The linear stack on X [M, D_in]; returns the [M, F] output (out, or the tag's workspace)."""
        s_ = stream_ptr()
        H = HIDDEN
        h = X
        for k, (name, o, _) in enumerate(self._linears):
            last = k == len(self._linears) - 1
            z = out if last and out is not None else self._buf(f"{tag}z{k + 1}", (M, o))
            L.linear_fwd(h, self.p[f"{name}.weight"], self.p[f"{name}.bias"], z, relu=False)
            if last:
                return z
            a = self._buf(f"{tag}a{k + 1}", (M, o))
            if k == 0 and self.batch_norm:
                C.jb_bn_elu_fwd(ptr(z), M, H, *self._bn_args("bn1", M, tag), ptr(self._partials(M, H, tag)), ptr(a), H,
                                0, 0, s_)
            else:
                C.jb_bn_elu_fwd(ptr(z), M, o, *_NO_BN, 0, ptr(a), o, 0, 0, s_)
            h = a

    def backward(self, dout, M, tag):
        """dout [M, F] = d loss / d forward(tag)'s output; fills self.grad (overwrites)."""
        s_ = stream_ptr()
        p, gr = self.p, self.g
        n = len(self._linears)
        dz = dout
        for k in range(n - 1, -1, -1):
            name, o, i = self._linears[k]
            x = self._buf(f"{tag}a{k}", (M, i)) if k > 0 else self._buf(tag + "x", (M, self.D_in))
            L.linear_bwd_dw(dz, x, gr[f"{name}.weight"], gr[f"{name}.bias"])
            if k == 0:
                break
            da = self._buf(f"{tag}da{k}", (M, i))
            L.linear_bwd_dx(dz, p[f"{name}.weight"], da)
            dzp = self._buf(f"{tag}dz{k}", (M, i))
            if k == 1 and self.batch_norm:
                H = HIDDEN
                C.jb_bn_elu_bwd(ptr(da), H, ptr(x), H, ptr(self._buf(f"{tag}z1", (M, H))), M, H, ptr(p["bn1.weight"]),
                                ptr(self._buf(tag + "bn1.mean", (H,))), ptr(self._buf(tag + "bn1.invstd", (H,))),
                                ptr(self._buf(tag + "xhat", (M, H))), ptr(self._partials(M, H, tag)), ptr(dzp),
                                ptr(gr["bn1.weight"]), ptr(gr["bn1.bias"]), s_)
            else:
                C.jb_bn_elu_bwd(ptr(da), i, ptr(x), i, 0, M, i, 0, 0, 0, 0, 0, ptr(dzp), 0, 0, s_)
            dz = dzp
        if self.head is not None:
            X = self._buf(tag + "x", (M, self.D_in))
            dX = self._buf(tag + "dx", (M, self.D_in))
            L.linear_bwd_dx(dz, p["fc1.weight"], dX, relu_act=X)          # X is the trunk's ReLU output
            self.head.backward(self, dX, M, tag)


class RND:
    """`cnn` = True: D_in is the frame stack's [C, H, W] and each network has its own CNN trunk (rnd_cnn)."""

    def __init__(self, D_in, batch_norm=True, device=None, seed=None, cnn=False):
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        F, H = FEATURE, HIDDEN
        self.target = _Branch(D_in, [("fc1", H, None), ("fc2", F, H)], False, cnn, device, gen)
        self.predictor = _Branch(D_in, [("fc1", H, None), ("fc2", H, H), ("fc3", F, H)], batch_norm, cnn, device, gen)
        self.device = self.predictor.device
        self.cnn, self.batch_norm = cnn, batch_norm
        self.D_in = self.predictor.D_in

    def parameters(self):
        """The trained parameters: the predictor's (the target is frozen)."""
        return self.predictor.parameters()

    def state_dict(self):
        out = OrderedDict()
        for prefix, net in (("target.", self.target), ("predictor.", self.predictor)):
            for k, v in net.state_dict().items():
                out[prefix + k] = v
        return out

    def load_state_dict(self, sd):
        for prefix, net in (("target.", self.target), ("predictor.", self.predictor)):
            net.load_state_dict({k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)})
        extra = [k for k in sd if not k.startswith(("target.", "predictor."))]
        if extra:
            raise KeyError(f"state_dict mismatch: unexpected {extra}")

    def buffer_tensors(self):
        return self.predictor.buffer_tensors()

    def prepass(self, s_next, NT, rms, ri):
        """Over all NT next-state rows: the target features into target_cache(NT) and r_i [NT] = mean_F (p - t)^2, with
        the predictor's BatchNorm normalising the whole rollout as one batch.  The CNN trunks run in chunks of rows."""
        chunk = self.predictor.head.max_rows if self.cnn else None       # conv1's im2col is 400 KB a row
        t = self.target_cache(NT)
        Xp = self.predictor.inputs(s_next, None, NT, rms, "pre.", chunk)
        Xt = self.target.inputs(s_next, None, NT, rms, "pre.", chunk) if self.cnn else Xp
        self.target.forward(Xt, NT, "pre.", out=t)
        p = self.predictor.forward(Xp, NT, "pre.")
        C.jb_rnd_loss(ptr(p), ptr(t), 0, NT, FEATURE, ptr(ri), 0, 0, 0, stream_ptr())
        return t

    def target_cache(self, NT):
        return self.target._buf("cache", (NT, FEATURE))

    def predict(self, s_next, idx, B, rms, tag):
        X = self.predictor.inputs(s_next, idx, B, rms, tag)
        return self.predictor.forward(X, B, tag)

    def backward(self, dp, B, tag):
        self.predictor.backward(dp, B, tag)
