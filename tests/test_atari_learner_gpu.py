"""The Atari learner at the benchmark's shapes (Ape-X: dueling CNN, H=512, B=512; Rainbow: CNN, H=512, B=32) vs
float64 references: the CNN network's forward and backward, many optimizer steps on the Ape-X network's flat
buffers, and one learn() per agent.

Tolerances (u = 2^-24, the fp32 unit roundoff):
  * Network Q and gradients, normwise per tensor: max|x - ref| <= TOL_NET * max|ref|, TOL_NET = 7.7e3 u ~ 4.6e-4.
    A sign-mixed fp32 sum of n terms rounds to within ~sqrt(n) u sum|t_i| (probabilistic bound) and
    sum|t_i| <~ sqrt(n) max|ref|, i.e. ~n u max|ref| per contraction; the errors of successive layers add.  Along
    the longest path n sums to 7.7e3: forward 256 + 512 + 576 + 3136 + 512 (conv1..3, l1, l2), backward
    4 + 2 * 512 + 64 + 64 (heads, l1 dx twice, conv3/conv2 dx) plus conv1's weight-gradient chain, at most
    204800 / 33 splits / 4 in-CTA groups = 1552 terms at B=512.  Dividing the frames by 256 instead of 255
    moves conv1's weight gradient by 3.9e-3 relative, 8x the bound.  A ReLU input within rounding of zero may
    land on either side, and then passes or blocks a whole gradient; the float64 reference therefore takes the
    kernels' ReLU masks, after checking that each disagreement sits within TOL_NET * max|pre-activation| of zero.
  * Optimizer steps, elementwise, from a float64 twin (torch.optim on the same fp32 gradients) that also tracks
    KU = 128 u of slack per update.  Per step the clip coefficient is off by <= 22 u (the norm is a sum of
    positive squares through chains of <= 41 additions), and each EMA state adds <= 3 u relative, so after 12
    steps a state is within ~80 u of its own magnitude.  A signed first moment (grad_avg, exp_avg) is bounded by
    KU times the same EMA of |g|; the centred variance s - a^2 >= (1 - W) s with W = 1 - alpha^t <= 0.114, so
    it amplifies relative error by at most 1.13x.  A parameter moves by <= 2 KU times the update's magnitude per
    step (numerator and denominator) plus u |p| for its own rounding; the bounds add over steps because p never
    feeds back into the update.  The gradient norm is compared at rtol KU.
  * learn() vs the CPU fp32 oracle: loss / max_Q / logit stats rtol 2e-5, priorities rtol 2e-4 atol 1e-6
    (test_dqn_gpu's).  Gradients rtol 2e-3 with the absolute floor raised from 2e-6 to 2 TOL_NET max|ref| per
    tensor: at B=512 the conv weight gradients contract over 25k-205k rows, both fp32 sides are only normwise
    within TOL_NET of exact, and the fp32 oracle itself differs from its float64 run by up to 5e-5 * max|ref|
    there.  Ape-X gradients are also checked normwise against a float64 oracle run at TOL_NET.  Parameters are
    checked against the float64 twin stepped with the kernel's own gradients (bounds as above), not against the
    oracle's parameters: the first RMSprop / Adam step is lr g / (c|g| + eps), which for |g| ~ eps turns a
    rounding-level gradient difference into an O(lr) parameter difference (0.24 lr between the fp32 and float64
    oracles at B=512)."""
import math

import numpy as np
import pytest
import torch

import gen_inputs as G
from helpers import q_oracle_inputs, run_q_oracle
from test_dqn_gpu import _run

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TOL_NET = 7.7e3 * U
KU = 128 * U
ALPHA, RMS_EPS, LR, CLIP = 0.99, 1.5e-7, 6.25e-5, 40.0


def _normwise(got, ref, tol, what):
    err = (got.detach().double().cpu() - ref.detach().double().cpu()).abs().max().item()
    scale = ref.detach().abs().max().item()
    assert err <= tol * scale, f"{what}: max|err| {err:.3e} > {tol:.2e} * max|ref| {scale:.3e}"


def _within(got, ref, bound, what):
    err = (got.detach().double().cpu() - ref.detach().double()).abs()
    bad = err > bound
    if bool(bad.any()):
        i = int(torch.argmax((err - bound).reshape(-1)))
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside the bound; worst |err| "
                             f"{err.reshape(-1)[i].item():.3e} vs bound {bound.reshape(-1)[i].item():.3e}")


def _dueling_cnn(shape, seed, bias_seed=None):
    """The Ape-X network; biases made nonzero so the bias epilogues are tested too."""
    from jorldy_b200.core.network.dueling import Dueling
    net = Dueling(shape, 4, 512, head="cnn", device="cuda", seed=seed)
    if bias_seed is not None:
        g = torch.Generator().manual_seed(bias_seed)
        with torch.no_grad():
            for k, v in net.p.items():
                if k.endswith(".bias"):
                    v.copy_(0.1 * torch.randn(v.shape, generator=g))
    return net


# ---- B1: CNN network forward and backward --------------------------------------------------------------------------
NET_CASES = [
    ((4, 84, 84), 1),     # one row: every conv product on the small tiles; conv1's weight gradient not split
    ((4, 84, 84), 5),     # ragged batch: conv1's weight gradient split 3 ways
    ((4, 84, 84), 32),    # Rainbow's batch: conv1's weight gradient split 25 ways
    ((4, 84, 84), 512),   # Ape-X's batch: conv1/conv2 forward and conv3/conv2 dx on the 128x64 tile, conv1 dW 33 splits
    ((3, 52, 61), 7),     # W % 4 != 0: the scalar im2col_u8 path, with a stride remainder and F = 768
]


def _relu_mask(pre, out, what):
    """The kernels' ReLU decision (out > 0) as a float64 mask.  It may differ from the float64 pre-activation's sign
    only where that pre-activation is within rounding (TOL_NET * max|pre|) of zero."""
    keep = out > 0
    pre = pre.detach()
    differ = keep != (pre > 0)
    assert bool((pre.abs()[differ] <= TOL_NET * pre.abs().max()).all()), f"{what}: ReLU mask differs away from zero"
    return keep.double()


def _dueling_f64(net, x, M):
    """oracle.nets.dueling in float64 on CPU copies of net.p, with the ReLU masks of the kernels' forward (tag "t.").
    A pre-activation within rounding of zero may round to either side; its gradient then passes or is blocked as a
    whole, which no rounding bound covers, so the reference follows the kernels there."""
    import torch.nn.functional as F
    p = {k: v.detach().cpu().double().requires_grad_(True) for k, v in net.p.items()}
    h = x.double() / 255.0
    for li, (name, _, co, _, st, _, (oh, ow)) in enumerate(net.head.layers):
        pre = F.conv2d(h, p[f"head.{name}.weight"], p[f"head.{name}.bias"], stride=st)
        y = net._buf(f"t.head.y{li}", (M * oh * ow, co)).view(M, oh, ow, co).permute(0, 3, 1, 2).cpu()
        h = pre * _relu_mask(pre, y, name)
    f = h.reshape(M, -1)
    xs = []
    for s in ("a", "v"):
        pre = F.linear(f, p[f"l1_{s}.weight"], p[f"l1_{s}.bias"])
        xs.append(pre * _relu_mask(pre, net._buf(f"t.x{s}", (M, net.D_hidden)).cpu(), "l1_" + s))
    a = F.linear(xs[0], p["l2_a.weight"], p["l2_a.bias"])
    q = a - a.mean(dim=1, keepdim=True) + F.linear(xs[1], p["l2_v.weight"], p["l2_v.bias"])
    return q, p


@pytest.mark.parametrize("shape,M", NET_CASES)
def test_cnn_dueling_forward_backward_vs_float64(shape, M):
    net = _dueling_cnn(shape, seed=M, bias_seed=100 + M)
    g = torch.Generator().manual_seed(M)
    x = torch.randint(0, 256, (M,) + shape, dtype=torch.uint8, generator=g)
    dq = torch.randn(M, 4, generator=g)
    xd, dqd = x.cuda(), dq.cuda()
    q = net.forward(xd, save=True).clone()
    net.backward(dqd, M)
    grads = {k: v.clone() for k, v in net.g.items()}
    net.backward(dqd, M)
    torch.cuda.synchronize()
    for k, v in net.g.items():
        assert torch.equal(v, grads[k]), f"second backward changed {k}"

    q_ref, p = _dueling_f64(net, x, M)
    q_ref.backward(dq.double())
    _normwise(q, q_ref, TOL_NET, "Q")
    for k, v in grads.items():
        _normwise(v, p[k].grad, TOL_NET, "grad " + k)


def test_cnn_dueling_forward_rows_vs_float64():
    """forward_rows cuts 300 rows into 256 + 44; the 256-row chunk's conv1 (102400 x 32 x 256) is a 128x64-tile product."""
    from oracle import nets as onets
    net = _dueling_cnn((4, 84, 84), seed=7, bias_seed=8)
    x = torch.randint(0, 256, (300, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(9))
    q = torch.empty(300, 4, device="cuda")
    net.forward_rows(x.cuda(), q)
    with torch.no_grad():
        q_ref = onets.dueling({k: v.cpu().double() for k, v in net.p.items()}, x.double())
    _normwise(q, q_ref, TOL_NET, "Q")


# ---- B2: optimizer steps -------------------------------------------------------------------------------------------
class _OptTwin:
    """torch.optim in float64 on CPU copies of fp32 parameters, plus elementwise error bounds for the fp32 kernels."""
    STATE = {"rmsprop": ("square_avg", "grad_avg"), "adam": ("exp_avg_sq", "exp_avg")}   # (second moment, signed mean)

    def __init__(self, kind, params, lr, eps):
        self.kind = kind
        self.p = [t.detach().cpu().double().clone().requires_grad_(True) for t in params]
        self.opt = (torch.optim.RMSprop(self.p, lr=lr, alpha=ALPHA, eps=eps, centered=True) if kind == "rmsprop"
                    else torch.optim.Adam(self.p, lr=lr, eps=eps))
        self.mag = [torch.zeros_like(t) for t in self.p]       # first-moment EMA of |clipped g|
        self.pbound = [torch.zeros_like(t) for t in self.p]

    def step(self, grads, max_norm):
        """One clip + step; returns the unclipped gradient norm."""
        for t, g in zip(self.p, grads):
            t.grad = g.detach().cpu().double().clone()
        norm = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(t.grad) for t in self.p])).item()
        if max_norm:
            torch.nn.utils.clip_grad_norm_(self.p, max_norm)
        self.opt.step()
        grp = self.opt.param_groups[0]
        lr, eps = grp["lr"], grp["eps"]
        decay = ALPHA if self.kind == "rmsprop" else grp["betas"][0]
        for i, t in enumerate(self.p):
            st, ga = self.opt.state[t], t.grad.abs()
            self.mag[i].mul_(decay).add_((1 - decay) * ga)
            if self.kind == "rmsprop":
                upd = lr * ga / ((st["square_avg"] - st["grad_avg"] ** 2).sqrt() + eps)
            else:
                b1, b2 = grp["betas"]
                n = float(st["step"])
                den = st["exp_avg_sq"].sqrt() / math.sqrt(1 - b2 ** n) + eps
                upd = lr / (1 - b1 ** n) * self.mag[i] / den
            self.pbound[i] += 2 * KU * upd + U * t.detach().abs()
        return norm

    def check(self, i, got_p, got_state, what):
        """got_state: {name: tensor} of the kernel's optimizer state for parameter i."""
        st = self.opt.state[self.p[i]]
        sq, mean = self.STATE[self.kind]
        _within(got_p, self.p[i], self.pbound[i], what + " param")
        _within(got_state[sq], st[sq], KU * st[sq], what + " " + sq)
        _within(got_state[mean], st[mean], KU * self.mag[i], what + " " + mean)


def _flat_optimizer(kind, net, lr=LR):
    from jorldy_b200.core.optimizer import Adam, RMSprop
    if kind == "rmsprop":
        return RMSprop(net.parameters(), lr=lr, alpha=ALPHA, eps=RMS_EPS, centered=True)
    return Adam(net.parameters(), lr=lr)


N_STEPS, LR_SWITCH = 12, 7


def _grad_sequence(net, seed):
    """Independent gradients with ||g|| alternating 4x and 0.25x CLIP, so clipping switches on and off."""
    g = torch.Generator().manual_seed(seed)
    for t in range(N_STEPS):
        raw = [torch.randn(v.shape, generator=g) for v in net.p.values()]
        norm = math.sqrt(sum(float((r.double() ** 2).sum()) for r in raw))
        scale = CLIP * (4.0 if t % 2 == 0 else 0.25) / norm
        yield [r * scale for r in raw]


def _run_steps(kind, net, seed, on_step=None):
    opt = _flat_optimizer(kind, net)
    for t, grads in enumerate(_grad_sequence(net, seed)):
        if t == LR_SWITCH:
            opt.param_groups[0]["lr"] = LR / 2      # the lr_decay path: _sync_lr rewrites the device-side lr
        for v, gk in zip(net.g.values(), grads):
            v.copy_(gk)
        opt.step(max_norm=CLIP)
        if on_step is not None:
            on_step(t, opt, grads)
    torch.cuda.synchronize()
    return opt


@pytest.mark.parametrize("kind", ["rmsprop", "adam"])
def test_optimizer_steps_vs_torch_optim(kind):
    """12 clipped steps over the Ape-X network's flat buffers (3.29 M floats: jb_grad_sumsq writes more partials than
    the 256 threads that fold them), with an lr change after step 7."""
    net = _dueling_cnn((4, 84, 84), seed=11)
    p0 = {k: v.detach().cpu().clone() for k, v in net.p.items()}
    twin = _OptTwin(kind, p0.values(), LR, RMS_EPS if kind == "rmsprop" else 1e-8)
    names = list(net.p)

    def on_step(t, opt, grads):
        assert opt._n_partials > 256
        if t == LR_SWITCH:
            twin.opt.param_groups[0]["lr"] = LR / 2
        norm = twin.step(grads, CLIP)
        assert (norm > CLIP) == (t % 2 == 0)
        np.testing.assert_allclose(opt.grad_norm.item(), norm, rtol=KU, err_msg=f"step {t} grad norm")
        state = opt.state_dict()["state"]
        for i, k in enumerate(names):
            twin.check(i, net.p[k], state[i], f"step {t} {k}")

    opt = _run_steps(kind, net, seed=12, on_step=on_step)
    first = [net.flat.clone()] + [s.clone() for s in opt.state_tensors()]
    net.load_state_dict(p0)
    opt = _run_steps(kind, net, seed=12)
    again = [net.flat] + opt.state_tensors()
    assert all(torch.equal(a, b) for a, b in zip(first, again)), "a repeated step sequence is not bit-identical"


@pytest.mark.parametrize("P", [1, 3, 5, 4097])
@pytest.mark.parametrize("kind", ["rmsprop", "adam"])
def test_optimizer_abi_tails(kind, P):
    """P % 4 != 0 takes the scalar tails of jb_grad_sumsq / jb_adam_step / jb_copy_f32, which FlatNetwork's 4-float
    padding never reaches.  Inputs hold NaN past P and outputs a sentinel, so a tail that reads or writes past P fails."""
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    gen = torch.Generator().manual_seed(P)
    n_part = C.jb_grad_partials_count(P)
    eps = RMS_EPS if kind == "rmsprop" else 1e-8
    for mode in ("clipped", "unclipped", "disabled"):
        p_host = torch.randn(P, generator=gen)
        twin = _OptTwin(kind, [p_host], LR, eps)
        p, s1, s2 = (torch.full((P + 8,), 7.0, device="cuda") for _ in range(3))
        p[:P] = p_host.cuda()
        s1[:P] = 0.0
        s2[:P] = 0.0
        lr = torch.tensor([LR], device="cuda")
        step = torch.zeros(1, dtype=torch.int64, device="cuda")
        partials = torch.full((n_part,), float("nan"), device="cuda")
        norm_out = torch.zeros(1, device="cuda")
        for t in range(3):
            gv = torch.randn(P, generator=gen) * (100.0 if mode == "disabled" else 1.0)
            norm = gv.double().norm().item()
            max_norm = {"clipped": 0.5 * norm, "unclipped": 2.0 * norm, "disabled": 0.0}[mode]
            g = torch.full((P + 8,), float("nan"), device="cuda")
            g[:P] = gv.cuda()
            s = stream_ptr()
            C.jb_grad_sumsq(ptr(g), P, ptr(partials), ptr(step), s)
            if kind == "rmsprop":
                C.jb_rmsprop_centered_step(ptr(p), ptr(g), ptr(s1), ptr(s2), P, ptr(lr), ALPHA, eps, ptr(partials), n_part,
                                           max_norm, ptr(norm_out), s)
            else:
                C.jb_adam_step(ptr(p), ptr(g), ptr(s1), ptr(s2), P, ptr(lr), 0.9, 0.999, eps, ptr(step), ptr(partials),
                               n_part, max_norm, ptr(norm_out), s)
            twin.step([gv], max_norm)
            torch.cuda.synchronize()
            what = f"{mode} step {t}"
            np.testing.assert_allclose(norm_out.item(), norm, rtol=KU, err_msg=what + " grad norm")
            names = ("square_avg", "grad_avg") if kind == "rmsprop" else ("exp_avg", "exp_avg_sq")
            twin.check(0, p[:P], {names[0]: s1[:P], names[1]: s2[:P]}, what)
            for buf in (p, s1, s2):
                assert bool((buf[P:] == 7.0).all()), what + ": write past P"
    dst = torch.full((P + 8,), 7.0, device="cuda")
    C.jb_copy_f32(ptr(dst), ptr(p), P, stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(dst[:P], p[:P]) and bool((dst[P:] == 7.0).all())


# ---- B3: one learn() at the benchmark's shapes ---------------------------------------------------------------------
_ATARI = dict(D=[4, 84, 84], A=4, H=512, head="cnn", gamma=0.99, n_step=3, lr=LR)
_APEX = dict(_ATARI, seed=51, agent="ape_x", net="dueling", B=512, buffer_size=512, alpha=0.6, clip=CLIP,
             optim={"name": "rmsprop", "eps": RMS_EPS, "lr": LR, "centered": True})
LEARN_CASES = {
    "ape_x_b512": _APEX,                                # ||g|| ~ 21 < 40: the clip coefficient is 1
    "ape_x_b512_clipped": dict(_APEX, clip=10.0),       # same batch with clip below ||g||: the clipped path
    "rainbow_b32": dict(_ATARI, seed=53, agent="rainbow", net="rainbow", B=32, buffer_size=32, K=51, v_min=-1, v_max=10,
                        alpha=0.5),
}


def _q_oracle_f64(case):
    from oracle import dqn as odqn
    params, tparams, batch, hp, optim, _ = q_oracle_inputs(case)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        b = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in batch.items()}
        return odqn.td_learn({k: v.double() for k, v in params.items()}, {k: v.double() for k, v in tparams.items()},
                             b, hp, optim)
    finally:
        torch.set_default_dtype(prev)


@pytest.mark.parametrize("name", list(LEARN_CASES))
def test_learn_at_benchmark_shapes(name):
    case = LEARN_CASES[name]
    agent, prio = _run(case)
    ref, _ = run_q_oracle(case)
    net = agent.network
    st = agent._stats.cpu().numpy()
    np.testing.assert_allclose(st[0], ref["loss"], rtol=2e-5, err_msg="loss")
    np.testing.assert_allclose(st[1], ref["max_Q"], rtol=2e-5, err_msg="max_Q")
    if "max_logit" in ref:
        np.testing.assert_allclose(st[2], ref["max_logit"], rtol=2e-5, err_msg="max_logit")
        np.testing.assert_allclose(st[3], ref["min_logit"], rtol=2e-5, err_msg="min_logit")
    np.testing.assert_allclose(prio.cpu().numpy(), ref["priority"].numpy(), rtol=2e-4, atol=1e-6, err_msg="priorities")
    for k, g in ref["grads"].items():
        atol = max(2e-6, 2 * TOL_NET * g.abs().max().item())
        np.testing.assert_allclose(net.g[k].cpu().numpy(), g.numpy(), rtol=2e-3, atol=atol, err_msg="grad " + k)
    if case["agent"] == "ape_x":
        ref64 = _q_oracle_f64(case)
        for k, g in ref64["grads"].items():
            _normwise(net.g[k], g, TOL_NET, "grad vs float64 " + k)

    clip = case.get("clip")
    gn = agent.optimizer.grad_norm.item()
    if clip is not None:
        assert (gn > clip) == name.endswith("_clipped"), f"||g|| = {gn}, clip {clip}"
    optim = case.get("optim", {"name": "adam"})
    params = G.q_params(case)
    twin = _OptTwin(optim["name"], [torch.from_numpy(params[k]) for k in net.p], case["lr"], optim.get("eps", 1e-8))
    twin.step([net.g[k] for k in net.p], clip)
    state = agent.optimizer.state_dict()["state"]
    for i, k in enumerate(net.p):
        twin.check(i, net.p[k], state[i], k)
