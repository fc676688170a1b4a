"""The Rainbow learner at the benchmark's shapes (rainbow_frames: C51 with K = 51 atoms, 3-step returns, NoisyNet, CNN on
84x84x4 frames, B = 32, A = 4) vs float64: jb_c51_loss / jb_c51_q through the C ABI, the NoisyNet kernels (injected and
Philox noise), the atom-wise dueling head, the noisy network forward / backward / forward_rows, and one learn().

Discontinuities are decided once, in fp32, and the rest is compared under a rounding bound.  The projection's l = floor(b),
u = ceil(b) come from an fp32 quotient, and a one-ulp difference next to an integer moves the target by O(1) (l == u drops
the atom's mass), so the reference takes b from numpy float32 in the kernel's and the reference's operation order
(((1 - d) gamma) Tz, then + r; clamp(Tz - v_min, 0, v_max - v_min) / fp32(delta_z)) and checks it bit-equal to torch-CPU
float32 running oracle/dqn.py's own expressions; softmax, expected Q, projection weights, KL, gradient and priority are
float64.  The ReLU masks of the networks are taken from the kernels (test_atari_learner_gpu._relu_mask).

Tolerances (u = 2^-24; expf / logf / powf / sqrtf are ulp-accurate):
  * softmax p = expf((x - max) - logf(s)): the two subtractions round by u |x - max| and u |arg|, logf(s) carries
    u |log s| plus s's relative error (a warp tree over K <= 64 terms, 6 u); exp turns the argument's absolute error
    into p's relative error.  With L = max row spread of x + log K, p is elementwise within E_p = (2 L + 12) u.
  * Expected Q = sum_k z_k p_k (a warp tree): within (E_p + 6 u) max|z|.  The a* inputs keep the top-two gap above
    100x that, except for deliberate bitwise ties (first index wins, as torch.argmax).
  * Target t: tp_i (E_p of the target logits) times exact-or-u projection weights, accumulated over K source atoms in
    sequence (K u), normalised by a warp sum (6 u): elementwise relative E_t = (K + 2 L_t + 24) u.
  * KL = -sum_k t_k log max(p_k, 1e-8) (a warp tree): within (E_t + 8 u) sum_k t_k |log p_k| + E_p.
  * dlogits = coef (p S - t g), S = sum t g: within |coef| ((E_p + E_t + 10 u) p S + (E_t + 2 u) t) + E_w |d| with
    E_w = (B / 32 + 8) u for Rainbow's batch-mean weight (lane sums of B / 32 terms, a warp tree, two divisions), else u.
    Actions not taken are exactly 0; rows whose mass is all dropped are exactly 0 (t = 0, KL = 0, priority 0).
  * priority = powf(KL, alpha): relative alpha * rel(KL) + 4 u.  loss = sum_b w KL_b / B (8 warps per CTA, then the CTAs
    in order): the KL bounds plus (B / 8 + 16) u sum |w KL| / B.  max_logit / min_logit are exact.
  * NoisyNet: f = sign(e) sqrt|e|, eps_w = f_i f_j, W = mu + sig eps_w, dsig = g eps_w are single IEEE operations in the
    reference's order (__fmul_rn / __fadd_rn, IEEE sqrtf), hence bit-exact against numpy float32.
  * Dueling head over A actions: mean by A - 1 sequential additions and a division, then two roundings:
    (A + 3) u (mean|adv| + |adv| + |v|); backward (A + 2) u sum|dout| for both outputs.
  * Network forward / backward normwise per tensor at TOL_NET = 7.7e3 u (test_atari_learner_gpu): along the Rainbow
    network's longest path the contraction lengths sum to about 7.0e3 (forward 256 + 512 + 576 conv, 3136 l, 512 a1,
    512 a2; backward 204 a2 dx, 512 a1 dx, 512 l dx, 64 + 64 conv dx and conv1's weight gradient at B = 32, 128 terms
    per split group), within the Ape-X network's 7.7e3.
  * learn() vs oracle/dqn.py::dist_learn in float64: the logits are within TOL_NET X normwise (X = max|logit| of the
    three forwards).  log-softmax is 2-Lipschitz in the max norm, so d logits = coef (p S - t g) moves by at most
    4 TOL_NET X relative to its own scale, and the gradients are compared normwise at TOL_NET (1 + 4 X).  KL moves by
    2 TOL_NET X (1 + KL) (sum_k t_k |log p_k| = KL); priorities by alpha times KL's relative error.  On this batch the
    float64 oracle's l / u equal the fp32 ones except in first-step-terminal rows, where the terminal average makes the
    target continuous in b; the test checks that.  Adam is checked with _OptTwin on the kernel's own gradients."""
import math

import numpy as np
import pytest
import torch

import gen_inputs as G
from helpers import q_oracle_inputs
from test_atari_learner_gpu import LEARN_CASES, TOL_NET, U, _OptTwin, _normwise, _relu_mask, _within
from test_dqn_gpu import _make, _run

pytestmark = pytest.mark.gpu

V_MIN, V_MAX, GAMMA, ALPHA = -1.0, 10.0, 0.99, 0.5
F32 = np.float32


def _abi():
    from jorldy_b200.core.dev import C, JbError, ptr, stream_ptr
    return C, JbError, ptr, stream_ptr


def _bits(t):
    return (t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)).astype(np.float32).view(np.int32)


def _support(K):
    """The support the reference builds (torch.linspace on the CPU) and fp32 delta_z as the kernel forms it."""
    return torch.linspace(V_MIN, V_MAX, K).numpy(), F32((V_MAX - V_MIN) / (K - 1))


def _tz_b(r, d, K):
    """numpy float32 in the kernel's and the reference's order: Tz = r + ((1 - d) gamma) Tz from the last step back,
    b = clamp(Tz - v_min, 0, v_max - v_min) / delta_z.  r, d: [B, n] float32."""
    z, dz = _support(K)
    tz = np.broadcast_to(z, (r.shape[0], K)).astype(F32)
    for s in range(r.shape[1] - 1, -1, -1):
        tz = r[:, s:s + 1] + ((F32(1) - d[:, s:s + 1]) * F32(GAMMA)) * tz
    return np.minimum(np.maximum(tz - F32(V_MIN), F32(0)), F32(V_MAX) - F32(V_MIN)) / dz


def _oracle_b(r, d, K, variant):
    """oracle/dqn.py::dist_learn's own Tz / b expressions in torch-CPU float32."""
    zt = torch.linspace(V_MIN, V_MAX, K).view(1, -1)
    rt, dt = torch.from_numpy(r).unsqueeze(-1), torch.from_numpy(d).unsqueeze(-1)
    if variant == 0 and r.shape[1] == 1:                         # c51.py
        Tz = rt[:, 0].expand(-1, K) + (1 - dt[:, 0]) * GAMMA * zt
    else:                                                        # rainbow.py
        Tz = zt
        for i in reversed(range(r.shape[1])):
            Tz = rt[:, i].expand(-1, K) + (1 - dt[:, i]) * GAMMA * Tz
    return (torch.clamp(Tz - V_MIN, 0, V_MAX - V_MIN) / ((V_MAX - V_MIN) / (K - 1))).numpy()


def _near(x):
    """4096 fp32 neighbours of x (by bit pattern)."""
    i = np.asarray(x, dtype=F32).view(np.int32) + np.arange(-2048, 2048, dtype=np.int32)
    return i.view(F32)


def _interior_integer(b, K):
    return (b == np.floor(b)) & (b > 0) & (b < K - 1)


_R0 = {}


def _integer_rewards(K, n):
    """First-step rewards that put b on an exact fp32 integer strictly inside the support: (terminal at step 0 -> all
    atoms at b = (r0 - v_min) / dz, live row with later rewards 0 -> at least one atom).  None when K leaves no interior."""
    if (K, n) in _R0:
        return _R0[(K, n)]
    out = None
    if K > 2:
        z, dz = _support(K)
        found = []
        for term in (True, False):
            k0 = K // 2
            base = F32(V_MIN + k0 * float(dz)) if term else F32(V_MIN + k0 * float(dz) - GAMMA ** n * float(z[k0]))
            cand = _near(base)
            r = np.zeros((cand.size, n), F32); r[:, 0] = cand
            d = np.zeros((cand.size, n), F32); d[:, 0] = 1.0 if term else 0.0
            hit = _interior_integer(_tz_b(r, d, K), K).any(1)
            assert hit.any(), f"no fp32 reward near {base} lands on an integer b (K={K}, n={n})"
            found.append(F32(cand[np.argmax(hit)]))
        out = tuple(found)
    _R0[(K, n)] = out
    return out


ROW_KINDS = ("random", "top", "bottom", "drop", "term0_int", "term_late", "live_int", "tie_spiky")


def _c51_inputs(B, A, K, n, variant, seed):
    rs = np.random.RandomState(seed)
    x = (1.5 * rs.standard_normal((B, A, K))).astype(F32)
    ramp = np.linspace(-1.0, 1.0, K)
    srcs = []
    for _ in range(2):                          # next_online, next_target: independent action preferences per row
        ranks = np.argsort(rs.random_sample((B, A)), 1)
        c = (2.0 * ranks - (A - 1)) / max(A - 1, 1)             # in [-1, 1]: the tilt moves Q without saturating p
        srcs.append((0.02 * rs.standard_normal((B, A, K)) + c[:, :, None] * 3.0 * ramp).astype(F32))
    online, target = srcs
    action = rs.randint(0, A, size=B)
    r = rs.choice([0.1, -1.0, 1.0, 2.5], size=(B, n)).astype(F32)
    d = (rs.uniform(size=(B, n)) < 0.15).astype(F32)
    w = rs.uniform(0.2, 1.0, size=B)
    ints = _integer_rewards(K, n)
    for b in range(B if B > 1 else 0):
        kind = ROW_KINDS[b % len(ROW_KINDS)]
        if kind == "top":
            r[b], d[b] = 2.5, 0.0
        elif kind == "bottom":
            r[b], d[b] = 0.0, 0.0
            r[b, 0] = -1.0
        elif kind == "drop":
            r[b], d[b] = 0.0, 0.0
            r[b, 0] = 100.0
        elif kind == "term0_int" and ints is not None:
            r[b, 0], d[b, 0] = ints[0], 1.0
        elif kind == "term_late" and n > 1:
            d[b] = 0.0
            d[b, n - 1] = 1.0
        elif kind == "live_int" and ints is not None:
            r[b], d[b] = 0.0, 0.0
            r[b, 0] = ints[1]
        elif kind == "tie_spiky":
            sel = online if variant == 1 else target
            if A > 1:
                top = int(np.argmax((_softmax64(sel[b]) * _support(K)[0]).sum(-1)))
                sel[b, 0] = sel[b, top]
                sel[b, A - 1] = sel[b, top]
            x[b, action[b], ::2] = -40.0 + rs.standard_normal(x[b, action[b], ::2].shape).astype(F32)
    return dict(logits=x, online=online, target=target, action=action, r=r, d=d, w=w)


def _softmax64(x):
    x = np.asarray(x, np.float64)
    e = np.exp(x - x.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _spread(x, K):
    return float((x.max(-1) - x.min(-1)).max()) + math.log(K)


def _c51_reference(inp, B, A, K, n, variant):
    z, dz = _support(K)
    zd = z.astype(np.float64)
    rows = np.arange(B)
    p = _softmax64(inp["logits"])
    q = (p * zd).sum(-1)
    src = inp["online"] if variant == 1 else inp["target"]
    qs = (_softmax64(src) * zd).sum(-1)
    a_star = qs.argmax(1)
    tp = _softmax64(inp["target"][rows, a_star])
    bb = _tz_b(inp["r"], inp["d"], K)
    l, u = np.floor(bb), np.ceil(bb)
    b64 = bb.astype(np.float64)
    j = np.arange(K)
    lo, uo = (l[:, :, None] == j), (u[:, :, None] == j)
    lluu = lo * (u - b64)[:, :, None] + uo * (b64 - l)[:, :, None]
    term = inp["d"][:, 0] > 0.5
    t = np.where(term[:, None], (lo * uo + lluu).mean(1), (tp[:, :, None] * lluu).sum(1))
    t = t / np.maximum(t.sum(1, keepdims=True), 1e-8)
    pa = p[rows, inp["action"]]
    g = pa >= 1e-8
    lp = np.log(np.maximum(pa, 1e-8))
    kl = -(t * lp).sum(1)
    wmean = float(inp["w"].astype(F32).astype(np.float64).mean()) if variant == 1 else 1.0
    coef = wmean / B
    S = (t * g).sum(1, keepdims=True)
    dl = np.zeros((B, A, K))
    dl[rows, inp["action"]] = coef * (pa * S - t * g)
    E_p = (2 * _spread(inp["logits"], K) + 12) * U
    E_t = (K + 2 * _spread(inp["target"], K) + 24) * U
    E_q = (2 * _spread(src, K) + 20) * U * np.abs(zd).max()
    E_w = (B / 32 + 8) * U if variant == 1 else U
    kl_bound = (E_t + 8 * U) * (t * np.abs(lp)).sum(1) + E_p
    d_bound = np.zeros((B, A, K))
    d_bound[rows, inp["action"]] = coef * ((E_p + E_t + 10 * U) * pa * S + (E_t + 2 * U) * t * g)
    d_bound += E_w * np.abs(dl)
    loss = (wmean * kl).sum() / B
    return dict(
        kl=kl, kl_bound=kl_bound, dl=dl, d_bound=d_bound, prio=kl ** ALPHA, loss=loss, E_q=E_q, E_w=E_w,
        loss_bound=(wmean * kl_bound).sum() / B + (B / 8 + 16) * U * wmean * np.abs(kl).sum() / B + E_w * abs(loss),
        max_q=q.max(), max_logit=inp["logits"].max(), min_logit=inp["logits"].min(),
        bb=bb, t=t, pa=pa, term=term, qs=qs, a_star=a_star, variant=variant)


_KINDS = {"int64": (torch.int64, 0), "int32": (torch.int32, 1), "float32": (torch.float32, 2)}


def _c51_run(inp, B, A, K, n, variant, dtype="int64"):
    C, _, ptr, sp = _abi()
    cu = lambda a, dt=torch.float32: torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dt)
    t_dtype, kind = _KINDS[dtype]
    logits, online, target = cu(inp["logits"]), cu(inp["online"]), cu(inp["target"])
    action = cu(inp["action"], t_dtype)
    r, d = cu(inp["r"]), cu(inp["d"])
    w = cu(inp["w"], torch.float64)
    z = torch.linspace(V_MIN, V_MAX, K).cuda()
    dl = torch.full((B, A, K), float("nan"), device="cuda")
    kl = torch.full((B,), float("nan"), device="cuda")
    prio = torch.full((B,), float("nan"), dtype=torch.float64, device="cuda")
    stats = torch.full((4,), float("nan"), device="cuda")
    scratch = torch.empty(4 * ((B + 7) // 8), device="cuda")
    C.jb_c51_loss(ptr(logits), ptr(online), ptr(target), ptr(action), kind, ptr(r), ptr(d), ptr(w),
                  ptr(z), B, A, K, GAMMA, V_MIN, V_MAX, ALPHA, n, variant, ptr(dl), ptr(kl), ptr(prio), ptr(stats),
                  ptr(scratch), sp())
    torch.cuda.synchronize()
    return dl.cpu(), kl.cpu(), prio.cpu(), stats.cpu()


def _tied_rows(inp, ref, A):
    src = inp["online"] if ref["variant"] == 1 else inp["target"]
    return np.array([A > 1 and np.array_equal(src[b, 0], src[b, A - 1]) and ref["a_star"][b] == 0
                     for b in range(src.shape[0])], bool)


def _c51_case(B, A, K, n, variant, seed):
    """Inputs and float64 reference; checks that fp32 b matches the oracle's expressions bit for bit and that the inputs
    keep every other fp32 decision away from rounding: a* gaps (ties are bitwise), the 1e-8 gradient mask."""
    inp = _c51_inputs(B, A, K, n, variant, seed)
    np.testing.assert_array_equal(_tz_b(inp["r"], inp["d"], K).view(np.int32),
                                  _oracle_b(inp["r"], inp["d"], K, variant).view(np.int32), "b: numpy fp32 != oracle")
    ref = _c51_reference(inp, B, A, K, n, variant)
    if A > 1:
        qs = np.sort(ref["qs"], 1)
        gap = (qs[:, -1] - qs[:, -2])[~_tied_rows(inp, ref, A)]
        assert bool((gap > 100 * ref["E_q"]).all()), f"a* gap {gap.min():.2e} within rounding"
    pa = ref["pa"]
    assert not bool(((pa > 1e-9) & (pa < 1e-7)).any()), "a taken-action probability sits at the 1e-8 mask"
    return inp, ref


def _check_c51(B, A, K, n, variant, dtype, seed):
    inp, ref = _c51_case(B, A, K, n, variant, seed)
    dl, kl, prio, st = _c51_run(inp, B, A, K, n, variant, dtype)
    rows = np.arange(B)
    off = np.ones((B, A), bool); off[rows, inp["action"]] = False
    assert bool((dl.numpy()[off] == 0).all()), "dlogits of actions not taken must be exactly 0"
    _within(dl, torch.from_numpy(ref["dl"]), torch.from_numpy(ref["d_bound"]), "dlogits")
    _within(kl, torch.from_numpy(ref["kl"]), torch.from_numpy(ref["kl_bound"]), "kl")
    pos = ref["kl"] > 0
    pb = np.zeros(B)
    pb[pos] = ref["prio"][pos] * (ALPHA * ref["kl_bound"][pos] / ref["kl"][pos] + 4 * U)
    _within(prio, torch.from_numpy(ref["prio"]), torch.from_numpy(pb), "priority")
    assert abs(st[0].item() - ref["loss"]) <= ref["loss_bound"], f"loss {st[0].item()} vs {ref['loss']}"
    assert abs(st[1].item() - ref["max_q"]) <= ref["E_q"] + 6 * U * abs(ref["max_q"]), "max_Q"
    assert st[2].item() == ref["max_logit"] and st[3].item() == ref["min_logit"], "logit stats"
    return inp, ref, (dl, kl, prio, st)


# ---- R1: jb_c51_loss -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", list(_KINDS))
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("B", [1, 7, 32, 33, 512])
@pytest.mark.parametrize("A", [1, 4, 18])
@pytest.mark.parametrize("K", [2, 32, 33, 51, 64])
def test_c51_loss_vs_float64(K, A, B, n, variant, dtype):
    _check_c51(B, A, K, n, variant, dtype, seed=K * 1000 + A * 100 + B + 7 * n + variant)


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("K", [51, 64])
def test_c51_inputs_reach_every_branch(K, n, variant):
    B, A = 512, 4
    inp, ref, (dl, kl, prio, _) = _check_c51(B, A, K, n, variant, "int64", seed=99 + K + n + variant)
    bb, live = ref["bb"], ~ref["term"]
    assert bool((bb == K - 1).any()) and bool((bb == 0).any()), "atoms clamped at both ends"
    assert bool((_interior_integer(bb, K) & live[:, None]).any()), "an interior exact-integer b in a live row"
    assert bool((_interior_integer(bb, K) & ref["term"][:, None]).any()), "an exact-integer b in a terminal row"
    dropped = live & (ref["t"].sum(1) == 0)
    assert bool(dropped.any()), "a row whose whole mass is dropped"
    assert bool((kl.numpy()[dropped] == 0).all()) and bool((prio.numpy()[dropped] == 0).all())
    assert bool((dl.numpy()[dropped] == 0).all())
    assert bool(ref["term"].any()), "terminal at step 0"
    if n > 1:
        assert bool((live & (inp["d"][:, 1:] > 0.5).any(1)).any()), "terminal at a later step"
    assert bool(((ref["pa"] < 1e-8) & (ref["t"] > 0)).any()), "masked taken-action probabilities with target mass"
    assert _tied_rows(inp, ref, A).any(), "bitwise-tied a* rows resolving to the first index"
    if variant == 1:
        a_tgt = (_softmax64(inp["target"]) * _support(K)[0]).sum(-1).argmax(1)
        assert int((a_tgt != ref["a_star"]).sum()) > B // 4, "online and target nets disagree on a*"


def test_c51_loss_rejects_bad_arguments():
    """K <= 1, K > 64 (buffers sized for 65 atoms, so nothing could be overrun), and Rainbow without next_online."""
    C, JbError, ptr, sp = _abi()
    B, A = 4, 2
    buf = torch.zeros(B, A, 65, device="cuda")
    act = torch.zeros(B, dtype=torch.int64, device="cuda")
    rd = torch.zeros(B, 1, device="cuda")
    kl, st, scr, z = (torch.zeros(n, device="cuda") for n in (B, 4, 4 * B, 65))
    for K, variant, online in ((1, 0, buf), (65, 0, buf), (0, 1, buf), (51, 1, None)):
        with pytest.raises(JbError):
            C.jb_c51_loss(ptr(buf), ptr(online), ptr(buf), ptr(act), 0, ptr(rd), ptr(rd), 0, ptr(z), B, A, K, GAMMA, V_MIN,
                          V_MAX, ALPHA, 1, variant, ptr(buf), ptr(kl), 0, ptr(st), ptr(scr), sp())
    for K in (1, 65):
        with pytest.raises(JbError):
            C.jb_c51_q(ptr(buf), ptr(z), 1, A, K, ptr(kl), sp())


def test_device_support_is_the_cpu_linspace():
    """The agents' support z is a CUDA linspace; the reference's is torch.linspace on the CPU."""
    from jorldy_b200.core import Agent
    for K in (2, 32, 33, 51, 64):
        assert torch.equal(torch.linspace(V_MIN, V_MAX, K, device="cuda").cpu(), torch.linspace(V_MIN, V_MAX, K)), K
    agent = Agent("c51", state_size=4, action_size=2, hidden_size=32, batch_size=4, buffer_size=16, device="cuda",
                  v_min=V_MIN, v_max=V_MAX, num_support=51)
    assert torch.equal(agent.z.cpu().view(-1), torch.linspace(V_MIN, V_MAX, 51))


# ---- R2: jb_c51_q (act) ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 64, 300])
@pytest.mark.parametrize("A", [1, 4, 18])
@pytest.mark.parametrize("K", [2, 32, 33, 51, 64])
def test_c51_q_vs_float64(K, A, M):
    C, _, ptr, sp = _abi()
    rs = np.random.RandomState(K * 7 + A * 3 + M)
    x = (20.0 * rs.standard_normal((M, A, K)) + 50.0).astype(F32)       # wide rows, far from 0: the max subtraction
    z = torch.linspace(V_MIN, V_MAX, K)
    q = torch.full((M, A), float("nan"), device="cuda")
    xd, zd = torch.from_numpy(x).cuda(), z.cuda()       # held: a temporary's block could be reused before the launch
    C.jb_c51_q(ptr(xd), ptr(zd), M, A, K, ptr(q), sp())
    torch.cuda.synchronize()
    p = _softmax64(x)
    zd = z.double().numpy()
    ref = (p * zd).sum(-1)
    bound = ((2 * _spread(x, K) + 20) * U) * (p * np.abs(zd)).sum(-1)
    _within(q, torch.from_numpy(ref), torch.from_numpy(bound), "expected Q")


# ---- R3: NoisyNet kernels --------------------------------------------------------------------------------------------
NOISY_SHAPES = [(512, 512), (512, 204), (512, 51), (3136, 512), (1, 1), (7, 13)]


def _noisy_make(mu_w, sig_w, mu_b, sig_b, eps_i=None, eps_j=None, seed=5, stream=1, ctr=None, is_train=1):
    C, _, ptr, sp = _abi()
    i, o = mu_w.shape
    fi, fj = torch.full((i,), float("nan"), device="cuda"), torch.full((o,), float("nan"), device="cuda")
    w, b = torch.full((i, o), float("nan"), device="cuda"), torch.full((o,), float("nan"), device="cuda")
    C.jb_noisy_make(ptr(mu_w), ptr(sig_w), ptr(mu_b), ptr(sig_b), i, o, ptr(eps_i), ptr(eps_j), seed, stream, ptr(ctr),
                    is_train, ptr(fi), ptr(fj), ptr(w), ptr(b), sp())
    torch.cuda.synchronize()
    return fi, fj, w, b


def _noisy_params(i, o, seed):
    g = torch.Generator().manual_seed(seed)
    return [t.cuda() for t in (torch.randn(i, o, generator=g) / math.sqrt(i), 0.5 / math.sqrt(i) * torch.rand(i, o, generator=g),
                               torch.randn(o, generator=g) * 0.1, 0.5 / math.sqrt(i) * torch.rand(o, generator=g))]


def _f_np(e):
    e = np.asarray(e, F32)
    return (np.sign(e) * np.sqrt(np.abs(e))).astype(F32)


@pytest.mark.parametrize("shape", NOISY_SHAPES)
def test_noisy_make_and_grad_injected_bit_exact(shape):
    C, _, ptr, sp = _abi()
    i, o = shape
    mu_w, sig_w, mu_b, sig_b = _noisy_params(i, o, i * 31 + o)
    g = torch.Generator().manual_seed(o)
    ei, ej = torch.randn(i, generator=g), torch.randn(o, generator=g)
    ei[0] = 0.0                                              # sign(0) = 0
    ctr = torch.tensor([11], dtype=torch.int64, device="cuda")
    fi, fj, w, b = _noisy_make(mu_w, sig_w, mu_b, sig_b, ei.cuda(), ej.cuda(), ctr=ctr)
    fi_r, fj_r = _f_np(ei.numpy()), _f_np(ej.numpy())
    eps_w = fi_r[:, None] * fj_r[None, :]
    sw, mw = sig_w.cpu().numpy(), mu_w.cpu().numpy()
    np.testing.assert_array_equal(_bits(fi), fi_r.view(np.int32), "f_i")
    np.testing.assert_array_equal(_bits(fj), fj_r.view(np.int32), "f_j")
    np.testing.assert_array_equal(_bits(w), (mw + sw * eps_w).astype(F32).view(np.int32), "W")
    np.testing.assert_array_equal(_bits(b), (mu_b.cpu().numpy() + sig_b.cpu().numpy() * fj_r).view(np.int32), "b")
    assert ctr.item() == 11, "injected normals must not advance the draw counter"

    dw, db = torch.randn(i, o, generator=g), torch.randn(o, generator=g)
    out = [torch.full_like(t, float("nan")) for t in (mu_w, sig_w, mu_b, sig_b)]
    dwd, dbd = dw.cuda(), db.cuda()
    C.jb_noisy_grad(ptr(dwd), ptr(dbd), ptr(fi), ptr(fj), i, o, *(ptr(t) for t in out), sp())
    torch.cuda.synchronize()
    np.testing.assert_array_equal(_bits(out[0]), _bits(dw), "dmu_w")
    np.testing.assert_array_equal(_bits(out[1]), (dw.numpy() * eps_w).view(np.int32), "dsig_w")
    np.testing.assert_array_equal(_bits(out[2]), _bits(db), "dmu_b")
    np.testing.assert_array_equal(_bits(out[3]), (db.numpy() * fj_r).view(np.int32), "dsig_b")

    fi0, fj0, w0, b0 = _noisy_make(mu_w, sig_w, mu_b, sig_b, ctr=ctr, is_train=0)
    assert torch.equal(w0, mu_w) and torch.equal(b0, mu_b), "is_train = 0 gives the mean weights"
    assert not bool(fi0.any()) and not bool(fj0.any()), "is_train = 0 zeroes the factors"
    assert ctr.item() == 11, "is_train = 0 must not advance the draw counter"
    _noisy_make(mu_w, sig_w, mu_b, sig_b, ctr=ctr)
    assert ctr.item() == 12, "a drawn layer advances the draw counter by one"
    if i + o <= 8192:
        _noisy_make(mu_w, sig_w, mu_b, sig_b, ei.cuda(), None, ctr=ctr)
        assert ctr.item() == 13, "a half-injected layer still draws"


def _draw(i, o, seed, stream, c):
    mu_w, sig_w, mu_b, sig_b = _noisy_params(i, o, 1)
    ctr = torch.tensor([c], dtype=torch.int64, device="cuda")
    fi, fj, _, _ = _noisy_make(mu_w, sig_w, mu_b, sig_b, seed=seed, stream=stream, ctr=ctr)
    assert ctr.item() == c + 1
    f = torch.cat([fi, fj]).double().cpu()
    return (f * f.abs()).numpy()


def test_noisy_philox_draws():
    """e = f |f| recovers the Box-Muller normal; 13 draws of an 8000 x 192 layer give 106 496 normals."""
    from scipy import stats
    i, o = 8000, 192
    draws = [_draw(i, o, 5, 1, c) for c in range(13)]
    e = np.concatenate(draws)
    assert e.size >= 10 ** 5
    assert stats.kstest(e, "norm").pvalue > 1e-3
    lim = 5.0 / math.sqrt(i + o)
    others = [_draw(i, o, 5, s, 0) for s in (2, 3, 4)] + [_draw(i, o, 6, 1, 0)]
    for k, x in enumerate(draws[1:4] + others):
        assert not np.array_equal(x, draws[0]), k
        assert abs(np.corrcoef(x, draws[0])[0, 1]) < lim, f"draw {k} correlates with draw 0"
    np.testing.assert_array_equal(_draw(i, o, 5, 1, 3), draws[3], "same seed, stream and counter: same bits")


def test_noisy_drawn_layer_size_limit():
    """Counter = draw * 4096 + factor / 2: a drawn layer may have at most 8192 factors; injected normals have no limit."""
    _, JbError, _, _ = _abi()
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    ok = _noisy_params(4096, 4096, 2)
    _noisy_make(*ok, ctr=ctr)
    assert ctr.item() == 1
    big = _noisy_params(4096, 4097, 2)
    with pytest.raises(JbError):
        _noisy_make(*big, ctr=ctr)
    g = torch.Generator().manual_seed(0)
    _noisy_make(*big, torch.randn(4096, generator=g).cuda(), torch.randn(4097, generator=g).cuda(), ctr=ctr)
    _noisy_make(*big, ctr=ctr, is_train=0)
    assert ctr.item() == 1


# ---- R4: atom-wise dueling head --------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 32, 300])
@pytest.mark.parametrize("A", [1, 4, 18])
@pytest.mark.parametrize("K", [1, 51])
def test_dueling_head_vs_float64(K, A, B):
    C, _, ptr, sp = _abi()
    g = torch.Generator().manual_seed(K + A * 10 + B)
    adv, val, dout = torch.randn(B, A, K, generator=g) * 3, torch.randn(B, K, generator=g), torch.randn(B, A, K, generator=g)
    out = torch.full((B, A, K), float("nan"), device="cuda")
    dadv, dval = torch.full((B, A, K), float("nan"), device="cuda"), torch.full((B, K), float("nan"), device="cuda")
    advd, vald, doutd = adv.cuda(), val.cuda(), dout.cuda()
    C.jb_dueling_fwd(ptr(advd), ptr(vald), B, A, K, ptr(out), sp())
    C.jb_dueling_bwd(ptr(doutd), B, A, K, ptr(dadv), ptr(dval), sp())
    torch.cuda.synchronize()
    a, v, do = adv.double(), val.double().unsqueeze(1), dout.double()
    mean = a.mean(1, keepdim=True)
    _within(out, a - mean + v, (A + 3) * U * (a.abs().mean(1, keepdim=True) + a.abs() + v.abs()), "dueling out")
    s = do.sum(1, keepdim=True)
    bound = (A + 2) * U * do.abs().sum(1, keepdim=True)
    _within(dval, s.squeeze(1), bound.squeeze(1), "dval = sum over actions")
    _within(dadv, do - s / A, bound.expand_as(do), "dadv = centred gradient")


# ---- R5: the network -------------------------------------------------------------------------------------------------
def _bias(net, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, v in net.p.items():
            if k.endswith(".bias"):
                v.copy_(0.1 * torch.randn(v.shape, generator=g))
    return net


def _rainbow_net(D, A, H, head, seed, K=51):
    from jorldy_b200.core.network.noisy import Rainbow
    return _bias(Rainbow(D, A, K, D_hidden=H, head=head, device="cuda", seed=seed), seed + 1)


def _head_f64(net, p, x, M, tag):
    import torch.nn.functional as F
    if net.head.kind == "mlp":
        pre = F.linear(x.double(), p["head.l.weight"], p["head.l.bias"])
        return pre * _relu_mask(pre, net._buf(tag + "head.h", (M, net.head.D_head_out)).cpu(), "head")
    h = x.double() / 255.0
    for li, (name, _, co, _, st, _, (oh, ow)) in enumerate(net.head.layers):
        pre = F.conv2d(h, p[f"head.{name}.weight"], p[f"head.{name}.bias"], stride=st)
        y = net._buf(f"{tag}head.y{li}", (M * oh * ow, co)).view(M, oh, ow, co).permute(0, 3, 1, 2).cpu()
        h = pre * _relu_mask(pre, y, name)
    return h.reshape(M, -1)


def _rainbow_f64(net, x, noise, tag="t."):
    """oracle.nets.rainbow_network in float64 with the kernels' ReLU masks; noise: float64 (eps_i, eps_j) x 4."""
    import torch.nn.functional as F
    from oracle import nets as onets
    M, H, A, K = x.shape[0], net.D_hidden, net.D_out, net.N_atom
    p = {k: v.detach().cpu().double().requires_grad_(True) for k, v in net.p.items()}
    nl = lambda h, lt, nz: onets.noisy_l(h, p[f"mu_w{lt}"], p[f"sig_w{lt}"], p[f"mu_b{lt}"], p[f"sig_b{lt}"], nz)
    pre = F.linear(_head_f64(net, p, x, M, tag), p["l.weight"], p["l.bias"])
    f = pre * _relu_mask(pre, net._buf(tag + "f", (M, H)).cpu(), "l")
    pre = nl(f, "_a1", noise[0])
    xa = pre * _relu_mask(pre, net._buf(tag + "xa", (M, H)).cpu(), "a1")
    pre = nl(f, "_v1", noise[1])
    xv = pre * _relu_mask(pre, net._buf(tag + "xv", (M, H)).cpu(), "v1")
    a = nl(xa, "_a2", noise[2]).reshape(-1, A, K)
    return a - a.mean(1, keepdim=True) + nl(xv, "_v2", noise[3]).reshape(-1, 1, K), p


def _normals(net, seed):
    g = torch.Generator().manual_seed(seed)
    H, AK, K = net.D_hidden, net.D_out * net.N_atom, net.N_atom
    return [(torch.randn(i, generator=g), torch.randn(o, generator=g)) for i, o in ((H, H), (H, H), (H, AK), (H, K))]


NET_CASES = {"cnn_b1": ((4, 84, 84), 4, "cnn", 1), "cnn_b5": ((4, 84, 84), 4, "cnn", 5),
             "cnn_b32": ((4, 84, 84), 4, "cnn", 32), "mlp_cartpole_b32": (4, 2, "mlp", 32)}


@pytest.mark.parametrize("name", list(NET_CASES))
def test_rainbow_network_forward_backward_vs_float64(name):
    D, A, head, M = NET_CASES[name]
    net = _rainbow_net(D, A, 512, head, seed=M + 3)
    g = torch.Generator().manual_seed(M)
    x = (torch.randint(0, 256, (M,) + D, dtype=torch.uint8, generator=g) if head == "cnn"
         else 0.7 * torch.randn(M, D, generator=g))
    dl = torch.randn(M, A * 51, generator=g) * 0.05
    noise = _normals(net, M + 100)
    out = net.forward(x.cuda(), True, tag="t.", noise=[(a.cuda(), b.cuda()) for a, b in noise]).clone()
    net.backward(dl.cuda(), M)
    grads = {k: v.clone() for k, v in net.g.items()}
    net.backward(dl.cuda(), M)
    torch.cuda.synchronize()
    for k, v in net.g.items():
        assert torch.equal(v, grads[k]), f"second backward changed {k}"
    ref, p = _rainbow_f64(net, x, [(a.double(), b.double()) for a, b in noise])
    ref.backward(dl.double().view(M, A, 51))
    _normwise(out, ref, TOL_NET, "logits")
    for k, v in grads.items():
        _normwise(v, p[k].grad, TOL_NET, "grad " + k)


def _philox_noise64(net, ctr, dims):
    """The factors jb_noisy_make draws for the layers `dims` [(tag, stream, in, out)] starting at draw counter ctr (each
    layer bumps it once), returned as float64 normals e = f |f| (sign(e) sqrt|e| gives back f exactly in float64)."""
    c = torch.tensor([ctr], dtype=torch.int64, device="cuda")
    out = []
    for lt, sid, i, o in dims:
        fi, fj, _, _ = _noisy_make(net.p[f"mu_w{lt}"], net.p[f"sig_w{lt}"], net.p[f"mu_b{lt}"], net.p[f"sig_b{lt}"],
                                   seed=net.noise_seed, stream=sid, ctr=c)
        out.append(tuple((f.double() * f.double().abs()).cpu() for f in (fi, fj)))
    return out


def _check_forward_rows(net, dims, ref_fn, nout):
    """forward_rows over 300 CNN rows (chunks of 256 + 44): one draw per layer per call, shared by both chunks."""
    x = torch.randint(0, 256, (300, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(9))
    xd = x.cuda()
    net._draw_ctr.fill_(5)
    out = torch.full((300,) + nout, float("nan"), device="cuda")
    net.forward_rows(xd, out)
    torch.cuda.synchronize()
    assert net._draw_ctr.item() == 5 + len(dims), "forward_rows must draw once per layer per call"
    noise = _philox_noise64(net, 5, dims)
    with torch.no_grad():
        ref = ref_fn({k: v.cpu().double() for k, v in net.p.items()}, x.double(), noise)
    _normwise(out, ref.reshape(out.shape), TOL_NET, "forward_rows output")
    for lo, hi in ((0, 256), (256, 300)):
        net._draw_ctr.fill_(5)
        part = torch.empty((hi - lo,) + nout, device="cuda")
        net.forward_rows(xd[lo:hi], part)
        torch.cuda.synchronize()
        assert torch.equal(part, out[lo:hi]), f"rows {lo}..{hi - 1} did not use the call's weights"


def test_rainbow_forward_rows_draws_once_per_call():
    from oracle import nets as onets
    net = _rainbow_net((4, 84, 84), 4, 512, "cnn", seed=7)
    dims = [("_a1", 1, 512, 512), ("_v1", 2, 512, 512), ("_a2", 3, 512, 204), ("_v2", 4, 512, 51)]
    _check_forward_rows(net, dims, lambda p, x, nz: onets.rainbow_network(p, x, nz, 4, 51), (4, 51))


def test_noisy_forward_rows_draws_once_per_call():
    from jorldy_b200.core.network.noisy import Noisy
    from oracle import nets as onets
    net = _bias(Noisy((4, 84, 84), 4, D_hidden=512, head="cnn", device="cuda", seed=8), 9)
    dims = [("1", 1, 3136, 512), ("2", 2, 512, 4)]
    _check_forward_rows(net, dims, onets.noisy_network, (4,))


# ---- R6: one learn() at the benchmark shapes -------------------------------------------------------------------------
RAINBOW_B32 = LEARN_CASES["rainbow_b32"]
C51_CARTPOLE = dict(seed=61, agent="c51", net="discrete_q_network", D=4, A=2, H=512, B=32, buffer_size=32, K=51,
                    v_min=V_MIN, v_max=V_MAX, gamma=GAMMA, lr=1e-4)


def _dist_f64(case, noise=None):
    from oracle import dqn as odqn
    params, tparams, batch, hp, optim, _ = q_oracle_inputs(case)
    if noise is not None:
        hp = dict(hp, noise=noise)
    elif hp.get("noise") is not None:
        hp = dict(hp, noise=[[(a.double(), b.double()) for a, b in layers] for layers in hp["noise"]])
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        b = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in batch.items()}
        return odqn.dist_learn({k: v.double() for k, v in params.items()}, {k: v.double() for k, v in tparams.items()},
                               b, hp, optim)
    finally:
        torch.set_default_dtype(prev)


def _run_philox(case):
    """The benchmark's path: every forward draws its own Philox noise."""
    agent = _make(case)
    inp = G.q_case_inputs(case)
    batch = {k: torch.from_numpy(inp[k]).cuda() for k in ("state", "next_state", "action", "reward", "done")}
    prio = agent._dist_learn(batch, torch.from_numpy(inp["weights"]).cuda(), 1, [None, None, None])
    torch.cuda.synchronize()
    return agent, prio


def _drawn_noise(agent):
    """The float64 normals behind the factors each of the three forwards drew: online t.*, online n.*, target n.*."""
    net = agent.network
    H, AK, K = net.D_hidden, net.D_out * net.N_atom, net.N_atom
    dims = (("_a1", H, H), ("_v1", H, H), ("_a2", H, AK), ("_v2", H, K))
    out = []
    for n, tag in ((net, "t."), (net, "n."), (agent.target_network, "n.")):
        layers = []
        for lt, i, o in dims:
            f = [n._buf(f"{tag}{lt}.{s}", (m,)).double().cpu() for s, m in (("fi", i), ("fj", o))]
            assert all(bool(v.any()) for v in f), f"{tag}{lt}: no factors drawn"
            layers.append(tuple(v * v.abs() for v in f))
        out.append(layers)
    return out


def _check_learn(case, agent, prio, ref):
    net = agent.network
    st = agent._stats.cpu().numpy()
    X = max(abs(ref["max_logit"]), abs(ref["min_logit"]))
    tol = TOL_NET * (1 + 4 * X)
    for k, g in ref["grads"].items():
        _normwise(net.g[k], g, tol, "grad vs float64 " + k)
    kl_ref = ref["KL"].double()
    kl_bound = (2 * TOL_NET * X + 64 * U) * (1 + kl_ref.abs())
    _within(net._buf("t.kl", (case["B"],)), kl_ref, kl_bound, "kl")
    if "priority" in ref:
        _within(prio, ref["priority"], ALPHA * ref["priority"] * kl_bound / kl_ref + 4 * U * ref["priority"], "priority")
    wmean = float(G.q_case_inputs(case)["weights"].astype(F32).astype(np.float64).mean()) if "priority" in ref else 1.0
    assert abs(st[0] - ref["loss"]) <= wmean * kl_bound.mean().item() + 64 * U * abs(ref["loss"]), "loss"
    assert abs(st[1] - ref["max_Q"]) <= 2 * TOL_NET * X * max(abs(V_MIN), abs(V_MAX)) + 64 * U, "max_Q"
    assert abs(st[2] - ref["max_logit"]) <= TOL_NET * X and abs(st[3] - ref["min_logit"]) <= TOL_NET * X, "logit stats"
    params = G.q_params(case)
    twin = _OptTwin("adam", [torch.from_numpy(params[k]) for k in net.p], case["lr"], 1e-8)
    twin.step([net.g[k] for k in net.p], None)
    state = agent.optimizer.state_dict()["state"]
    for i, k in enumerate(net.p):
        twin.check(i, net.p[k], state[i], k)


def _decisions_agree(case):
    """The float64 oracle decides l / u in float64; on this batch it must agree with the kernels' fp32 decisions except
    in rows terminal at step 0, whose target is continuous in b."""
    inp = G.q_case_inputs(case)
    B, K = case["B"], case["K"]
    r = inp["reward"].reshape(B, -1).astype(F32)
    d = inp["done"].reshape(B, -1).astype(F32)
    b32 = _tz_b(r, d, K)
    z64 = torch.linspace(V_MIN, V_MAX, K, dtype=torch.float64).numpy()
    tz = np.broadcast_to(z64, (B, K))
    for s in range(r.shape[1] - 1, -1, -1):
        tz = r[:, s:s + 1].astype(np.float64) + (1 - d[:, s:s + 1].astype(np.float64)) * GAMMA * tz
    b64 = np.clip(tz - V_MIN, 0, V_MAX - V_MIN) / ((V_MAX - V_MIN) / (K - 1))
    live = d[:, 0] < 0.5
    assert np.array_equal(np.floor(b32)[live], np.floor(b64)[live]) and np.array_equal(np.ceil(b32)[live], np.ceil(b64)[live])


def test_rainbow_learn_injected_noise_vs_float64():
    _decisions_agree(RAINBOW_B32)
    agent, prio = _run(RAINBOW_B32)
    assert torch.equal(agent.z.cpu().view(-1), torch.linspace(V_MIN, V_MAX, 51))
    _check_learn(RAINBOW_B32, agent, prio, _dist_f64(RAINBOW_B32))


def test_rainbow_learn_philox_noise_vs_float64():
    """No injected noise: the float64 reference is built from the factors the three forwards drew."""
    _decisions_agree(RAINBOW_B32)
    agent, prio = _run_philox(RAINBOW_B32)
    assert agent.network._draw_ctr.item() == 8 and agent.target_network._draw_ctr.item() == 4
    _check_learn(RAINBOW_B32, agent, prio, _dist_f64(RAINBOW_B32, noise=_drawn_noise(agent)))


def test_c51_learn_vs_float64():
    _decisions_agree(dict(C51_CARTPOLE, n_step=1))
    agent, prio = _run(C51_CARTPOLE)
    _check_learn(C51_CARTPOLE, agent, prio, _dist_f64(C51_CARTPOLE))


@pytest.mark.parametrize("runner", ["injected", "philox"])
def test_rainbow_learn_is_bit_reproducible(runner):
    run = _run if runner == "injected" else _run_philox
    a1, p1 = run(RAINBOW_B32)
    first = (a1.network.flat.clone(), p1.clone())
    a2, p2 = run(RAINBOW_B32)
    assert torch.equal(first[0], a2.network.flat), "parameters differ between two identical learns"
    assert torch.equal(first[1], p2), "priorities differ between two identical learns"
