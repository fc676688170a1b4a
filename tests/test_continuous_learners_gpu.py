"""The continuous off-policy family (DDPG, TD3, SAC) at the benchmark's shapes against float64: the actor-critic row
kernels of csrc/actor_critic.cu through the C ABI, the state-action critic and the two actors, runs of learns at the
`sac_hopper` shape (D=11, A=3, H=512, B=256) re-anchored on the kernels' own state, and CUDA-graph replays.

Tolerances.  u = 2^-24 is the fp32 unit roundoff; CUDA's tanhf / expf are accurate to 2 ulp and logf to 1 ulp, and
one ulp of x is at most 2u|x|.  Every bound below is a first-order rounding bound of the fp32 computation against
the float64 restatement of the same formula:
  * Elementwise chains (jb_sac_sample, jb_sac_actor_bwd, jb_tanh_*): a chain of at most K_EW = 16 roundings and
    ulp-accurate functions is within K_EW u of the value it would have with every term replaced by its absolute
    value ("the absolute form").  Where a value depends on 1 - a^2 with a = tanh z rounded to fp32, the rounding of
    a*a and of 1 - a*a adds up to 3u absolute to 1 - a^2 (|a| <= 1), which propagates through the derivative of the
    expression in 1 - a^2: that term is written out separately.  Two regions follow from it:
      - float64 region, 1 - a^2 >= 2^-8: the 3u of 1 - a^2 costs at most 3u / (1 - a^2 + 1e-7) <= 768u absolute
        in log(1 - a^2 + 1e-7) and 3u |da| in da (1 - a^2); the reference is float64.
      - saturated region, |z| >= 9.5: 1 - tanh^2 z < 4.5e-8, below half an ulp under 1 (2^-25 = 2.98e-8 is the
        rounding boundary for 1 - tanh z), so fp32 tanh is exactly +-1 on the device and on the CPU, 1 - a*a is 0 and
        the log-prob term is log(1e-7f) exactly.  No float64 value is within rounding of that quantisation, so the
        reference is oracle.actor_critic.sac_sample_action (and the same composite's autograd) in torch-CPU fp32; the
        bound is twice the absolute-form bound of the remaining terms (each side rounds them), and the quantised
        term must agree exactly.
    Elements with 2^-8 > 1 - a^2 and |z| < 9.5 are conditioned by neither reference; their action is still checked
    (tanh is 1-Lipschitz there), their log-prob and gradient only for finiteness.
  * Single-CTA reductions (jb_ac_critic_loss, jb_ac_neg_mean, jb_sac_minq) accumulate ceil(B/256) terms per thread,
    then a 5-level warp tree and an 8-way warp tree: a chain of depth(B) = ceil(B/256) + 10 additions, so a sum is
    within depth(B) u of the sum of absolute values.  The per-row TD target takes 4 roundings, each at most u times
    |r| + gamma (|min nq| + alpha |next_logp|); d q_i = 2 (q_i - y) / B adds the subtraction's and two more.  dq of
    jb_ac_neg_mean and the tie split of jb_sac_minq are exact in fp32 and compared bit for bit.
  * Dense layers (ContinuousQ_Network, DeterministicPolicy, ContinuousPolicy): fp32 FFMA chains.  A contraction of
    n terms is within n u of its absolute form (|W| |x| + |b|), and errors of successive layers add along the path,
    so every output and gradient is checked elementwise against N u times the float64 autograd of the same network
    evaluated on |params|, |inputs| and |d out| with the same ReLU masks ("the absolute chain").  N is the sum of the
    contraction lengths along the longest path, max(D_in) + 4H + B: forward D_in, 2H (l) and H (q / the heads),
    backward H (l dx or dx2) and B (weight gradients).  A ReLU input within rounding of zero may land on either side
    and then passes or blocks a whole gradient, which no rounding bound covers; the float64 reference therefore takes
    the kernels' ReLU masks, after checking that every disagreement sits within N u of its absolute form of zero
    (test_atari_learner_gpu.py's method).
  * Runs of learns: the gradients of one learn are checked normwise per tensor, max|err| <= TOL_LEARN max|ref|,
    TOL_LEARN = N_LEARN u with N_LEARN = 2 (D + 4H) + 2H + B (5.4e3 u ~ 3.2e-4 at H=512, B=256): the
    actor's gradient runs through the target actor / actor forward (D + 2H plus the heads), the critic forward
    (D + 3H), the critics' d q / d action (2H) and the weight-gradient contraction (B).  A sign-mixed fp32 sum of n
    terms rounds to within ~sqrt(n) u sum|t_i| (probabilistic bound) and sum|t_i| <~ sqrt(n) max|ref|, i.e. ~n u
    max|ref| per contraction (test_atari_learner_gpu.py's argument).  SAC's reparameterisation noise is drawn with
    |eps| <= 1.5 so that |z| <= 1.5 e + |mu| ~ 4.4 stays where 1 - a^2 > 5e-4: there the quantisation of a costs at
    most 3u / 5e-4 ~ 3.6e-4 absolute in one log-prob element, about TOL_LEARN, instead of O(1) near saturation.
    The result dict is checked at the same TOL_LEARN against the float64 magnitude of each statistic's terms.
    Parameters are checked against a float64 Adam step that applies the kernel's own gradient, m, v, step and lr:
    m and v are within 3u and 4u of their absolute forms, the update within 16u of itself plus the step size times
    m's bound over the denominator, the parameter within u of itself.  Comparing with an independent fp32 run would
    turn rounding-level gradient differences into O(lr) parameter differences (Adam's first step is lr g / |g|).
    Target networks are checked bit for bit against the soft update tau p + (1 - tau) t in torch-CPU fp32.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"

U = 2.0 ** -24
K_EW = 16
LOG_SQRT_2PI = math.log(math.sqrt(2 * math.pi))
GAMMA = 0.99
G32 = float(np.float32(GAMMA))          # the kernels receive gamma as an fp32 argument
B_VALUES = [1, 255, 256, 257, 1000, 4096]
F64_REGION = 2.0 ** -8                  # 1 - a^2 at or above this: float64 reference
SAT_Z = 9.5                             # |z| at or above this: fp32 tanh is exactly +-1


def _abi():
    from jorldy_b200.core.dev import C, JbError, ptr, stream_ptr
    return C, JbError, ptr, stream_ptr


def _cuda(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(DEV)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _np(t):
    torch.cuda.synchronize()
    return t.detach().cpu().double().numpy()


def _within(got, ref, bound, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    bound = np.broadcast_to(np.asarray(bound, np.float64), ref.shape)
    err = np.abs(got - ref)
    excess = np.where(np.isnan(err), np.inf, err - bound)
    if bool((excess > 0).any()):
        i = int(np.argmax(excess.reshape(-1)))
        raise AssertionError(f"{what}: {int((excess > 0).sum())} of {err.size} elements outside the bound; worst got "
                             f"{got.reshape(-1)[i]:.9g} ref {ref.reshape(-1)[i]:.9g} |err| {err.reshape(-1)[i]:.3e} "
                             f"bound {bound.reshape(-1)[i]:.3e}")


def _depth(B):
    return math.ceil(B / 256) + 10


# =====================================================================================================================
# 1. Row kernels through the C ABI
# =====================================================================================================================
@pytest.mark.parametrize("B", B_VALUES)
@pytest.mark.parametrize("form", ["ddpg", "td3", "sac"])
def test_critic_loss_vs_float64(form, B):
    """DDPG: one critic, no entropy (q2, nq2, alpha, next_logp NULL); TD3: twin critics; SAC: twin critics + entropy."""
    C, _, ptr, sp = _abi()
    rs = np.random.RandomState(B + {"ddpg": 0, "td3": 1, "sac": 2}[form])
    f = lambda *s: rs.standard_normal(s).astype(np.float32)
    q1, q2, nq1, nq2, nlogp, r = 3 * f(B), 3 * f(B), 3 * f(B), 3 * f(B), 2 * f(B), f(B)
    nq2[::5] = nq1[::5]
    alpha = np.float32(0.37)
    twin, sac = form != "ddpg", form == "sac"
    done0 = (rs.uniform(size=B) < 0.3).astype(np.float32)
    for done in (done0, 1 - done0):                    # every row sees done = 0 and done = 1
        dev = {k: _cuda(v) for k, v in dict(q1=q1, q2=q2, nq1=nq1, nq2=nq2, nlogp=nlogp, r=r, d=done,
                                            alpha=[alpha]).items()}
        dq1, dq2, stats = _nan(B), _nan(B), _nan(3)
        C.jb_ac_critic_loss(ptr(dev["q1"]), ptr(dev["q2"]) if twin else 0, ptr(dev["nq1"]), ptr(dev["nq2"]) if twin else 0,
                            ptr(dev["alpha"]) if sac else 0, ptr(dev["nlogp"]) if sac else 0, ptr(dev["r"]), ptr(dev["d"]),
                            B, GAMMA, ptr(dq1), ptr(dq2) if twin else 0, ptr(stats), sp())
        nq = np.minimum(nq1, nq2).astype(np.float64) if twin else nq1.astype(np.float64)
        s_y = np.abs(r) + G32 * (np.abs(nq) + (float(alpha) * np.abs(nlogp) if sac else 0.0))
        if sac:
            nq = nq + float(alpha) * -nlogp.astype(np.float64)
        y = r + (1.0 - done) * G32 * nq
        st = _np(stats)
        _within(st[2], y.max(), 4 * U * s_y.max(), f"{form} B={B} max y")
        for i, (q, dq) in enumerate(((q1, dq1), (q2, dq2))):
            if i == 1 and not twin:
                assert st[1] == 0.0, "DDPG form: stats[1] must be 0"
                assert torch.isnan(dq2).all(), "DDPG form wrote dq2"
                continue
            e = q - y
            e_err = 4 * U * s_y + U * (np.abs(q) + np.abs(y))
            _within(_np(dq), 2 * e / B, (2.0 / B) * (e_err + 2 * U * np.abs(e)), f"{form} B={B} dq{i + 1}")
            loss_b = (2 * np.abs(e) * e_err + e_err ** 2).sum() / B + (_depth(B) + 2) * U * (e * e).mean()
            _within(st[i], (e * e).mean(), loss_b, f"{form} B={B} loss{i + 1}")


@pytest.mark.parametrize("B", B_VALUES)
def test_neg_mean_and_minq_vs_float64(B):
    C, _, ptr, sp = _abi()
    rs = np.random.RandomState(B)
    f = lambda *s: rs.standard_normal(s).astype(np.float32)
    inv = np.float32(1) / np.float32(B)
    # -mean(q): dq = -1/B exactly
    q = 3 * f(B)
    dq, stat, qd = _nan(B), _nan(1), _cuda(q)
    C.jb_ac_neg_mean(ptr(qd), B, ptr(dq), ptr(stat), sp())
    assert bool((dq == -torch.tensor(float(inv))).all()), "neg_mean dq != -1/B"
    _within(_np(stat)[0], -q.astype(np.float64).mean(), (_depth(B) + 2) * U * np.abs(q).mean(), f"B={B} -mean q")
    # SAC actor objective: d min(q1, q2): -1/B to the smaller critic, -1/(2B) to each on ties
    q1, q2, logp = 3 * f(B), 3 * f(B), 2 * f(B)
    q2[::3] = q1[::3]
    al, te = np.float32(0.37), -3.0
    dq1, dq2, st = _nan(B), _nan(B), _nan(4)
    dev = [_cuda(v) for v in (q1, q2, logp, [al])]          # held: a freed temporary's block is reused at once
    C.jb_sac_minq(*map(ptr, dev), te, B, ptr(dq1), ptr(dq2), ptr(st), sp())
    tie = q1 == q2
    want1 = np.where(q1 < q2, -inv, np.where(tie, np.float32(-0.5) * inv, np.float32(0)))
    want2 = np.where(q2 < q1, -inv, np.where(tie, np.float32(-0.5) * inv, np.float32(0)))
    assert np.array_equal(_np(dq1), want1) and np.array_equal(_np(dq2), want2), "minq gradient (ties split in half)"
    assert tie.any()
    mn = np.minimum(q1, q2).astype(np.float64)
    ent = -logp.astype(np.float64)
    d = _depth(B)
    st = _np(st)
    _within(st[0], -(float(al) * ent + mn).mean(), (d + 3) * U * (float(al) * np.abs(ent) + np.abs(mn)).mean(), "actor loss")
    _within(st[1], mn.mean(), (d + 2) * U * np.abs(mn).mean(), "mean min q")
    _within(st[2], ent.mean(), (d + 2) * U * np.abs(ent).mean(), "entropy")
    _within(st[3], ent.mean() - te, (d + 2) * U * np.abs(ent).mean() + U * (abs(ent.mean()) + abs(te)), "entropy - target")


# ---- SAC sample / backward ------------------------------------------------------------------------------------------
EDGE = [(m, l, e) for m in (4.99, -4.99, 5.0, -5.0, 7.0, -7.0) for l in (20.0, -20.0, 0.3)
        for e in (6.0, -6.0, 3.0, -3.0, 0.5, -0.5, 0.0)]
SAMPLE_M = 300


def _sac_inputs(A, nout, seed):
    """raw [M, nout] (padding columns NaN, so a wrong stride shows), eps [M, A].  Edge element k sits at (k, k % A):
    raw_mu at +-4.99, exactly +-5 and +-7, raw_log_std at +-20 (tanh saturates, std = e^+-1), eps up to +-6."""
    rs = np.random.RandomState(seed)
    M = SAMPLE_M
    raw = np.full((M, nout), np.nan, np.float32)
    raw[:, :A] = 0.5 * rs.standard_normal((M, A))
    raw[:, A:2 * A] = 0.5 * rs.standard_normal((M, A))
    eps = rs.standard_normal((M, A)).astype(np.float32)
    for k, (m, l, e) in enumerate(EDGE):
        raw[k, k % A], raw[k, A + k % A], eps[k, k % A] = m, l, e
    return raw, eps


def _sample_f64(raw, eps, A):
    r, e = raw.astype(np.float64), eps.astype(np.float64)
    mu, t = np.clip(r[:, :A], -5, 5), np.tanh(r[:, A:2 * A])
    sd = np.exp(t)
    z = mu + e * sd
    a = np.tanh(z)
    om = 1 - a * a
    t1 = (z - mu) ** 2 / (2 * sd * sd)
    logw = np.log(om + 1e-7)
    lp = -t1 - t - LOG_SQRT_2PI - logw
    # absolute-form bounds (module docstring)
    e_a = K_EW * U * (np.abs(a) + om * (np.abs(e * sd) + np.abs(mu)))
    e_rest = K_EW * U * (t1 + np.abs(t) + LOG_SQRT_2PI + np.abs(logw) + np.abs(e) * (np.abs(e) + np.abs(z) / sd))
    e_log = (2 * np.abs(a) * e_a + 3 * U) / (om + 1e-7)
    return dict(mu=mu, t=t, sd=sd, z=z, a=a, om=om, lp=lp, e_a=e_a, e_rest=e_rest, e_log=e_log)


def _sample_fp32(raw, eps, A):
    """oracle.actor_critic.sac_sample_action in torch-CPU fp32, one log-prob per element."""
    from oracle import actor_critic as oac
    r = torch.from_numpy(np.ascontiguousarray(raw[:, :2 * A]))
    mu, sd = torch.clamp(r[:, :A], -5.0, 5.0), torch.tanh(r[:, A:]).exp()
    e = torch.from_numpy(eps)
    cols = [oac.sac_sample_action(mu[:, j:j + 1], sd[:, j:j + 1], e[:, j:j + 1]) for j in range(A)]
    return torch.cat([c[0] for c in cols], 1).double().numpy(), torch.cat([c[1] for c in cols], 1).double().numpy()


@pytest.mark.parametrize("A", [1, 3, 6, 8])
@pytest.mark.parametrize("pad", [0, 3])
def test_sac_sample_vs_float64_and_fp32_saturation(A, pad):
    C, _, ptr, sp = _abi()
    nout = 2 * A + pad
    raw, eps = _sac_inputs(A, nout, seed=10 * A + pad)
    M = SAMPLE_M
    act, logp = _nan(M, A), _nan(M)
    rd, ed = _cuda(raw), _cuda(eps)
    C.jb_sac_sample(ptr(rd), nout, ptr(ed), M, A, ptr(act), ptr(logp), sp())
    ref = _sample_f64(raw, eps, A)
    a_k, lp_k = _np(act), _np(logp)
    _within(a_k, ref["a"], ref["e_a"], f"A={A} nout={nout} action")
    sat = np.abs(ref["z"]) >= SAT_Z
    f64 = ref["om"] >= F64_REGION
    a32, lp32 = _sample_fp32(raw, eps, A)
    assert np.array_equal(a_k[sat], np.sign(ref["z"][sat])) and np.array_equal(a32[sat], np.sign(ref["z"][sat])), \
        "tanh of |z| >= 9.5 must round to exactly +-1 in fp32"
    lp_el = np.where(sat, lp32, ref["lp"])
    b_el = np.where(sat, 2 * ref["e_rest"], ref["e_rest"] + ref["e_log"])
    rows = (sat | f64).all(1)
    assert rows.sum() >= M // 2 and (rows & sat.any(1)).sum() >= 8, (rows.sum(), (rows & sat.any(1)).sum())
    bound = b_el.sum(1) + A * U * np.abs(lp_el).sum(1)
    _within(lp_k[rows], lp_el.sum(1)[rows], bound[rows], f"A={A} nout={nout} log-prob")
    assert np.isfinite(lp_k).all()


def _actor_bwd_ref(raw, eps, da, alpha, B, A, dtype):
    """Autograd of the composite: clamp, tanh/exp of log_std, rsample, tanh, the log-prob with its 1e-7, and the
    alpha * logp / B term; the action's own gradient is da."""
    from oracle import actor_critic as oac
    r = torch.tensor(raw, dtype=dtype, requires_grad=True)
    mu, sd = torch.clamp(r[:, :A], -5.0, 5.0), torch.tanh(r[:, A:]).exp()
    a, logp = oac.sac_sample_action(mu, sd, torch.tensor(eps, dtype=dtype))
    ((torch.tensor(da, dtype=dtype) * a).sum() + torch.tensor(alpha, dtype=dtype) / B * logp.sum()).backward()
    return r.grad.double().numpy()


@pytest.mark.parametrize("A", [1, 3, 6, 8])
def test_sac_actor_bwd_vs_float64_autograd(A):
    C, JbError, ptr, sp = _abi()
    raw, eps = _sac_inputs(A, 2 * A, seed=100 + A)
    M = B = SAMPLE_M
    ref = _sample_f64(raw, eps, A)
    act = ref["a"].astype(np.float32)                     # the sampled action, rounded once
    rs = np.random.RandomState(A)
    da = (rs.standard_normal((M, A)) / B).astype(np.float32)
    alpha = np.float32(0.37)
    dout = _nan(M, 2 * A)
    rd, ed, ad, dad, ald = (_cuda(v) for v in (raw, eps, act, da, [alpha]))
    C.jb_sac_actor_bwd(ptr(rd), 2 * A, ptr(ed), ptr(ad), ptr(dad), ptr(ald), B, A, ptr(dout), sp())
    got = _np(dout)
    g64 = _actor_bwd_ref(raw, eps, da, float(alpha), B, A, torch.float64)
    g32 = _actor_bwd_ref(raw, eps, da, float(alpha), B, A, torch.float32)
    om, a, sd, t, e = ref["om"], ref["a"], ref["sd"], ref["t"], eps.astype(np.float64)
    ab = float(alpha) / B
    rr = om / (om + 1e-7)
    gz = da * om + ab * 2 * a * rr
    e_gz = K_EW * U * (np.abs(da) * om + ab * 2 * np.abs(a) * rr) + 3 * U * np.abs(da) \
        + ab * 2 * np.abs(a) * 1e-7 * 3 * U / (om + 1e-7) ** 2
    abs_gs = np.abs(gz * e) + ab / sd
    e_gs = np.abs(e) * e_gz + K_EW * U * abs_gs
    e_ls = (e_gs * (1 - t * t) + abs_gs * (K_EW * U * (1 - t * t) + 3 * U)) * sd
    rmu = raw[:, :A].astype(np.float64)
    beyond = np.abs(rmu) > 5
    sat, f64 = np.abs(ref["z"]) >= SAT_Z, om >= F64_REGION
    e_sat = 2 * K_EW * U * (abs_gs + ab * e * e / sd) * sd
    want = np.where(np.concatenate([sat, sat], 1), g32, g64)
    bound = np.concatenate([np.where(sat, e_sat, np.where(beyond, 0.0, e_gz)), np.where(sat, e_sat, e_ls)], 1)
    mask = np.concatenate([sat | f64, sat | f64], 1)
    assert (sat & ~beyond).any() and (f64 & (np.abs(rmu) == 5)).any() and (f64 & beyond).any()
    _within(got[mask], want[mask], bound[mask], f"A={A} d raw")
    assert (got[:, :A][beyond] == 0).all(), "gradient past the +-5 clamp must be 0"
    assert np.isfinite(got).all()
    for bad in (2 * A - 1, 2 * A + 1):
        with pytest.raises(JbError):
            C.jb_sac_actor_bwd(ptr(rd), bad, ptr(ed), ptr(ad), ptr(dad), ptr(ald), B, A, ptr(dout), sp())


def test_sac_alpha():
    C, _, ptr, sp = _abi()
    stats4 = _cuda([1.5, -0.25, 2.75, -1.25])
    for la in (-2.0, 0.0, 0.7):
        la32 = np.float32(la)
        alpha, grad, loss, lad = _nan(1), _nan(1), _nan(1), _cuda([la32])
        C.jb_sac_alpha(ptr(lad), ptr(stats4), ptr(alpha), ptr(grad), ptr(loss), sp())
        assert _np(grad)[0] == -1.25
        _within(_np(loss)[0], float(la32) * -1.25, U * abs(float(la32) * 1.25), "alpha_loss")
        _within(_np(alpha)[0], math.exp(float(la32)), 4 * U * math.exp(float(la32)), "alpha")
        alpha2, loss2 = _nan(1), _nan(1)
        C.jb_sac_alpha(ptr(lad), ptr(stats4), ptr(alpha2), 0, ptr(loss2), sp())     # static alpha: no grad
        assert torch.equal(alpha2, alpha) and torch.equal(loss2, loss)


def test_tanh_act_and_bwd_vs_float64():
    C, _, ptr, sp = _abi()
    rs = np.random.RandomState(4)
    pre = (2 * rs.standard_normal(1003)).astype(np.float32)
    pre[:8] = [0.0, 20.0, -20.0, SAT_Z, -SAT_Z, 3.0, -3.0, 1e-30]
    noise = rs.standard_normal(1003).astype(np.float32)
    noise[8:16] = [2.5, -2.5, 5.0, -5.0, 2.5, -2.5, 2.5, -2.5]          # noise * 0.2 exactly +-0.5, and beyond it
    pre[12:16] = [3.0, -3.0, 0.2, -0.2]                                 # tanh + 0.5 beyond +-1, and inside
    assert np.float32(2.5) * np.float32(0.2) == np.float32(0.5)
    n = pre.size
    pd, nd = _cuda(pre), _cuda(noise)
    t = np.tanh(pre.astype(np.float64))
    out = _nan(n)
    C.jb_tanh_act(ptr(pd), 0, n, 0.0, 0.0, 0.0, ptr(out), sp())         # policy head: tanh only
    a_plain = _np(out)
    _within(a_plain, t, 4 * U * np.abs(t), "tanh")
    assert (np.abs(a_plain[np.abs(pre) >= SAT_Z]) == 1).all()
    for scale, clip in ((0.1, 0.0), (0.2, 0.5)):                        # TD3 act noise; TD3 target smoothing
        out = _nan(n)
        C.jb_tanh_act(ptr(pd), ptr(nd), n, scale, clip, 1.0, ptr(out), sp())
        ns = noise.astype(np.float64) * float(np.float32(scale))
        z = np.clip(ns, -float(np.float32(clip)), float(np.float32(clip))) if clip else ns
        want = np.clip(t + z, -1, 1)
        got = _np(out)
        _within(got, want, 4 * U * np.abs(t) + U * np.abs(ns) + U * np.abs(t + z), f"tanh + noise (scale {scale}, clip {clip})")
        assert (np.abs(got[np.abs(t + z) > 1 + 1e-6]) == 1).all(), "outputs beyond +-1 clip to exactly +-1"
    # dpre = da (1 - a^2) at the kernel's own a, including |pre| large where a = +-1 and the gradient is 0
    da = rs.standard_normal(n).astype(np.float32)
    dpre, dad, ad = _nan(n), _cuda(da), _cuda(a_plain)
    C.jb_tanh_bwd(ptr(dad), ptr(ad), n, ptr(dpre), sp())
    want = da * (1 - a_plain * a_plain)
    got = _np(dpre)
    _within(got, want, 3 * U * np.abs(da) + U * np.abs(want), "tanh backward")
    assert (got[np.abs(pre) >= SAT_Z] == 0).all()


def test_ou_act_vs_oracle():
    """Several steps with the f64 state X carried across calls; the greedy path; the Philox path."""
    from oracle import actor_critic as oac
    C, _, ptr, sp = _abi()
    M, A = 300, 3
    theta, mu, sigma = 0.15, 0.1, 0.2
    rs = np.random.RandomState(8)
    pre = (2 * rs.standard_normal((M, A))).astype(np.float32)
    pre[0] = [20.0, -20.0, 0.0]
    x0 = 0.5 * rs.standard_normal((M, A))
    t = np.tanh(pre.astype(np.float64))
    pd = _cuda(pre)
    X = torch.tensor(x0, dtype=torch.float64, device=DEV)
    ctr = torch.zeros(M, dtype=torch.int64, device=DEV)
    act = _nan(M, A)
    xr, e_x = x0.copy(), np.zeros((M, A))
    for step in range(4):
        nrm = rs.standard_normal(M) * (3.0 if step == 2 else 1.0)       # step 2 drives X past the +-1 clip
        nd = _cuda(nrm, torch.float64)
        C.jb_ou_act(ptr(pd), M, A, ptr(X), ptr(nd), 7, 0, ptr(ctr), theta, mu, sigma, 0, ptr(act), sp())
        dx_abs = np.abs(xr) + theta * np.abs(mu - xr) + sigma * np.abs(nrm)[:, None]
        xr = np.concatenate([oac.ou_step(xr[m:m + 1], mu, theta, sigma, nrm[m]) for m in range(M)])
        e_x += 4 * 2.0 ** -53 * dx_abs
        _within(_np(X), xr, e_x, f"step {step} X")
        want = t + np.clip(xr, -1, 1)
        _within(_np(act), want, 4 * U * np.abs(t) + U * np.abs(want) + e_x, f"step {step} action")
    assert (np.abs(xr) > 1).any()
    assert int(ctr.abs().sum()) == 0, "injected normals must not advance the Philox row counters"
    Xg = X.clone()
    C.jb_ou_act(ptr(pd), M, A, ptr(X), 0, 7, 0, ptr(ctr), theta, mu, sigma, 1, ptr(act), sp())  # greedy
    _within(_np(act), t, 4 * U * np.abs(t), "greedy action")
    assert torch.equal(X, Xg) and int(ctr.abs().sum()) == 0
    # Philox: each call draws Philox(seed, stream_base + m, row_ctr[m]) -> the first Box-Muller output, one per env
    # and step, shared by the A dimensions; row_ctr[m] advances by one per call
    base = 1 << 20
    for call in range(2):
        X.copy_(torch.tensor(x0, device=DEV))
        C.jb_ou_act(ptr(pd), M, A, ptr(X), 0, 7, base, ptr(ctr), theta, mu, sigma, 0, ptr(act), sp())
        assert bool((ctr == call + 1).all()), "row counters advance by one per call"
        implied = (_np(X) - x0 - theta * (mu - x0)) / sigma
        pair = torch.empty(2 * M, device=DEV)
        C.jb_philox_fill(ptr(pair), 2 * M, 0, 0.0, 1.0, 7, base, call, 0, sp())
        np.testing.assert_allclose(implied, np.repeat(_np(pair)[0::2, None], A, 1), rtol=0, atol=1e-12,
                                   err_msg=f"call {call}: implied normal")
        if call == 0:
            first = implied[:, 0].copy()
    assert (implied[:, 0] != first).all(), "the second call draws fresh normals"


def test_philox_fill():
    from scipy import stats
    C, _, ptr, sp = _abi()
    n = 100_001                                                   # odd: the last pair's second slot lies past the end
    out = torch.full((n + 4,), 7.0, device=DEV)
    C.jb_philox_fill(ptr(out), n, 0, 0.0, 1.0, 123, 5, 0, 0, sp())
    x = _np(out)
    assert (x[n:] == 7.0).all(), "written past n"
    assert stats.kstest(x[:n], "norm").pvalue > 1e-3
    lo, hi = -2.5, 0.5
    C.jb_philox_fill(ptr(out), n, 1, lo, hi, 123, 5, 0, 0, sp())
    x = _np(out)
    assert (x[n:] == 7.0).all() and x[:n].min() >= lo and x[:n].max() < hi
    assert stats.kstest(x[:n], "uniform", args=(lo, hi - lo)).pvalue > 1e-3
    # device counter: pair p draws at ctr + ctr_dev[0], then ctr_dev[0] += 1
    cd = torch.tensor([5], dtype=torch.int64, device=DEV)
    a, b, c = torch.empty(999, device=DEV), torch.empty(999, device=DEV), torch.empty(999, device=DEV)
    C.jb_philox_fill(ptr(a), 999, 0, 0.0, 1.0, 9, 3, 2, ptr(cd), sp())
    C.jb_philox_fill(ptr(b), 999, 0, 0.0, 1.0, 9, 3, 7, 0, sp())
    C.jb_philox_fill(ptr(c), 999, 0, 0.0, 1.0, 9, 3, 2, ptr(cd), sp())
    torch.cuda.synchronize()
    assert torch.equal(a, b) and int(cd.item()) == 7 and not torch.equal(a, c)


def test_invalid_shapes_are_rejected():
    C, JbError, ptr, sp = _abi()
    buf = torch.zeros(64, 32, device=DEV)
    p = ptr(buf)
    with pytest.raises(JbError):
        C.jb_sac_sample(p, 18, p, 4, 9, p, p, sp())                   # A over AC_MAX_A = 8
    with pytest.raises(JbError):
        C.jb_sac_sample(p, 5, p, 4, 3, p, p, sp())                    # nout < 2A
    with pytest.raises(JbError):
        C.jb_sac_actor_bwd(p, 18, p, p, p, p, 4, 9, p, sp())          # A over AC_MAX_A = 8
    with pytest.raises(JbError):
        C.jb_sac_actor_bwd(p, 5, p, p, p, p, 4, 3, p, sp())           # nout < 2A


# =====================================================================================================================
# 2. The state-action critic and the two actors against float64 autograd
# =====================================================================================================================
def _relu(pre, mask):
    return torch.relu(pre) if mask is None else pre * mask


def _q64(p, x1, x2, masks=None):
    """oracle.actor_critic.continuous_q_network with each ReLU optionally replaced by a 0/1 mask; returns (q, pres)."""
    m = masks or (None, None, None)
    p1 = F.linear(x1, p["head.l.weight"], p["head.l.bias"])
    p2 = F.linear(x2, p["e.weight"], p["e.bias"])
    p3 = F.linear(torch.cat([_relu(p1, m[0]), _relu(p2, m[1])], dim=-1), p["l.weight"], p["l.bias"])
    return F.linear(_relu(p3, m[2]), p["q.weight"], p["q.bias"]), (p1, p2, p3)


def _pol64(p, x, heads, masks=None):
    """The actors' trunk + heads before their activations (forward_raw); returns (out, pres)."""
    m = masks or (None, None)
    p1 = F.linear(x, p["head.l.weight"], p["head.l.bias"])
    p2 = F.linear(_relu(p1, m[0]), p["l.weight"], p["l.bias"])
    h = _relu(p2, m[1])
    return torch.cat([F.linear(h, p[f"{n}.weight"], p[f"{n}.bias"]) for n in heads], dim=-1), (p1, p2)


def _leaf(net, absval=False):
    return {k: (v.detach().cpu().double().abs() if absval else v.detach().cpu().double()).requires_grad_(True)
            for k, v in net.p.items()}


def _mask(pre, pre_abs, out, n, what):
    """The kernel's ReLU decision (out > 0); a disagreement with the float64 sign must sit within n u of zero."""
    keep = out.cpu() > 0
    differ = keep != (pre.detach() > 0)
    assert bool((pre.detach().abs()[differ] <= n * U * pre_abs.detach()[differ]).all()), f"{what}: mask differs away from 0"
    return keep.double()


def _random_biases(net, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, v in net.p.items():
            if k.endswith(".bias"):
                v.copy_(0.1 * torch.randn(v.shape, generator=g))


Q_DIMS = [(3, 1), (11, 3), (17, 6), (11, 8)]


def _q_case(B, d1, d2, H, seed):
    from jorldy_b200.core.network.q_network import ContinuousQ_Network
    net = ContinuousQ_Network(d1, d2, D_hidden=H, device=DEV, seed=seed)
    _random_biases(net, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    x1 = 0.7 * torch.randn(B, d1, generator=g)
    x2 = torch.tanh(torch.randn(B, d2, generator=g))
    dq = torch.randn(B, 1, generator=g) / B
    return net, x1, x2, dq


def _q_reference(net, x1, x2, dq, B, n):
    """Float64 value and absolute chain of q, every parameter gradient and d q / d x2, with the kernel's masks."""
    H = net.D_hidden
    p, pa = _leaf(net), _leaf(net, absval=True)
    x1d, x2d = x1.double(), x2.double().requires_grad_(True)
    x2a = x2.double().abs().requires_grad_(True)
    q_plain, pres = _q64(p, x1d, x2d)
    _, pres_abs = _q64(pa, x1d.abs(), x2a.detach())
    cat, h2 = net._buf("t.cat", (B, 2 * H)), net._buf("t.h2", (B, H))
    d_in = max(net.D_in1, net.D_in2)
    masks = (_mask(pres[0], pres_abs[0], cat[:, :H], d_in, "head"), _mask(pres[1], pres_abs[1], cat[:, H:], d_in, "e"),
             _mask(pres[2], pres_abs[2], h2, d_in + 2 * H, "l"))
    from oracle import actor_critic as oac
    with torch.no_grad():
        torch.testing.assert_close(q_plain.detach(), oac.continuous_q_network(p, x1d, x2d), rtol=1e-12, atol=1e-12)
    q, _ = _q64(p, x1d, x2d, masks)
    q.backward(dq.double())
    qa, _ = _q64(pa, x1d.abs(), x2a, masks)
    qa.backward(dq.double().abs())
    return q.detach(), qa.detach(), p, pa, x2d.grad, x2a.grad


@pytest.mark.parametrize("H", [64, 512])
@pytest.mark.parametrize("d1,d2", Q_DIMS)
@pytest.mark.parametrize("B", [1, 37, 256, 1024])
def test_continuous_q_network_vs_float64(B, d1, d2, H):
    net, x1, x2, dq = _q_case(B, d1, d2, H, seed=B + 10 * d1 + d2 + H)
    q = net.forward(x1.to(DEV), x2.to(DEV), tag="t.").clone()
    dx2 = net.backward(dq.to(DEV), B, tag="t.", params=True, want_dx2=True).clone()
    torch.cuda.synchronize()
    n = max(d1, d2) + 4 * H + B
    q_ref, q_abs, p, pa, dx2_ref, dx2_abs = _q_reference(net, x1, x2, dq, B, n)
    _within(_np(q), q_ref.numpy(), (max(d1, d2) + 3 * H) * U * q_abs.numpy(), "q")
    for k in net.p:
        _within(_np(net.g[k]), p[k].grad.numpy(), n * U * pa[k].grad.numpy(), "grad " + k)
    _within(_np(dx2), dx2_ref.numpy(), n * U * dx2_abs.numpy(), "dx2")


@pytest.mark.parametrize("d2", [3, 8])
def test_continuous_q_network_dx2_accumulates(d2):
    """Critic 2 adds its d q / d action onto critic 1's (jb_gemm accumulate = 1 on the [B, A] output): the result must be
    prefill + own contribution.  A = 3 takes the generic 32x32 kernel (ldb = 3), A = 8 the cp.async panel kernel."""
    B, d1, H = 256, 11, 512
    net, x1, x2, dq = _q_case(B, d1, d2, H, seed=77 + d2)
    net.forward(x1.to(DEV), x2.to(DEV), tag="t.")
    prefill = 10 * torch.randn(B, d2, generator=torch.Generator().manual_seed(5))
    buf = prefill.to(DEV)
    out = net.backward(dq.to(DEV), B, tag="t.", params=False, want_dx2=True, dx2=buf, accumulate=True)
    assert out.data_ptr() == buf.data_ptr()
    torch.cuda.synchronize()
    n = max(d1, d2) + 4 * H + B
    _, _, _, _, dx2_ref, dx2_abs = _q_reference(net, x1, x2, dq, B, n)
    want = prefill.double() + dx2_ref
    _within(_np(buf), want.numpy(), n * U * dx2_abs.numpy() + U * want.abs().numpy(), "prefill + dx2")


POL_DIMS = [(3, 1), (11, 3), (17, 6), (11, 8)]


@pytest.mark.parametrize("H", [64, 512])
@pytest.mark.parametrize("D,A", POL_DIMS)
@pytest.mark.parametrize("B", [1, 37, 256, 1024])
@pytest.mark.parametrize("kind", ["deterministic", "continuous"])
def test_policy_forward_backward_vs_float64(kind, B, D, A, H):
    from oracle import actor_critic as oac
    from jorldy_b200.core.network.policy import ContinuousPolicy, DeterministicPolicy
    seed = B + 10 * D + A + H
    cls, heads = (DeterministicPolicy, ("pi",)) if kind == "deterministic" else (ContinuousPolicy, ("mu", "log_std"))
    net = cls(D, A, D_hidden=H, device=DEV, seed=seed)
    _random_biases(net, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    x = 0.7 * torch.randn(B, D, generator=g)
    dout = torch.randn(B, len(heads) * A, generator=g) / B
    out = net.forward_raw(x.to(DEV), tag="t.").clone()
    net.backward_raw(dout.to(DEV), B, tag="t.")
    torch.cuda.synchronize()
    n = D + 4 * H + B
    p, pa = _leaf(net), _leaf(net, absval=True)
    xd = x.double()
    plain, pres = _pol64(p, xd, heads)
    _, pres_abs = _pol64(pa, xd.abs(), heads)
    with torch.no_grad():
        if kind == "deterministic":
            torch.testing.assert_close(torch.tanh(plain), oac.deterministic_policy(p, xd), rtol=1e-12, atol=1e-12)
        else:
            mu, sd = oac.continuous_policy(p, xd)
            torch.testing.assert_close(torch.clamp(plain[:, :A], -5, 5), mu, rtol=1e-12, atol=1e-12)
            torch.testing.assert_close(torch.tanh(plain[:, A:]).exp(), sd, rtol=1e-12, atol=1e-12)
    masks = (_mask(pres[0], pres_abs[0], net._buf("t.head.h", (B, H)), D, "head"),
             _mask(pres[1], pres_abs[1], net._buf("t.h2", (B, H)), D + H, "l"))
    ref, _ = _pol64(p, xd, heads, masks)
    ref.backward(dout.double())
    ref_abs, _ = _pol64(pa, xd.abs(), heads, masks)
    ref_abs.backward(dout.double().abs())
    _within(_np(out), ref.detach().numpy(), (D + 2 * H) * U * ref_abs.detach().numpy(), "forward_raw")
    for k in net.p:
        _within(_np(net.g[k]), p[k].grad.numpy(), n * U * pa[k].grad.numpy(), "grad " + k)


# =====================================================================================================================
# 3. Runs of learns at the sac_hopper shape, re-anchored on the kernels' own state
# =====================================================================================================================
BENCH_OPTIM = {"actor": "adam", "critic": "adam", "alpha": "adam", "actor_lr": 5e-4, "critic_lr": 1e-3, "alpha_lr": 3e-4}
N_REPLAY, RUN_STEP = 2048, 40          # cos(pi/2 * step / 40): lr falls by 0.1 % to 5 % over the first eight learns


def _make_agent(kind, D, A, B, use_cuda_graph=False, **extra):
    from jorldy_b200.core import Agent
    torch.manual_seed(1000 + D + A)        # the networks' orthogonal init draws from torch's default generator
    kw = dict(state_size=D, action_size=A, hidden_size=512, optim_config=dict(BENCH_OPTIM), gamma=GAMMA,
              buffer_size=N_REPLAY, batch_size=B, start_train_step=0, run_step=RUN_STEP, lr_decay=True, device=DEV,
              seed=3, use_cuda_graph=use_cuda_graph)
    if kind == "sac":
        kw.update(tau=5e-3)
    if kind == "td3":
        kw.update(update_delay=2)
    kw.update(extra)
    return Agent(kind, **kw)


def _replay(D, A, seed):
    rs = np.random.RandomState(seed)
    n = N_REPLAY
    return {"state": (0.7 * rs.standard_normal((n, D))).astype(np.float32),
            "next_state": (0.7 * rs.standard_normal((n, D))).astype(np.float32),
            "action": np.tanh(rs.standard_normal((n, A))).astype(np.float32), "reward": rs.standard_normal((n, 1)),
            "done": rs.uniform(size=(n, 1)) < 0.2}


def _nets(agent):
    out = {"actor": agent.actor}
    for i, c in enumerate(agent.critics):
        out[f"critic{i + 1}"] = c
        out[f"target_critic{i + 1}"] = agent.target_critics[i]
    if hasattr(agent, "target_actor"):
        out["target_actor"] = agent.target_actor
    return out


def _opts(agent):
    out = {"actor": (agent.actor, agent.actor_optimizer)}
    for i, (c, o) in enumerate(zip(agent.critics, agent.critic_optimizers)):
        out[f"critic{i + 1}"] = (c, o)
    if getattr(agent, "alpha_optimizer", None) is not None:
        out["log_alpha"] = (agent.log_alpha, agent.alpha_optimizer)
    return out


def _snapshot(agent):
    torch.cuda.synchronize()
    snap = {"p": {k: n.flat.detach().cpu().clone() for k, n in _nets(agent).items()},
            "opt": {k: (o.exp_avg.cpu().clone(), o.exp_avg_sq.cpu().clone(), int(o._step_dev.item()),
                        float(np.float32(o.param_groups[0]["lr"]))) for k, (_, o) in _opts(agent).items()}}
    if hasattr(agent, "log_alpha"):
        snap["log_alpha"] = agent.log_alpha.flat[:1].cpu().clone()
        snap["alpha"] = agent.alpha.cpu().clone()
    return snap


def _params64(net, flat):
    """Named float64 CPU views of a flat fp32 parameter buffer (the kernel's own parameters)."""
    out = {}
    for k, v in net.p.items():
        off = v.storage_offset() - net.flat.storage_offset()
        out[k] = flat[off:off + v.numel()].view(v.shape).double()
    return out


def _normwise(got, ref, tol, what):
    err = (got.detach().cpu().double() - ref.detach().cpu().double()).abs().max().item()
    scale = ref.detach().abs().max().item()
    assert err <= tol * scale, f"{what}: max|err| {err:.3e} > {tol:.2e} * max|ref| {scale:.3e}"


def _check_adam(name, net, opt, snap, tag):
    """The kernel's post-learn parameters, m and v against one float64 Adam step from its pre-learn state with its own
    gradient, step and lr."""
    p0 = snap["p"][name].double() if name in snap["p"] else snap["log_alpha_flat"].double()
    m0, v0, step0, lr = (t if isinstance(t, (int, float)) else t.double() for t in snap["opt"][name])
    g = net.grad.detach().cpu().double()
    b1, b2, eps = 0.9, 0.999, 1e-8
    step = step0 + 1
    assert int(opt._step_dev.item()) == step
    m = b1 * m0 + (1 - b1) * g
    v = b2 * v0 + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    den = v.sqrt() / math.sqrt(bc2) + eps
    upd = lr / bc1 * m / den
    p = p0 - upd
    e_m = 3 * U * (m0.abs() + g.abs())
    _within(opt.exp_avg.cpu(), m, e_m, f"{tag} {name} exp_avg")
    _within(opt.exp_avg_sq.cpu(), v, 4 * U * (b2 * v0 + (1 - b2) * g * g), f"{tag} {name} exp_avg_sq")
    _within(net.flat.detach().cpu(), p, U * p.abs() + 16 * U * upd.abs() + lr / bc1 * e_m / den, f"{tag} {name} param")


def _check_soft(agent, snap, pairs, tag):
    tau = float(agent.tau)
    nets = _nets(agent)
    for t, o in pairs:
        want = tau * nets[o].flat.detach().cpu() + (1 - tau) * snap["p"][t]
        assert torch.equal(nets[t].flat.detach().cpu(), want), f"{tag}: {t} != soft update of {o}"


def _sac_sample64(raw, eps, A):
    from oracle import actor_critic as oac
    mu, sd = torch.clamp(raw[:, :A], -5.0, 5.0), torch.tanh(raw[:, A:]).exp()
    return oac.sac_sample_action(mu, sd, eps)


def _learn_reference(kind, agent, snap, batch, noise, num_learn):
    """Float64 gradients and results of one learn at the kernel's pre-learn parameters; the actor's gradient runs
    through the critics as the kernel left them after its critic step (its post-learn critics)."""
    from oracle import actor_critic as oac
    B, A, H = batch["reward"].shape[0], agent.action_size, agent.critics[0].D_hidden
    s, a, r, d, ns = (batch[k] for k in ("state", "action", "reward", "done", "next_state"))
    nets = _nets(agent)
    P = {k: _params64(nets[k], snap["p"][k]) for k in nets}
    post = {k: _params64(nets[k], nets[k].flat.detach().cpu()) for k in nets}
    leaf = lambda d: {k: v.clone().requires_grad_(True) for k, v in d.items()}
    cmask = lambda c, tag: (c._buf(tag + "cat", (B, 2 * H))[:, :H].cpu() > 0, c._buf(tag + "cat", (B, 2 * H))[:, H:].cpu() > 0,
                            c._buf(tag + "h2", (B, H)).cpu() > 0)
    amask = (agent.actor._buf("t.head.h", (B, H)).cpu() > 0, agent.actor._buf("t.h2", (B, H)).cpu() > 0)
    out = {"grads": {}, "res": {}, "scale": {}}
    n_crit = len(agent.critics)
    with torch.no_grad():
        if kind == "sac":
            alpha0 = float(snap["alpha"].item())
            na, nlogp = _sac_sample64(_pol64(P["actor"], ns, ("mu", "log_std"))[0], noise["next"].double(), A)
        else:
            na = oac.deterministic_policy(P["target_actor"], ns)
            if kind == "td3":
                na = (na + (noise["target"].double() * float(np.float32(agent.target_noise_std)))
                      .clamp(-float(np.float32(agent.target_noise_clip)), float(np.float32(agent.target_noise_clip)))).clamp(-1, 1)
        nqs = [oac.continuous_q_network(P[f"target_critic{i + 1}"], ns, na) for i in range(n_crit)]
        nq = torch.min(nqs[0], nqs[1]) if n_crit == 2 else nqs[0]
        y_abs = r.abs() + G32 * nq.abs()
        if kind == "sac":
            nq = nq + alpha0 * -nlogp
            y_abs = y_abs + G32 * alpha0 * nlogp.abs()
        y = r + (1 - d) * G32 * nq
    out["res"]["max_Q"], out["scale"]["max_Q"] = y.max().item(), y_abs.max().item()
    names = ["critic_loss"] if kind == "ddpg" else ["critic_loss1", "critic_loss2"]
    for i in range(n_crit):
        c = f"critic{i + 1}"
        p = leaf(P[c])
        q = _q64(p, s, a, [m.double() for m in cmask(agent.critics[i], "t.")])[0]
        loss = ((q - y) ** 2).mean()
        loss.backward()
        out["grads"][c] = {k: v.grad for k, v in p.items()}
        out["res"][names[i]] = loss.item()
        out["scale"][names[i]] = 2 * ((q.detach().abs() + y.abs()) ** 2).mean().item()
    if kind == "td3" and num_learn % agent.update_delay != 0:
        return out
    pa = leaf(P["actor"])
    amk = [m.double() for m in amask]
    if kind == "sac":
        act, logp = _sac_sample64(_pol64(pa, s, ("mu", "log_std"), amk)[0], noise["actor"].double(), A)
        qs = [_q64(post[f"critic{i + 1}"], s, act, [m.double() for m in cmask(agent.critics[i], "a.")])[0] for i in range(2)]
        minq = torch.min(qs[0], qs[1])
        loss = -(alpha0 * -logp + minq).mean()
        ent = -logp.detach()
        te = agent.target_entropy
        out["alpha_grad"], out["alpha_grad_scale"] = (ent - te).mean().item(), (ent.abs() + abs(te)).mean().item()
        la0 = float(snap["log_alpha"].item())
        out["res"].update(alpha_loss=la0 * out["alpha_grad"], mean_Q=minq.mean().item(), entropy=ent.mean().item(),
                          alpha=math.exp(la0))
        out["scale"].update(alpha_loss=abs(la0) * out["alpha_grad_scale"], mean_Q=minq.detach().abs().mean().item(),
                            entropy=ent.abs().mean().item(), actor_loss=(alpha0 * ent.abs() + minq.detach().abs()).mean().item())
    else:
        act = torch.tanh(_pol64(pa, s, ("pi",), amk)[0])
        q = _q64(post["critic1"], s, act, [m.double() for m in cmask(agent.critics[0], "a.")])[0]
        loss = -q.mean()
        out["scale"]["actor_loss"] = q.detach().abs().mean().item()
    loss.backward()
    out["grads"]["actor"] = {k: v.grad for k, v in pa.items()}
    out["res"]["actor_loss"] = loss.item()
    return out


def _run_learns(kind, D, A, n_learns, seed, **extra):
    B = 256
    agent = _make_agent(kind, D, A, B, **extra)
    agent.memory.store([_replay(D, A, seed)])
    rs = np.random.RandomState(seed + 1)
    tol = (2 * (D + 4 * 512) + 2 * 512 + B) * U
    lrs = []
    for i in range(n_learns):
        tag = f"{kind} D={D} A={A} learn {i}"
        snap = _snapshot(agent)
        if "log_alpha" in _opts(agent):
            snap["log_alpha_flat"] = agent.log_alpha.flat.detach().cpu().clone()
        idx = rs.randint(N_REPLAY, size=B)
        noise = None
        if kind == "sac":
            eps = lambda: torch.from_numpy(np.clip(rs.standard_normal((B, A)), -1.5, 1.5).astype(np.float32))
            noise = {"next": eps(), "actor": eps()}
        elif kind == "td3":
            nz = rs.standard_normal((B, A)).astype(np.float32)
            nz[:4, 0] = [2.5, -2.5, 6.0, -6.0]            # target_noise_std 0.2 x 2.5 = the 0.5 clip exactly, and beyond
            noise = {"target": torch.from_numpy(nz)}
        agent._inject_idx = idx
        agent._inject_noise = {k: v.to(DEV) for k, v in noise.items()} if noise else None
        num_learn = agent.num_learn
        res = agent.learn()
        torch.cuda.synchronize()
        agent._inject_noise = None
        g = agent.memory.gather_device(torch.as_tensor(idx, device=DEV))
        f = lambda k, w: g[k].to(torch.float32).reshape(B, w).cpu().double()
        batch = {"state": f("state", D), "action": f("action", A), "reward": f("reward", 1), "done": f("done", 1),
                 "next_state": f("next_state", D)}
        ref = _learn_reference(kind, agent, snap, batch, noise, num_learn)
        nets = _nets(agent)
        for net_name, grads in ref["grads"].items():
            for k, gref in grads.items():
                _normwise(nets[net_name].g[k], gref, tol, f"{tag} grad {net_name}.{k}")
        actor_stepped = "actor" in ref["grads"]
        for name, (net, opt) in _opts(agent).items():
            if name == "actor" and not actor_stepped:
                assert torch.equal(net.flat.detach().cpu(), snap["p"]["actor"]), f"{tag}: TD3 actor moved off its delay"
                continue
            _check_adam(name, net, opt, snap, tag)
        for k, v in ref["res"].items():
            if k in res and k in ref["scale"]:
                _within(res[k], v, tol * ref["scale"][k], f"{tag} result {k}")
        if kind == "sac":
            got_g = agent.log_alpha.grad[0].item()
            _within(got_g, ref["alpha_grad"], tol * ref["alpha_grad_scale"], f"{tag} d alpha_loss / d log_alpha")
            la0 = float(snap["log_alpha"].item())
            # one-step lag: the alpha this learn leaves behind is exp(log_alpha BEFORE its own step)
            _within(agent.alpha.item(), math.exp(la0), 4 * U * math.exp(la0), f"{tag} alpha")
            _within(res["alpha"], math.exp(la0), 4 * U * math.exp(la0), f"{tag} result alpha")
            if not agent.use_dynamic_alpha:
                assert torch.equal(agent.log_alpha.flat[:1].cpu(), snap["log_alpha"]), "static log_alpha moved"
        if kind == "td3":
            if actor_stepped and num_learn > 0:
                _check_soft(agent, snap, [("target_critic1", "critic1"), ("target_critic2", "critic2"),
                                          ("target_actor", "actor")], tag)
            else:
                for t in ("target_critic1", "target_critic2", "target_actor"):
                    assert torch.equal(nets[t].flat.detach().cpu(), snap["p"][t]), f"{tag}: {t} moved"
        else:
            snap2 = _snapshot(agent)
            agent.update_target_soft()
            pairs = [(f"target_critic{j + 1}", f"critic{j + 1}") for j in range(len(agent.critics))]
            if hasattr(agent, "target_actor"):
                pairs.append(("target_actor", "actor"))
            torch.cuda.synchronize()
            _check_soft(agent, snap2, pairs, tag)
        agent.learning_rate_decay(i + 1, agent._optimizers())
        lrs.append(agent.actor_optimizer.param_groups[0]["lr"])
    assert len(set(lrs)) == len(lrs), "lr must change between learns"
    return agent


LEARN_RUNS = {
    "sac_dynamic": ("sac", 11, 3, 8, {"use_dynamic_alpha": True}),
    "sac_static": ("sac", 11, 3, 4, {"use_dynamic_alpha": False, "static_log_alpha": -2.0}),
    "td3": ("td3", 11, 3, 8, {}),
    "ddpg": ("ddpg", 11, 3, 8, {}),
    "sac_d17_a6": ("sac", 17, 6, 1, {"use_dynamic_alpha": True}),
}


@pytest.mark.parametrize("name", list(LEARN_RUNS))
def test_learns_at_bench_shape_vs_float64(name):
    kind, D, A, n, extra = LEARN_RUNS[name]
    _run_learns(kind, D, A, n, seed=len(name), **extra)


GRAPH_RUNS = {"ddpg": ("ddpg", {}), "td3": ("td3", {"update_delay": 2}), "sac_dynamic": ("sac", {"use_dynamic_alpha": True}),
              "sac_static": ("sac", {"use_dynamic_alpha": False})}


@pytest.mark.parametrize("name", list(GRAPH_RUNS))
def test_cuda_graph_learn_is_bit_identical_at_bench_shape(name):
    """learn() as CUDA-graph replays (Philox draws from device counters, lr rewritten on the device between replays) vs
    the eager path at D=11, A=3, H=512, B=256: results and every network bit for bit over 8 learns (TD3: the first
    learn's actor step without target update, then alternating critic-only and actor + target learns)."""
    kind, extra = GRAPH_RUNS[name]
    a, b = _make_agent(kind, 11, 3, 256, use_cuda_graph=True, **extra), _make_agent(kind, 11, 3, 256, **extra)
    for x, y in zip(_nets(a).values(), _nets(b).values()):
        y.flat.copy_(x.flat)
    tr = _replay(11, 3, 31)
    a.memory.store([tr])
    b.memory.store([tr])
    rs = np.random.RandomState(32)
    for i in range(8):
        a._inject_idx = b._inject_idx = rs.randint(N_REPLAY, size=256)
        ra, rb = a.learn(), b.learn()
        assert ra == rb, (name, i, ra, rb)
        if kind != "td3":
            a.update_target_soft()
            b.update_target_soft()
        for ag in (a, b):
            ag.learning_rate_decay(i + 1, ag._optimizers())
    torch.cuda.synchronize()
    for (k, x), y in zip(_nets(a).items(), _nets(b).values()):
        assert torch.equal(x.flat, y.flat), (name, k)
    for (k, (_, oa)), (_, ob) in zip(_opts(a).items(), _opts(b).values()):
        assert all(torch.equal(s, t) for s, t in zip(oa.state_tensors(), ob.state_tensors())), (name, k)
    assert len(a._graphs) == (2 if kind == "td3" else 1) and not b._graphs
