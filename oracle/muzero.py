"""Float64 oracle of the MuZero agent — TEST INFRASTRUCTURE, never imported by the product.

MuZero (Schrittwieser et al., arXiv:1911.08265, Appendix B/C/G and its pseudocode) restated in torch float64 and plain
python from a parameter dict keyed like the product's state_dict.  Parity with an upstream JORLDY class is unpinned;
tests/test_muzero_reference.py compares when JORLDY_REFERENCE is set.

value_h(), value_h_inv()          h(x) = sign(x)(sqrt(|x| + 1) - 1) + 1e-3 x and its closed-form inverse (oracle/r2d2.py)
scalar_to_support(), support_to_scalar()   two-hot of clamp(h(x), -V, V); h^-1 of the softmax expectation
scale()                           per-row min-max scaling to [0, 1], range at least 1e-5
represent(), dynamics(), predict()   the three networks
targets()                         n-step value targets z, reward targets u and the absorbing mask of B windows
loss()                            the unrolled cross-entropy loss, its stats and the priorities
unroll_loss()                     h, K dynamics steps (gradient into each latent input scaled by 0.5), f, loss()
learn()                           one learn: unroll_loss, autograd, clip_grad_norm, one torch.optim.Adam step
Tree, search()                    one env's MCTS with a model callback: scripted (arrays of logits per simulation) or the
                                  float64 networks (network_model())
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .r2d2 import value_h, value_h_inv  # noqa: F401

PB_C_BASE, PB_C_INIT = 19652.0, 1.25
SCALE_MIN_RANGE = 1e-5


def scalar_to_support(x, V):
    """x [...] -> [..., 2V + 1]."""
    y = value_h(torch.as_tensor(x, dtype=torch.float64)).clamp(-V, V)
    lo = torch.floor(y)
    up = y - lo
    idx = (lo + V).long()
    out = torch.zeros(*y.shape, 2 * V + 1, dtype=torch.float64)
    out.scatter_(-1, idx.unsqueeze(-1), (1 - up).unsqueeze(-1))
    hi = (idx + 1).clamp(max=2 * V)
    out.scatter_add_(-1, hi.unsqueeze(-1), torch.where(idx < 2 * V, up, torch.zeros_like(up)).unsqueeze(-1))
    return out


def support_to_scalar(logits, V):
    p = torch.softmax(torch.as_tensor(logits, dtype=torch.float64), -1)
    atoms = torch.arange(-V, V + 1, dtype=torch.float64)
    return value_h_inv((p * atoms).sum(-1))


def scale(x):
    mn = x.min(-1, keepdim=True).values
    mx = x.max(-1, keepdim=True).values
    return (x - mn) / torch.clamp(mx - mn, min=SCALE_MIN_RANGE)


def represent(p, x):
    h = F.relu(F.linear(x, p["h.l1.weight"], p["h.l1.bias"]))
    return scale(F.linear(h, p["h.l2.weight"], p["h.l2.bias"]))


def dynamics(p, s, a, A):
    z = torch.cat([s, F.one_hot(a.long(), A).to(s.dtype)], -1)
    h = F.relu(F.linear(z, p["g.l1.weight"], p["g.l1.bias"]))
    return scale(F.linear(h, p["g.s.weight"], p["g.s.bias"])), F.linear(h, p["g.r.weight"], p["g.r.bias"])


def predict(p, s):
    h = F.relu(F.linear(s, p["f.l1.weight"], p["f.l1.bias"]))
    return F.linear(h, p["f.pi.weight"], p["f.pi.bias"]), F.linear(h, p["f.v.weight"], p["f.v.bias"])


def targets(reward, done, root_value, K, n, gamma):
    """Windows [B, L = K + n + 1] -> z [B, K + 1], u [B, K + 1] (u[:, 0] unused), absorbing [B, K + 1] bool."""
    reward, done, root_value = (np.asarray(t, dtype=np.float64) for t in (reward, done, root_value))
    B = reward.shape[0]
    z, u = np.zeros((B, K + 1)), np.zeros((B, K + 1))
    absorbing = np.zeros((B, K + 1), dtype=bool)
    for b in range(B):
        for k in range(K + 1):
            absorbing[b, k] = bool(np.any(done[b, :k] != 0))
            if not absorbing[b, k]:
                g = root_value[b, k + n]
                for i in reversed(range(n)):
                    g = reward[b, k + i] + (1.0 - done[b, k + i]) * gamma * g
                z[b, k] = g
            if k > 0 and not (k >= 2 and absorbing[b, k - 1]):
                u[b, k] = reward[b, k - 1]
    return z, u, absorbing


def loss(pi, v, r, batch, weights, hp):
    """pi [K + 1, B, A], v [K + 1, B, 2V + 1], r [K, B, 2R + 1] logits (tensors, may require grad); batch: reward, done,
    root_value [B, L], policy [B, L, A].  Returns (loss, stats dict, priorities [B])."""
    K, n, V, R, gamma = hp["K"], hp["n"], hp["V"], hp["R"], hp["gamma"]
    B = pi.shape[1]
    z, u, absorbing = targets(batch["reward"], batch["done"], batch["root_value"], K, n, gamma)
    w = torch.ones(B, dtype=torch.float64) if weights is None else torch.as_tensor(weights, dtype=torch.float64)
    policy = torch.as_tensor(np.asarray(batch["policy"]), dtype=torch.float64)
    lv = lr = lp = 0.0
    for k in range(K + 1):
        c = (1.0 if k == 0 else 1.0 / K) * w
        ce_v = -(scalar_to_support(torch.as_tensor(z[:, k]), V) * F.log_softmax(v[k], -1)).sum(-1)
        lv = lv + (c * hp["value_loss_coef"] * ce_v).sum() / B
        keep = torch.as_tensor(~absorbing[:, k], dtype=torch.float64)
        ce_p = -(policy[:, k] * keep.unsqueeze(-1) * F.log_softmax(pi[k], -1)).sum(-1)
        lp = lp + (c * ce_p).sum() / B
        if k > 0:
            ce_r = -(scalar_to_support(torch.as_tensor(u[:, k]), R) * F.log_softmax(r[k - 1], -1)).sum(-1)
            lr = lr + (c * ce_r).sum() / B
    v0 = support_to_scalar(v[0].detach(), V)
    prio = (v0 - torch.as_tensor(z[:, 0])).abs() ** hp["alpha"]
    total = lv + lr + lp
    f = lambda t: float(t.detach()) if torch.is_tensor(t) else float(t)
    stats = {"loss": f(total), "value_loss": f(lv), "reward_loss": f(lr), "policy_loss": f(lp)}
    return total, stats, prio


def unroll_loss(p, batch, weights, hp):
    A, K = hp["A"], hp["K"]
    x = torch.as_tensor(np.asarray(batch["state"]), dtype=torch.float64)
    action = torch.as_tensor(np.asarray(batch["action"])).long()
    s = represent(p, x)
    pis, vs, rs = [], [], []
    for k in range(K + 1):
        pi_k, v_k = predict(p, s)
        pis.append(pi_k)
        vs.append(v_k)
        if k < K:
            s_in = 0.5 * s + 0.5 * s.detach()          # the pseudocode's scale_gradient(hidden_state, 0.5)
            s, r_k = dynamics(p, s_in, action[:, k], A)
            rs.append(r_k)
    return loss(torch.stack(pis), torch.stack(vs), torch.stack(rs), batch, weights, hp)


def learn(params, batch, weights, hp, lr, clip, adam_state=None):
    """One learn from float64 copies of `params`; returns (new params, stats, priorities, grads)."""
    p = {k: torch.as_tensor(v, dtype=torch.float64).clone().requires_grad_(True) for k, v in params.items()}
    total, stats, prio = unroll_loss(p, batch, weights, hp)
    total.backward()
    grads = {k: v.grad.clone() for k, v in p.items()}
    torch.nn.utils.clip_grad_norm_(list(p.values()), clip)
    opt = torch.optim.Adam(list(p.values()), lr=lr)
    opt.step()
    return {k: v.detach() for k, v in p.items()}, stats, prio, grads


# ---- search -------------------------------------------------------------------------------------------------------------
def _softmax(z):
    z = np.asarray(z, dtype=np.float64)
    e = np.exp(z - z.max())
    return e / e.sum()


class Tree:
    """One env's tree with the product's layout: per node A edges (n, w, p, r, child)."""

    def __init__(self, A, S):
        self.A, self.S = A, S
        self.n = np.zeros((S + 1, A), dtype=np.int64)
        self.w = np.zeros((S + 1, A))
        self.p = np.zeros((S + 1, A))
        self.r = np.zeros((S + 1, A))
        self.child = -np.ones((S + 1, A), dtype=np.int64)
        self.latent = [None] * (S + 1)
        self.count, self.qmin, self.qmax = 1, math.inf, -math.inf
        self.path = []

    def select(self, gamma):
        node, pn = 0, int(self.n[0].sum())
        self.path = []
        while True:
            scores = []
            for a in range(self.A):
                n = self.n[node, a]
                q = 0.0
                if n > 0:
                    q = self.r[node, a] + gamma * self.w[node, a] / n
                    if self.qmax > self.qmin:
                        q = (q - self.qmin) / (self.qmax - self.qmin)
                pb = (math.log((pn + PB_C_BASE + 1) / PB_C_BASE) + PB_C_INIT) * math.sqrt(pn) / (n + 1)
                scores.append(q + pb * self.p[node, a])
            a = int(np.argmax(scores))          # first index on ties
            self.path.append((node, a))
            c = self.child[node, a]
            if c < 0 or len(self.path) > self.S:
                return node, a, scores
            pn = int(self.n[node, a])
            node = c

    def expand_backup(self, latent, pi_logits, reward, value, gamma):
        nn = self.count
        node, a = self.path[-1]
        self.latent[nn] = latent
        self.p[nn] = _softmax(pi_logits)
        self.child[node, a] = nn
        self.r[node, a] = reward
        self.count += 1
        g = value
        for node, a in reversed(self.path):
            self.w[node, a] += g
            self.n[node, a] += 1
            q = self.r[node, a] + gamma * self.w[node, a] / self.n[node, a]
            self.qmin, self.qmax = min(self.qmin, q), max(self.qmax, q)
            g = self.r[node, a] + gamma * g

    def act(self, gamma, training, temperature=1.0, u=None):
        n = self.n[0].astype(np.float64)
        tot = n.sum()
        pi = n / tot if tot > 0 else np.zeros_like(n)
        root_value = float((n * self.r[0] + gamma * self.w[0]).sum() / tot) if tot > 0 else 0.0
        if training:
            wl = n ** (1.0 / temperature)
            c = np.cumsum(wl)
            hit = np.nonzero((u * c[-1] < c) & (wl > 0))[0]
            a = int(hit[0]) if hit.size else 0
        else:
            a = int(np.argmax(n))
        return a, pi, root_value


def search(root_pi_logits, root_latent, model, A, S, gamma, V, R, noise=None, frac=0.25, training=False,
           temperature=1.0, u=None, margins=None):
    """One env's search.  model(sim, latent, action) -> (latent, pi_logits, v_logits, r_logits) of the new leaf.
    noise: gamma draws [A] (Dirichlet = noise / sum) mixed at `frac`.  margins (a list): receives the gap between the top
    two pUCT scores of every selection after the first (whose scores are all exactly 0).  Returns (tree, action, pi, root_value)."""
    t = Tree(A, S)
    prior = _softmax(root_pi_logits)
    if noise is not None:
        g = np.asarray(noise, dtype=np.float64)
        prior = (1 - frac) * prior + frac * g / g.sum()
    t.p[0] = prior
    t.latent[0] = root_latent
    for sim in range(S):
        node, a, scores = t.select(gamma)
        if margins is not None and sim > 0 and len(scores) > 1:      # sim 0: every score is exactly 0 (parent N = 0)
            top = np.sort(np.asarray(scores))[::-1]
            margins.append(top[0] - top[1])
        latent, pi_l, v_l, r_l = model(sim, t.latent[node], a)
        r = float(support_to_scalar(torch.as_tensor(r_l), R))
        v = float(support_to_scalar(torch.as_tensor(v_l), V))
        t.expand_backup(latent, pi_l, r, v, gamma)
    a, pi, rv = t.act(gamma, training, temperature, u)
    return t, a, pi, rv


def network_model(p, A):
    """A search model from float64 network parameters."""
    def model(sim, latent, a):
        s = torch.as_tensor(latent, dtype=torch.float64).view(1, -1)
        s2, r_l = dynamics(p, s, torch.tensor([a]), A)
        pi_l, v_l = predict(p, s2)
        return s2[0], pi_l[0], v_l[0], r_l[0]
    return model
