"""Float64 oracle of the R2D2 agent — TEST INFRASTRUCTURE, never imported by the product.

R2D2 (Kapturowski et al., ICLR 2019) restated in torch from a parameter dict keyed like the product's state_dict.
Parity with the upstream JORLDY class is unpinned: its key names, the previous-action input, squared TD against a Huber
loss, and zero padding against the reset of the recurrent state at episode starts are assumptions that
tests/test_r2d2_reference.py checks when JORLDY_REFERENCE is set.

lstm()         torch.nn.LSTM's cell over [S, B, Z] inputs, gate order i, f, g, o, with (h, c) read as zero at the steps
               where reset[s, b] != 0
network()      head -> [feat, onehot(prev_action)] -> lstm -> dueling, batch-major [B, S] inputs, Q of the steps from
               grad_from on; the burn-in runs under no_grad and its final state is detached
value_h(), value_h_inv()   h(x) = sign(x)(sqrt(|x| + 1) - 1) + eps x and its inverse, eps = 1e-3
loss()         double-Q n-step targets under h, (1/(B T)) sum w_b td^2, and (eta max |td| + (1 - eta) mean |td|)^alpha
learn()        one learn() on a sampled batch: forward (online on s and s', target on s'), loss, autograd, clip_grad_norm,
               one torch.optim.Adam step
"""
import torch
import torch.nn.functional as F

from . import nets

EPS = 1e-3


def value_h(x):
    return torch.sign(x) * (torch.sqrt(x.abs() + 1.0) - 1.0) + EPS * x


def value_h_inv(x):
    s = (torch.sqrt(1.0 + 4.0 * EPS * (x.abs() + 1.0 + EPS)) - 1.0) / (2.0 * EPS)
    return torch.sign(x) * (s * s - 1.0)


def lstm(p, z, reset, h, c):
    """z [S, B, Z], reset [S, B] -> (hs [S, B, H], (h, c))."""
    w_ih, w_hh = p["lstm.weight_ih_l0"], p["lstm.weight_hh_l0"]
    b = p["lstm.bias_ih_l0"] + p["lstm.bias_hh_l0"]
    out = []
    for s in range(z.shape[0]):
        keep = (reset[s] == 0).to(z.dtype).unsqueeze(-1)
        h, c = h * keep, c * keep
        gi, gf, gg, go = (z[s] @ w_ih.T + b + h @ w_hh.T).chunk(4, dim=-1)
        c = torch.sigmoid(gf) * c + torch.sigmoid(gi) * torch.tanh(gg)
        h = torch.sigmoid(go) * torch.tanh(c)
        out.append(h)
    return torch.stack(out), (h, c)


def _dueling(p, h):
    xa = F.relu(F.linear(h, p["l1_a.weight"], p["l1_a.bias"]))
    xv = F.relu(F.linear(h, p["l1_v.weight"], p["l1_v.bias"]))
    a = F.linear(xa, p["l2_a.weight"], p["l2_a.bias"])
    return F.linear(xv, p["l2_v.weight"], p["l2_v.bias"]) + (a - a.mean(-1, keepdim=True))


def network(p, x, prev_action, reset, h0, c0, grad_from, A):
    """x [B, S, ...], prev_action int64 [B, S] (-1: none), reset [B, S], (h0, c0) [B, H] -> Q [B, S - grad_from, A]."""
    B, S = prev_action.shape
    feat = nets.head(p, x.reshape(B * S, *x.shape[2:])).reshape(B, S, -1)
    onehot = (prev_action.unsqueeze(-1) == torch.arange(A)).to(feat.dtype)
    z = torch.cat([feat, onehot], -1).transpose(0, 1)
    rs = reset.transpose(0, 1)
    h, c = h0, c0
    if grad_from > 0:
        with torch.no_grad():
            _, (h, c) = lstm(p, z[:grad_from], rs[:grad_from], h, c)
        h, c = h.detach(), c.detach()
    hs, _ = lstm(p, z[grad_from:], rs[grad_from:], h, c)
    return _dueling(p, hs).transpose(0, 1)


def loss(q, q_next, qt_next, action, reward, done, weights, gamma, n, eta, alpha):
    """q, q_next, qt_next [B, T, A]; action [B, T]; reward / done [B, T + n] -> (loss, td [B, T], prio [B])."""
    B, T, _ = q.shape
    a_star = q_next.argmax(-1, keepdim=True)
    y = value_h_inv(qt_next.gather(-1, a_star).squeeze(-1))
    for i in range(n - 1, -1, -1):
        y = reward[:, i:i + T] + (1.0 - done[:, i:i + T]) * gamma * y
    y = value_h(y).detach()
    td = y - q.gather(-1, action.unsqueeze(-1)).squeeze(-1)
    w = torch.ones(B, dtype=q.dtype) if weights is None else weights
    L = (w.unsqueeze(-1) * td * td).sum() / (B * T)
    a = td.detach().abs()
    prio = (eta * a.max(1).values + (1.0 - eta) * a.mean(1)) ** alpha
    return L, td, prio


def learn(params, target_params, batch, weights, hp, opt_state=None):
    """batch (batch-major): state [B, L, ...], action, prev_action, reset, reward, done [B, L], h0, c0 [B, H].
    hp: gamma, n_step, n_burn_in, seq_len, eta, alpha, lr, eps, clip, A."""
    Tb, T, n, A = hp["n_burn_in"], hp["seq_len"], hp["n_step"], hp["A"]
    S = Tb + T
    d = lambda t: t.to(torch.float64)
    x = d(batch["state"])
    prev, reset = batch["prev_action"].long(), d(batch["reset"])
    h0, c0 = d(batch["h0"]), d(batch["c0"])
    tp = {k: d(v) for k, v in target_params.items()}
    p = {k: d(v).clone().requires_grad_(True) for k, v in params.items()}
    w = None if weights is None else d(weights)
    with torch.no_grad():
        q_next = network(p, x[:, n:], prev[:, n:], reset[:, n:], h0, c0, Tb, A)
        qt_next = network(tp, x[:, n:], prev[:, n:], reset[:, n:], h0, c0, Tb, A)
    q = network(p, x[:, :S], prev[:, :S], reset[:, :S], h0, c0, Tb, A)
    L, td, prio = loss(q, q_next, qt_next, batch["action"][:, Tb:S].long(), d(batch["reward"][:, Tb:]),
                       d(batch["done"][:, Tb:]), w, hp["gamma"], n, hp["eta"], hp["alpha"])
    opt = torch.optim.Adam(list(p.values()), lr=hp["lr"], eps=hp["eps"])
    if opt_state is not None:
        opt.load_state_dict(opt_state)
    L.backward()
    grads = {k: v.grad.clone() for k, v in p.items()}
    torch.nn.utils.clip_grad_norm_(list(p.values()), hp["clip"])
    opt.step()
    result = {"loss": L.item(), "max_Q": q.gather(-1, batch["action"][:, Tb:S].long().unsqueeze(-1)).max().item()}
    return {"result": result, "prio": prio, "grads": grads, "params": {k: v.detach().clone() for k, v in p.items()},
            "q": q.detach(), "q_next": q_next, "qt_next": qt_next}
