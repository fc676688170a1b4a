"""Float64 oracle of MuZero's root masking for board games — TEST INFRASTRUCTURE, never imported by the product.

The MuZero paper (arXiv:1911.08265, Appendix B) masks illegal actions at the root of the search, where the env can be
queried, and nowhere inside the tree.  Restated on top of oracle/muzero.py, which it leaves unchanged:

root_prior()       the softmax over the legal logits (0 elsewhere), mixed with noise normalised over the legal actions
LegalTree          oracle/muzero.py's Tree whose select() never takes an illegal action at depth 0
search_legal()     oracle/muzero.py's search() with the masked root
A mask with no legal action counts every action legal, as the kernels do.
"""
import math

import numpy as np
import torch

from . import muzero as om


def _mask(legal, A):
    legal = np.asarray(legal, dtype=bool).reshape(A)
    return legal if legal.any() else np.ones(A, dtype=bool)


def root_prior(pi_logits, legal, noise=None, frac=0.25):
    z = np.asarray(pi_logits, dtype=np.float64)
    ok = _mask(legal, z.shape[0])
    prior = np.zeros_like(z)
    prior[ok] = om._softmax(z[ok])
    if noise is not None:
        g = np.where(ok, np.asarray(noise, dtype=np.float64), 0.0)
        prior = np.where(ok, (1 - frac) * prior + frac * g / g.sum(), 0.0)
    return prior


class LegalTree(om.Tree):
    def __init__(self, A, S, legal):
        super().__init__(A, S)
        self.legal = _mask(legal, A)

    def select(self, gamma):
        node, pn = 0, int(self.n[0].sum())
        self.path = []
        while True:
            scores = []
            for a in range(self.A):
                if node == 0 and len(self.path) == 0 and not self.legal[a]:
                    scores.append(-math.inf)
                    continue
                n = self.n[node, a]
                q = 0.0
                if n > 0:
                    q = self.r[node, a] + gamma * self.w[node, a] / n
                    if self.qmax > self.qmin:
                        q = (q - self.qmin) / (self.qmax - self.qmin)
                pb = (math.log((pn + om.PB_C_BASE + 1) / om.PB_C_BASE) + om.PB_C_INIT) * math.sqrt(pn) / (n + 1)
                scores.append(q + pb * self.p[node, a])
            a = int(np.argmax(scores))          # first index on ties; an illegal root action scores -inf
            self.path.append((node, a))
            c = self.child[node, a]
            if c < 0 or len(self.path) > self.S:
                return node, a, scores
            pn = int(self.n[node, a])
            node = c


def search_legal(root_pi_logits, root_latent, model, A, S, gamma, V, R, legal, noise=None, frac=0.25, training=False,
                 temperature=1.0, u=None, margins=None):
    """oracle/muzero.py search() with the root masked by legal [A].  margins: the gap between the top two finite pUCT
    scores of every selection after the first.  Returns (tree, action, pi, root_value)."""
    t = LegalTree(A, S, legal)
    t.p[0] = root_prior(root_pi_logits, t.legal, noise, frac)
    t.latent[0] = root_latent
    for sim in range(S):
        node, a, scores = t.select(gamma)
        finite = np.sort(np.asarray([x for x in scores if np.isfinite(x)]))[::-1]
        if margins is not None and sim > 0 and finite.size > 1:
            margins.append(finite[0] - finite[1])
        latent, pi_l, v_l, r_l = model(sim, t.latent[node], a)
        r = float(om.support_to_scalar(torch.as_tensor(r_l), R))
        v = float(om.support_to_scalar(torch.as_tensor(v_l), V))
        t.expand_backup(latent, pi_l, r, v, gamma)
    a, pi, rv = t.act(gamma, training, temperature, u)
    return t, a, pi, rv
