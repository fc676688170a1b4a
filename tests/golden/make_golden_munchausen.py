"""Golden fixture for the Munchausen agents: runs the UNMODIFIED reference M-DQN and M-IQN for one learn() each on one
injected minibatch (memory.sample patched; for M-IQN, torch.rand patched to record every fraction draw in call order)
with the constructor keys alpha, tau and l_0, and records the initial online / target parameters, the minibatch, the
fractions, the result dict and the post-learn parameters.  Parity of this project's Munchausen agents with the reference
classes is not pinned by a committed fixture: no upstream checkout was available when they were written, so neither the
key spelling nor M-IQN's draw order has been confirmed.  tests/test_munchausen_reference.py mints this file into a
temporary directory and compares it with oracle/munchausen.py when a checkout is available.
`python tests/golden/make_golden_munchausen.py [out_dir]`."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from refimport import import_reference  # noqa: E402

CASE = dict(D=4, A=3, H=32, B=8, N=8, gamma=0.99, lr=1e-3, seed=0, alpha=0.9, tau=0.03, l_0=-1)


def batch(case):
    rs = np.random.RandomState(case["seed"] + 1)
    B, D, A = case["B"], case["D"], case["A"]
    return {"state": rs.standard_normal((B, D)).astype(np.float32), "next_state": rs.standard_normal((B, D)).astype(np.float32),
            "action": rs.randint(A, size=(B, 1)).astype(np.int64), "reward": rs.standard_normal((B, 1)).astype(np.float32),
            "done": (rs.uniform(size=(B, 1)) < 0.3).astype(np.float32)}


def gen(agent_mod, case=CASE, out_dir=HERE):
    out = {}
    tr = batch(case)
    for k, v in tr.items():
        out[f"batch.{k}"] = v
    m = dict(alpha=case["alpha"], tau=case["tau"], l_0=case["l_0"])
    for name, extra in (("m_dqn", m), ("m_iqn", dict(m, num_sample=case["N"]))):
        torch.manual_seed(case["seed"])
        agent = agent_mod.Agent(name, state_size=case["D"], action_size=case["A"], hidden_size=case["H"],
                                optim_config={"name": "adam", "lr": case["lr"]}, gamma=case["gamma"], buffer_size=64,
                                batch_size=case["B"], device="cpu", run_step=1000, lr_decay=False, **extra)
        for net in ("network", "target_network"):
            for k, v in getattr(agent, net).state_dict().items():
                out[f"{name}.init.{net}.{k}"] = v.detach().numpy().copy()
        agent.memory.sample = lambda bs: {k: v.copy() for k, v in tr.items()}
        taus, real_rand = [], torch.rand

        def rand(*shape, **kw):                        # records every fraction draw of learn(), in call order
            t = real_rand(*shape, **kw)
            taus.append(t.detach().numpy().copy())
            return t

        torch.rand = rand
        try:
            res = agent.learn()
        finally:
            torch.rand = real_rand
        for i, t in enumerate(taus):
            out[f"{name}.tau{i}"] = t
        for k, v in res.items():
            out[f"{name}.result.{k}"] = np.float64(v)
        for k, v in agent.network.state_dict().items():
            out[f"{name}.param.{k}"] = v.detach().numpy().copy()
    path = os.path.join(out_dir, "munchausen_small.npz")
    np.savez_compressed(path, **out)
    return path


def main():
    agent_mod, _, _ = import_reference()
    print(gen(agent_mod, out_dir=sys.argv[1] if len(sys.argv) > 1 else HERE))


if __name__ == "__main__":
    main()
