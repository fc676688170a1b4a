"""Golden fixture for Rainbow-IQN: runs the UNMODIFIED reference `rainbow_iqn` agent for one learn() on one injected PER
minibatch (memory.sample patched to return the batch, IS weights and tree indices; memory.update_priority patched to record
the new priorities), with torch.rand (fractions) and torch.randn (noise) patched to record every draw in call order, and
records the initial online / target parameters, the minibatch, the weights, the draws, the result dict, the priorities and
the post-learn parameters.  Parity of this project's Rainbow-IQN with the reference class is not pinned by a committed
fixture: no upstream checkout was available when it was written, so the parameter names, the draw order and the priority
L_b^alpha have not been confirmed.  tests/test_rainbow_iqn_reference.py mints this file into a temporary directory and
compares it with oracle/rainbow_iqn.py when a checkout is available.
`python tests/golden/make_golden_rainbow_iqn.py [out_dir]`."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from refimport import import_reference  # noqa: E402

CASE = dict(D=4, A=3, H=32, B=8, N=8, n=3, gamma=0.99, lr=1e-3, seed=0, alpha=0.6, beta=0.4, buffer_size=64)


def batch(case):
    rs = np.random.RandomState(case["seed"] + 1)
    B, D, A, n = case["B"], case["D"], case["A"], case["n"]
    return {"state": rs.standard_normal((B, D)).astype(np.float32), "next_state": rs.standard_normal((B, D)).astype(np.float32),
            "action": rs.randint(A, size=(B, 1)).astype(np.int64), "reward": rs.standard_normal((B, n, 1)).astype(np.float32),
            "done": (rs.uniform(size=(B, n, 1)) < 0.3).astype(np.float32)}


def weights_and_indices(case):
    rs = np.random.RandomState(case["seed"] + 2)
    w = rs.uniform(0.1, 1.0, size=case["B"])
    w[0] = 1.0
    return w, case["buffer_size"] - 1 + rs.randint(case["buffer_size"], size=case["B"])


def gen(agent_mod, case=CASE, out_dir=HERE):
    out = {}
    tr = batch(case)
    w, idx = weights_and_indices(case)
    for k, v in tr.items():
        out[f"batch.{k}"] = v
    out["weights"], out["indices"] = w, idx
    torch.manual_seed(case["seed"])
    agent = agent_mod.Agent("rainbow_iqn", state_size=case["D"], action_size=case["A"], hidden_size=case["H"],
                            optim_config={"name": "adam", "lr": case["lr"]}, gamma=case["gamma"],
                            buffer_size=case["buffer_size"], batch_size=case["B"], n_step=case["n"], alpha=case["alpha"],
                            beta=case["beta"], num_sample=case["N"], device="cpu", run_step=1000, lr_decay=False)
    for net in ("network", "target_network"):
        for k, v in getattr(agent, net).state_dict().items():
            out[f"init.{net}.{k}"] = v.detach().numpy().copy()
    agent.memory.sample = lambda beta, bs: ({k: v.copy() for k, v in tr.items()}, w.copy(), idx.copy(), 1.0, 1.0)
    prios = []
    agent.memory.update_priority = lambda p, i: prios.append((float(np.asarray(p).reshape(-1)[0]), int(i)))
    draws, real = {"rand": [], "randn": []}, {"rand": torch.rand, "randn": torch.randn}

    def recorder(name):
        def fn(*shape, **kw):
            t = real[name](*shape, **kw)
            draws[name].append(t.detach().numpy().copy())
            return t
        return fn

    torch.rand, torch.randn = recorder("rand"), recorder("randn")
    try:
        res = agent.learn()
    finally:
        torch.rand, torch.randn = real["rand"], real["randn"]
    for name, ts in draws.items():
        for i, t in enumerate(ts):
            out[f"{name}{i}"] = t
    for k, v in res.items():
        out[f"result.{k}"] = np.float64(v)
    out["prio.p"] = np.array([p for p, _ in prios])
    out["prio.index"] = np.array([i for _, i in prios])
    for k, v in agent.network.state_dict().items():
        out[f"param.{k}"] = v.detach().numpy().copy()
    path = os.path.join(out_dir, "rainbow_iqn_small.npz")
    np.savez_compressed(path, **out)
    return path


def main():
    agent_mod, _, _ = import_reference()
    print(gen(agent_mod, out_dir=sys.argv[1] if len(sys.argv) > 1 else HERE))


if __name__ == "__main__":
    main()
