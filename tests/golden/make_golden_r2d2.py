"""Golden fixture for R2D2: runs the UNMODIFIED reference `r2d2` agent for one learn() on one injected PER minibatch of
sequences (memory.sample patched to return the batch, IS weights and tree indices; memory.update_priority patched to
record the new priorities) and records the initial online / target parameters, the batch, the weights, the result dict,
the priorities and the post-learn parameters.  Parity of this project's R2D2 with the reference class is not pinned by a
committed fixture: no upstream checkout was available when it was written, so these are assumptions the reference test
exists to check:
  - the upstream key names: the batch keys state, action, prev_action, reward, done, hidden_h, hidden_c and the network's
    parameter names;
  - the previous action as an LSTM input (one-hot, none at an episode's first step);
  - the squared TD loss (against a Huber loss);
  - the reset of the recurrent state at episode starts inside a sequence (against the upstream zero padding).
tests/test_r2d2_reference.py mints this file into a temporary directory and compares it with oracle/r2d2.py when a
checkout is available.  `python tests/golden/make_golden_r2d2.py [out_dir]`."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from refimport import import_reference  # noqa: E402

CASE = dict(D=4, A=3, H=32, B=4, Tb=2, T=4, n=2, gamma=0.997, lr=1e-3, seed=0, alpha=0.9, beta=0.6, eta=0.9,
            buffer_size=64)


def batch(case):
    rs = np.random.RandomState(case["seed"] + 1)
    B, D, A, H = case["B"], case["D"], case["A"], case["H"]
    L = case["Tb"] + case["T"] + case["n"]
    done = np.zeros((B, L), np.float32)
    action = rs.randint(A, size=(B, L)).astype(np.int64)
    prev = np.concatenate([np.full((B, 1), -1), action[:, :-1]], 1).astype(np.int64)
    return {"state": rs.standard_normal((B, L, D)).astype(np.float32), "action": action, "prev_action": prev,
            "reset": np.concatenate([np.ones((B, 1)), np.zeros((B, L - 1))], 1).astype(np.float32),
            "reward": rs.standard_normal((B, L)).astype(np.float32), "done": done,
            "h0": np.zeros((B, H), np.float32), "c0": np.zeros((B, H), np.float32)}


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
    upstream = {"state": tr["state"], "action": tr["action"][..., None], "prev_action": tr["prev_action"][..., None],
                "reward": tr["reward"][..., None], "done": tr["done"][..., None], "hidden_h": tr["h0"][:, None],
                "hidden_c": tr["c0"][:, None]}
    torch.manual_seed(case["seed"])
    agent = agent_mod.Agent("r2d2", state_size=case["D"], action_size=case["A"], hidden_size=case["H"],
                            optim_config={"name": "adam", "lr": case["lr"]}, gamma=case["gamma"],
                            buffer_size=case["buffer_size"], batch_size=case["B"], n_step=case["n"], alpha=case["alpha"],
                            beta=case["beta"], eta=case["eta"], seq_len=case["T"], n_burn_in=case["Tb"], device="cpu",
                            run_step=1000, lr_decay=False)
    for net in ("network", "target_network"):
        for k, v in getattr(agent, net).state_dict().items():
            out[f"init.{net}.{k}"] = v.detach().numpy().copy()
    agent.memory.sample = lambda beta, bs: ({k: v.copy() for k, v in upstream.items()}, w.copy(), idx.copy(), 1.0, 1.0)
    prios = []
    agent.memory.update_priority = lambda p, i: prios.append((float(np.asarray(p).reshape(-1)[0]), int(i)))
    res = agent.learn()
    for k, v in res.items():
        out[f"result.{k}"] = np.float64(v)
    out["prio.p"] = np.array([p for p, _ in prios])
    out["prio.index"] = np.array([i for _, i in prios])
    for k, v in agent.network.state_dict().items():
        out[f"param.{k}"] = v.detach().numpy().copy()
    path = os.path.join(out_dir, "r2d2_small.npz")
    np.savez_compressed(path, **out)
    return path


def main():
    agent_mod, _, _ = import_reference()
    print(gen(agent_mod, out_dir=sys.argv[1] if len(sys.argv) > 1 else HERE))


if __name__ == "__main__":
    main()
