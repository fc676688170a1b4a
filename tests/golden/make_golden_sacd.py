"""Golden fixture for the discrete-action SAC: runs the UNMODIFIED reference SAC with `actor="discrete_policy"`,
`critic="discrete_q_network"` for three learn() calls on one injected minibatch (memory.sample patched) and records the
initial parameters of every network, the minibatch, each learn's result dict, the post-learn parameters and
log_alpha / alpha.  Parity of this project's discrete SAC with the reference class is not pinned by a committed fixture;
tests/test_sac_discrete_reference.py mints this file into a temporary directory and compares it with
oracle/sac_discrete.py when an upstream checkout is available.  Run in the build container:
`python tests/golden/make_golden_sacd.py [out_dir]`."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from refimport import import_reference  # noqa: E402

CASE = dict(D=4, A=3, H=32, B=8, gamma=0.99, tau=5e-3, actor_lr=3e-4, critic_lr=1e-3, alpha_lr=2e-3, dynamic_alpha=True,
            learns=3, seed=0)
NETS = ("actor", "critic1", "critic2", "target_critic1", "target_critic2")


def batch(case):
    rs = np.random.RandomState(case["seed"] + 1)
    B, D, A = case["B"], case["D"], case["A"]
    return {"state": rs.standard_normal((B, D)).astype(np.float32), "next_state": rs.standard_normal((B, D)).astype(np.float32),
            "action": rs.randint(A, size=(B, 1)).astype(np.int64), "reward": rs.standard_normal((B, 1)).astype(np.float32),
            "done": (rs.uniform(size=(B, 1)) < 0.3).astype(np.float32)}


def gen(agent_mod, case=CASE, out_dir=HERE):
    torch.manual_seed(case["seed"])
    optim = {"actor": "adam", "critic": "adam", "alpha": "adam", "actor_lr": case["actor_lr"], "critic_lr": case["critic_lr"],
             "alpha_lr": case["alpha_lr"]}
    agent = agent_mod.Agent("sac", state_size=case["D"], action_size=case["A"], hidden_size=case["H"], actor="discrete_policy",
                            critic="discrete_q_network", optim_config=optim, gamma=case["gamma"], tau=case["tau"],
                            buffer_size=64, batch_size=case["B"], use_dynamic_alpha=case["dynamic_alpha"], device="cpu",
                            run_step=1000, lr_decay=False)
    out = {}
    for n in NETS:
        for k, v in getattr(agent, n).state_dict().items():
            out[f"init.{n}.{k}"] = v.detach().numpy().copy()
    out["init.log_alpha"] = np.float64(agent.log_alpha.detach().item())
    tr = batch(case)
    for k, v in tr.items():
        out[f"batch.{k}"] = v
    agent.memory.sample = lambda bs: {k: v.copy() for k, v in tr.items()}
    for i in range(case["learns"]):
        for k, v in agent.learn().items():
            out[f"result{i}.{k}"] = np.float64(v)
        out[f"log_alpha{i}"] = np.float64(agent.log_alpha.detach().item())
    for n in NETS:
        for k, v in getattr(agent, n).state_dict().items():
            out[f"param.{n}.{k}"] = v.detach().numpy().copy()
    path = os.path.join(out_dir, "sacd_small.npz")
    np.savez_compressed(path, **out)
    return path


def main():
    agent_mod, _, _ = import_reference()
    print(gen(agent_mod, out_dir=sys.argv[1] if len(sys.argv) > 1 else HERE))


if __name__ == "__main__":
    main()
