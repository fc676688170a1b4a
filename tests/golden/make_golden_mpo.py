"""Golden fixture for MPO: runs the UNMODIFIED reference `mpo` agent for one learn() on one fixed batch of n-step windows
(its replay sample patched to return the batch), discrete actions, and records the initial actor / critic parameters,
the batch, the result dict, the multipliers and the post-learn parameters.  The discrete E-step is exact over the
actions, so one learn draws no noise.  Parity of this project's MPO with the reference class is not pinned by a committed
fixture: no upstream checkout was available when it was written, so these are assumptions the reference test exists to
check:
  - the constructor key names (critic_loss_type, num_sample, n_step, target_update_period, min_eta, min_alpha_mu,
    min_alpha_sigma, eps_eta, eps_alpha_mu, eps_alpha_sigma, eta, alpha_mu, alpha_sigma) and the result keys
    (actor_loss, critic_loss, eta_loss, alpha_loss, eta, alpha_mu, alpha_sigma, mean_Q);
  - a replayed item as a window of n steps: state [n+1, D], action / reward / done / log_mu [n];
  - the critic loss as a mean of squares (no factor 1/2), one optimiser over actor.parameters() + the multipliers with
    clip_grad_norm_ on the actor only, and the target copy every target_update_period learns.
tests/test_mpo_reference.py mints this file into a temporary directory and compares it with oracle/mpo.py when a
checkout is available.  `python tests/golden/make_golden_mpo.py [out_dir]`."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from refimport import import_reference  # noqa: E402

HP = dict(min_eta=1e-8, min_alpha_mu=1e-8, min_alpha_sigma=1e-8, eps_eta=0.01, eps_alpha_mu=0.01, eps_alpha_sigma=5e-5,
          eta=1.0, alpha_mu=1.0, alpha_sigma=1.0, critic_loss_type="retrace", num_sample=30, target_update_period=100,
          clip_grad_norm=1.0)
CASES = {"mpo_discrete": dict(D=4, A=2, H=32, n=4, B=8, lr=1e-3, gamma=0.99, seed=51)}


def batch(case):
    rs = np.random.RandomState(case["seed"])
    B, n, D, A = case["B"], case["n"], case["D"], case["A"]
    return dict(state=rs.standard_normal((B, n + 1, D)).astype(np.float32),
                action=rs.randint(0, A, (B, n)).astype(np.int64),
                reward=rs.standard_normal((B, n)).astype(np.float32),
                done=(rs.uniform(size=(B, n)) < 0.2).astype(np.float32),
                log_mu=np.log(rs.uniform(0.2, 0.8, (B, n))).astype(np.float32))


def gen(agent_mod, name, case, out_dir=HERE):
    torch.manual_seed(case["seed"])
    agent = agent_mod.Agent(
        "mpo", state_size=case["D"], action_size=case["A"], hidden_size=case["H"], actor="discrete_policy",
        critic="discrete_q_network", optim_config={"name": "adam", "lr": case["lr"]}, gamma=case["gamma"],
        n_step=case["n"], batch_size=case["B"], run_step=1000, lr_decay=False, device="cpu", **HP)
    b = batch(case)
    out = {f"batch.{k}": v for k, v in b.items()}
    out.update({f"init.actor.{k}": v.numpy().copy() for k, v in agent.actor.state_dict().items()})
    out.update({f"init.critic.{k}": v.numpy().copy() for k, v in agent.critic.state_dict().items()})
    agent.memory.sample = lambda batch_size: {k: v.copy() for k, v in b.items()}
    result = agent.learn()
    out.update({f"result.{k}": np.float64(v) for k, v in result.items()})
    out.update({f"param.actor.{k}": v.detach().numpy() for k, v in agent.actor.state_dict().items()})
    out.update({f"param.critic.{k}": v.detach().numpy() for k, v in agent.critic.state_dict().items()})
    path = os.path.join(out_dir, name + ".npz")
    np.savez_compressed(path, **out)
    return path


if __name__ == "__main__":
    mod = import_reference()[0]
    for n, c in CASES.items():
        print(gen(mod, n, c, sys.argv[1] if len(sys.argv) > 1 else HERE))
