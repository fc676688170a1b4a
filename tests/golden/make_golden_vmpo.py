"""Golden fixture for V-MPO: runs the UNMODIFIED reference `vmpo` agent for one learn() on one stored rollout with the
minibatch permutations injected (np.random.shuffle patched, as make_golden.py does for PPO), discrete and continuous,
and records the initial parameters, the result dict, the multipliers and the post-learn parameters.  Parity of this
project's V-MPO with the reference class is not pinned by a committed fixture: no upstream checkout was available when
it was written, so these are assumptions the reference test exists to check:
  - the constructor key names (min_eta, min_alpha_mu, min_alpha_sigma, eps_eta, eps_alpha_mu, eps_alpha_sigma, eta,
    alpha_mu, alpha_sigma) and the result keys (actor_loss, critic_loss, eta_loss, alpha_loss, eta, alpha_mu,
    alpha_sigma, mean_ret);
  - the critic loss as F.mse_loss (no factor 1/2) and the discrete log pi as the log-softmax of the chosen action;
  - one optimiser over network.parameters() + [eta, alpha_mu, alpha_sigma], clip_grad_norm_ on the network only.
tests/test_vmpo_reference.py mints this file into a temporary directory and compares it with oracle/vmpo.py when a
checkout is available.  `python tests/golden/make_golden_vmpo.py [out_dir]`."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gen_inputs as G  # noqa: E402
from refimport import import_reference  # noqa: E402

HP = dict(min_eta=1e-8, min_alpha_mu=1e-8, min_alpha_sigma=1e-8, eps_eta=0.01, eps_alpha_mu=0.01, eps_alpha_sigma=5e-5,
          eta=1.0, alpha_mu=5.0, alpha_sigma=1.0)
CASES = {
    "vmpo_discrete": dict(G.PPO_CASES["ppo_discrete_small"], seed=41),
    "vmpo_continuous": dict(G.PPO_CASES["ppo_continuous_small"], seed=42),
}


def gen(agent_mod, name, case, out_dir=HERE):
    torch.manual_seed(0)
    inp = G.ppo_case_inputs(case)
    params = G.make_params(G.ppo_shapes(case), case["seed"])
    net = "continuous_policy_value" if case["continuous"] else "discrete_policy_value"
    agent = agent_mod.Agent(
        "vmpo", state_size=case["D"], action_size=case["A"], hidden_size=case["H"], network=net,
        optim_config={"name": "adam", "lr": case["lr"]}, gamma=case["gamma"], use_standardization=case["standardize"],
        run_step=1000, lr_decay=False, device="cpu", batch_size=case["batch_size"], n_step=case["T"],
        n_epoch=case["n_epoch"], _lambda=case["lam"], clip_grad_norm=case["clip_grad_norm"], **HP)
    agent.network.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    NT = case["N"] * case["T"]
    agent.memory.first_store = False
    agent.memory.store([{k: inp[k][i:i + 1] for k in ("state", "action", "reward", "next_state", "done")}
                        for i in range(NT)])
    perms = iter(inp["perms"])

    def fake_shuffle(arr):
        arr[:] = next(perms)

    real_shuffle = np.random.shuffle
    np.random.shuffle = fake_shuffle
    try:
        result = agent.learn()
    finally:
        np.random.shuffle = real_shuffle
    out = {f"result.{k}": np.float64(v) for k, v in result.items()}
    out.update({f"init.{k}": v for k, v in params.items()})
    for k, v in agent.network.state_dict().items():
        out[f"param.{k}"] = v.numpy()
    path = os.path.join(out_dir, name + ".npz")
    np.savez_compressed(path, **out)
    return path


if __name__ == "__main__":
    mod = import_reference()[0]
    for n, c in CASES.items():
        print(gen(mod, n, c, sys.argv[1] if len(sys.argv) > 1 else HERE))
