"""Golden fixture for RND-PPO: runs the UNMODIFIED reference `rnd_ppo` agent for one learn() on one stored rollout with
the minibatch permutations injected (np.random.shuffle patched, as make_golden.py does for PPO), discrete and continuous,
and records the agent's own initial policy and RND parameters, the result dict and the post-learn parameters.  Parity of
this project's RND-PPO with the reference class is not pinned by a committed fixture: no upstream checkout was available
when it was written, so these are assumptions the reference test exists to check:
  - the constructor key names (rnd_network, gamma_i, extrinsic_coeff, intrinsic_coeff, obs_normalize, ri_normalize,
    batch_norm, non_episodic) and the result keys (PPO's six plus r_i, rnd_loss);
  - the policy network's heads (PPO's plus v_i) and the RND as the agent's `rnd` attribute with the state_dict keys of
    core/network/rnd.py (target.fc1, target.fc2, predictor.fc1, predictor.bn1, predictor.fc2, predictor.fc3);
  - BatchNorm on the predictor only, the advantage mix and the pre-pass order of DESIGN.md section 5g.
tests/test_rnd_ppo_reference.py mints this file into a temporary directory and compares it with oracle/rnd_ppo.py when a
checkout is available.  `python tests/golden/make_golden_rnd_ppo.py [out_dir]`."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gen_inputs as G  # noqa: E402
from refimport import import_reference  # noqa: E402

HP = dict(rnd_network="rnd_mlp", gamma_i=0.99, extrinsic_coeff=2.0, intrinsic_coeff=1.0, obs_normalize=True,
          ri_normalize=True, batch_norm=True, non_episodic=True)
CASES = {
    "rnd_ppo_discrete": dict(G.PPO_CASES["ppo_discrete_small"], seed=61),
    "rnd_ppo_continuous": dict(G.PPO_CASES["ppo_continuous_small"], seed=62),
}


def gen(agent_mod, name, case, out_dir=HERE):
    torch.manual_seed(case["seed"])
    inp = G.ppo_case_inputs(case)
    net = "continuous_policy_value" if case["continuous"] else "discrete_policy_value"
    agent = agent_mod.Agent(
        "rnd_ppo", state_size=case["D"], action_size=case["A"], hidden_size=case["H"], network=net,
        optim_config={"name": "adam", "lr": case["lr"]}, gamma=case["gamma"], use_standardization=case["standardize"],
        run_step=1000, lr_decay=False, device="cpu", batch_size=case["batch_size"], n_step=case["T"],
        n_epoch=case["n_epoch"], _lambda=case["lam"], clip_grad_norm=case["clip_grad_norm"],
        epsilon_clip=case["eps_clip"], vf_coef=case["vf_coef"], ent_coef=case["ent_coef"], **HP)
    out = {f"init.{k}": v.clone().numpy() for k, v in agent.network.state_dict().items()}
    out.update({f"rnd_init.{k}": v.clone().numpy() for k, v in agent.rnd.state_dict().items()})
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
    out.update({f"result.{k}": np.float64(v) for k, v in result.items()})
    for k, v in agent.network.state_dict().items():
        out[f"param.{k}"] = v.numpy()
    for k, v in agent.rnd.state_dict().items():
        out[f"rnd.{k}"] = v.numpy()
    path = os.path.join(out_dir, name + ".npz")
    np.savez_compressed(path, **out)
    return path


if __name__ == "__main__":
    mod = import_reference()[0]
    for n, c in CASES.items():
        print(gen(mod, n, c, sys.argv[1] if len(sys.argv) > 1 else HERE))
