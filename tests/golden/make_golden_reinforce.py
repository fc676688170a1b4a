"""Golden fixture for REINFORCE: runs the UNMODIFIED reference `reinforce` agent for one learn() on one stored episode,
discrete and continuous, from given parameters, and records the initial parameters, the stored episode, the result
dict and the post-learn parameters.  Parity of this project's REINFORCE with the reference class is not pinned by a
committed fixture: no upstream checkout was available when it was written, so these are assumptions the reference
test exists to check:
  - the constructor keys (state_size, action_size, hidden_size, network, head, optim_config, gamma,
    use_standardization, run_step, lr_decay, device) and the result key "loss";
  - the returns: ret = reward copied, then ret[t] += gamma * ret[t + 1] backwards over the whole buffer, with no reset
    at done flags;
  - the standardisation (ret - mean) / (std + 1e-7) in numpy, std with ddof = 0;
  - the discrete loss -(log(pi.gather(1, a)) * ret).mean() with no probability clamp;
  - the continuous loss -(Normal(mu, std).log_prob(atanh(clamp(a, +-(1 - 1e-7)))) * ret).mean() over M*A elements,
    with no sum over action dims and no tanh Jacobian;
  - one optimiser step with no gradient clipping; the checkpoint {"network", "optimizer"} in path/ckpt.
tests/test_reinforce_reference.py mints this file into a temporary directory and compares it with oracle/reinforce.py
when a checkout is available.  `python tests/golden/make_golden_reinforce.py [out_dir]`."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gen_inputs as G  # noqa: E402
from refimport import import_reference  # noqa: E402

CASES = {
    "reinforce_discrete": dict(continuous=False, D=4, A=2, H=32, T=23, gamma=0.99, lr=1e-3, seed=51),
    "reinforce_continuous": dict(continuous=True, D=3, A=2, H=32, T=29, gamma=0.99, lr=1e-3, seed=52),
}


def shapes(case):
    D, A, H = case["D"], case["A"], case["H"]
    out = {"head.l.weight": (H, D), "head.l.bias": (H,), "l.weight": (H, H), "l.bias": (H,)}
    for name in (("mu", "log_std") if case["continuous"] else ("pi",)):
        out[f"{name}.weight"], out[f"{name}.bias"] = (A, H), (A,)
    return out


def episode(case):
    """One stored episode: state [T, D], action ([T, A] in (-1, 1) or int [T, 1]), reward [T], done (last step only)."""
    rs = np.random.RandomState(case["seed"] + 1000)
    T, D, A = case["T"], case["D"], case["A"]
    state = rs.standard_normal((T, D)).astype(np.float32)
    action = (np.tanh(rs.standard_normal((T, A))).astype(np.float32) if case["continuous"]
              else rs.randint(0, A, (T, 1)).astype(np.int64))
    reward = rs.standard_normal(T).astype(np.float32).astype(np.float64)
    done = np.zeros(T, bool)
    done[-1] = True
    return state, action, reward, done


def gen(agent_mod, name, case, out_dir=HERE):
    torch.manual_seed(0)
    params = G.make_params(shapes(case), case["seed"])
    agent = agent_mod.Agent(
        "reinforce", state_size=case["D"], action_size=case["A"], hidden_size=case["H"],
        network="continuous_policy" if case["continuous"] else "discrete_policy",
        optim_config={"name": "adam", "lr": case["lr"]}, gamma=case["gamma"], use_standardization=True,
        run_step=1000, lr_decay=False, device="cpu")
    agent.network.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    state, action, reward, done = episode(case)
    agent.memory.first_store = False
    agent.memory.store([{"state": state[i:i + 1], "action": action[i:i + 1], "reward": reward[i:i + 1].reshape(1, 1),
                         "next_state": state[i:i + 1], "done": done[i:i + 1].reshape(1, 1)} for i in range(case["T"])])
    result = agent.learn()
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
