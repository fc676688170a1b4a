"""Golden fixture for MuZero: runs pieces of the UNMODIFIED reference `muzero` agent and records what this project's
oracle and agent must agree with.  Parity of this project's MuZero with the reference class is not pinned by a committed
fixture: no upstream checkout was available when it was written, so these are assumptions the reference test exists to
check:
  - the value converter is `core.network.utils.Converter(support)` with `scalar2vector(x [B, 1]) -> [B, 2 support + 1]`
    (two-hot of h(x) = sign(x)(sqrt(|x| + 1) - 1) + 1e-3 x clamped to the support) and `vector2scalar(p [B, 2 support
    + 1]) -> [B, 1]` (h^-1 of the expectation of the probabilities p);
  - the constructor accepts config.muzero.cartpole's agent keys (num_simulation, num_unroll, td_steps, value_support,
    reward_support, value_loss_coef, hidden_size, latent_size, alpha, beta, ...) on a flat-observation MLP network;
  - act(state, training=False) returns {"action": int array [1, 1]} in [0, A);
  - the checkpoint is {"network", "optimizer"} in path/ckpt.
tests/test_muzero_reference.py mints this file into a temporary directory and compares it with oracle/muzero.py and
this project's config when a checkout is available.  `python tests/golden/make_golden_muzero.py [out_dir]`."""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
from refimport import import_reference  # noqa: E402

CASES = {
    "muzero_transform": dict(kind="transform", V=20, B=64, seed=61),
    "muzero_agent": dict(kind="agent", D=4, A=2, seed=62),
}


def inputs(case):
    """Scalars (inside, at and beyond the support) and probability rows of the transform case."""
    rs = np.random.RandomState(case["seed"])
    V, B = case["V"], case["B"]
    x = np.concatenate([rs.standard_normal(B - 4) * 100.0, [0.0, 333.0, 1e6, -1e6]])
    logits = rs.standard_normal((B, 2 * V + 1)) * 2.0
    p = np.exp(logits - logits.max(-1, keepdims=True))
    return x, p / p.sum(-1, keepdims=True)


def agent_keys():
    sys.path.insert(0, ROOT)
    from jorldy_b200 import config as cfg
    keys = dict(cfg.load("config.muzero.cartpole").agent)
    keys.pop("name")
    return keys


def gen(agent_mod, name, case, out_dir=HERE):
    torch.manual_seed(0)
    out = {}
    if case["kind"] == "transform":
        from core.network.utils import Converter
        conv = Converter(case["V"])
        x, p = inputs(case)
        out["scalar2vector"] = conv.scalar2vector(torch.as_tensor(x).view(-1, 1)).detach().numpy().astype(np.float64)
        out["vector2scalar"] = conv.vector2scalar(torch.as_tensor(p)).detach().numpy().astype(np.float64)
    else:
        agent = agent_mod.Agent("muzero", state_size=case["D"], action_size=case["A"],
                                optim_config={"name": "adam", "lr": 3e-4}, run_step=1000, device="cpu", **agent_keys())
        state = np.random.RandomState(case["seed"]).standard_normal((1, case["D"])).astype(np.float32)
        out["action"] = np.asarray(agent.act(state, training=False)["action"])
        with tempfile.TemporaryDirectory() as d:
            agent.save(d)
            ck = torch.load(os.path.join(d, "ckpt"), map_location="cpu", weights_only=False)
        out["ckpt_keys"] = np.array(sorted(ck))
    path = os.path.join(out_dir, name + ".npz")
    np.savez_compressed(path, **out)
    return path


if __name__ == "__main__":
    mod = import_reference()[0]
    for n, c in CASES.items():
        print(gen(mod, n, c, sys.argv[1] if len(sys.argv) > 1 else HERE))
