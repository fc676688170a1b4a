"""Runs on the GPU: saves checkpoints written by jorldy_b200 agents (after one optimiser step, so the optimizer state is
populated) together with the agents' own eval-mode outputs on a fixed input, under the directory given as the first
argument (default: <tmp>/ckpt_fixtures).  Committed under tests/golden/ckpt/, they are what
tests/test_checkpoint_reference.py (CPU) loads with the UNMODIFIED reference classes (SURVEY.md §8f-1, dqn.py:184-199)."""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from jorldy_b200.core import Agent  # noqa: E402

OUT = sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), "ckpt_fixtures")
CASES = {
    "ppo": dict(kw=dict(state_size=4, action_size=2, hidden_size=64, batch_size=32, n_step=8), D=4),
    "ppo_continuous": dict(name="ppo", kw=dict(state_size=11, action_size=3, hidden_size=64, batch_size=32, n_step=8,
                                               network="continuous_policy_value"), D=11),
    "dqn": dict(kw=dict(state_size=4, action_size=3, hidden_size=64, buffer_size=64, batch_size=8), D=4),
    "rainbow": dict(kw=dict(state_size=4, action_size=3, hidden_size=64, buffer_size=64, batch_size=8, n_step=3,
                            v_min=-1, v_max=10, num_support=51), D=4),
    "ape_x": dict(kw=dict(state_size=4, action_size=3, hidden_size=64, buffer_size=64, batch_size=8, n_step=3,
                          network="dueling", num_workers=2,
                          optim_config={"name": "rmsprop", "lr": 1e-3, "eps": 1.5e-7, "centered": True}), D=4),
}


def main():
    rs = np.random.RandomState(0)
    for tag, c in CASES.items():
        name = c.get("name", tag)
        agent = Agent(name, device="cuda", run_step=100, seed=3, **c["kw"])
        for g in agent.network.g.values():
            g.normal_()
        agent.optimizer.step(max_norm=1.0)
        d = os.path.join(OUT, tag)
        os.makedirs(d, exist_ok=True)
        agent.save(d)
        state = (0.7 * rs.standard_normal((16, c["D"]))).astype(np.float32)
        out = {"state": state, "action_eval": agent.act(state, training=False)["action"]}
        s = torch.from_numpy(state).cuda()
        if name == "ppo":
            o = agent.network._buf("fx.out", (16, agent.network.nout))
            agent.network.forward_rows(s, o)
            out["head_out"] = o.cpu().numpy()
        elif name == "rainbow":
            lg = agent.network._buf("fx.logits", (16, 3, 51))
            agent.network.forward_rows(s, lg, is_train=False)
            out["logits"] = lg.cpu().numpy()
        else:
            out["q"] = agent._q_values(s, False).cpu().numpy().copy()
        np.savez_compressed(os.path.join(d, "outputs.npz"), **out)
        print(tag, "saved", {k: v.shape for k, v in out.items()})


AC_CASES = {
    "ddpg": dict(state_size=3, action_size=2, hidden_size=64, buffer_size=64, batch_size=8),
    "td3": dict(state_size=3, action_size=2, hidden_size=64, buffer_size=64, batch_size=8),
    "sac": dict(state_size=3, action_size=2, hidden_size=64, buffer_size=64, batch_size=8, use_dynamic_alpha=True),
}


def main_ac():
    """DDPG / TD3 / SAC: two learn() calls (every optimiser has state), then save + the agents' own eval outputs."""
    rs = np.random.RandomState(1)
    for tag, kw in AC_CASES.items():
        agent = Agent(tag, device="cuda", run_step=100, seed=3, start_train_step=1, **kw)
        s = (0.7 * rs.standard_normal((16, 3))).astype(np.float32)
        a = np.tanh(rs.standard_normal((16, 2))).astype(np.float32)
        tr = {"state": s, "next_state": s[::-1].copy(), "reward": rs.standard_normal((16, 1)), "done": rs.uniform(size=(16, 1)) < 0.2,
              "action": a}
        for step in (1, 2):
            agent.process([tr], step)
        assert agent.num_learn == 2
        d = os.path.join(OUT, tag)
        os.makedirs(d, exist_ok=True)
        agent.save(d)
        sd, ad = torch.from_numpy(s).cuda(), torch.from_numpy(a).cuda()
        out = {"state": s, "action": a, "action_eval": agent.act(s, training=False)["action"]}
        for i, c in enumerate(agent.critics):
            out[f"q{i + 1}"] = c.forward(sd, ad, tag="fx.").cpu().numpy().copy()
        if tag == "sac":
            out["log_alpha"] = agent.log_alpha.flat[:1].cpu().numpy()
        np.savez_compressed(os.path.join(d, "outputs.npz"), **out)
        print(tag, "saved", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    if "--ac-only" not in sys.argv:
        main()
    main_ac()
