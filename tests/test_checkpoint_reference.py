"""SURVEY.md §8f-1 (CPU): a checkpoint WRITTEN by a jorldy_b200 agent on the GPU (tests/golden/ckpt/<agent>/ckpt,
produced by scripts/make_ckpt_fixtures.py) is loaded by the UNMODIFIED reference agent class (`load`, dqn.py:193-199 /
reinforce.py:138-142) and the reference network's eval-mode forward on the recorded input equals what the GPU agent
computed (fp32 tolerance 2e-5) — i.e. the reference's --eval can run GPU-trained weights.  Needs an upstream JORLDY
checkout (JORLDY_REFERENCE=<checkout>/jorldy, tests/golden/refimport.py); skipped without one."""
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
CKPT = os.path.join(HERE, "golden", "ckpt")
CASES = {
    "ppo": ("ppo", dict(state_size=4, action_size=2, hidden_size=64, batch_size=32, n_step=8)),
    "ppo_continuous": ("ppo", dict(state_size=11, action_size=3, hidden_size=64, batch_size=32, n_step=8,
                                   network="continuous_policy_value")),
    "dqn": ("dqn", dict(state_size=4, action_size=3, hidden_size=64, buffer_size=64, batch_size=8)),
    "rainbow": ("rainbow", dict(state_size=4, action_size=3, hidden_size=64, buffer_size=64, batch_size=8, n_step=3,
                                v_min=-1, v_max=10, num_support=51)),
    "ape_x": ("ape_x", dict(state_size=4, action_size=3, hidden_size=64, buffer_size=64, batch_size=8, n_step=3,
                            network="dueling", num_workers=2,
                            optim_config={"name": "rmsprop", "lr": 1e-3, "eps": 1.5e-7, "centered": True})),
}


@pytest.fixture(scope="module")
def agent_mod():
    from refimport import REF_ROOT, import_reference
    if not REF_ROOT or not os.path.isdir(REF_ROOT):
        pytest.skip("reference not present (set JORLDY_REFERENCE to an upstream JORLDY checkout's jorldy/ directory)")
    return import_reference()[0]


@pytest.mark.parametrize("tag", list(CASES))
def test_reference_loads_b200_checkpoint(agent_mod, tag):
    d = os.path.join(CKPT, tag)
    if not os.path.exists(os.path.join(d, "ckpt")):
        pytest.skip(f"no checkpoint fixture for {tag}")
    name, kw = CASES[tag]
    agent = agent_mod.Agent(name, device="cpu", run_step=100, **kw)
    agent.load(d)                                   # the reference's own load()
    exp = dict(np.load(os.path.join(d, "outputs.npz")))
    x = torch.from_numpy(exp["state"])
    agent.network.eval()
    with torch.no_grad():
        if name == "ppo" and "network" not in kw:
            pi, v = agent.network(x)
            ho = torch.from_numpy(exp["head_out"])
            np.testing.assert_allclose(pi.numpy(), torch.softmax(ho[:, :-1], -1).numpy(), rtol=2e-5, atol=2e-6)
            np.testing.assert_allclose(v.numpy(), ho[:, -1:].numpy(), rtol=2e-5, atol=2e-6)
        elif name == "ppo":
            mu, std, v = agent.network(x)
            ho, A = torch.from_numpy(exp["head_out"]), kw["action_size"]
            np.testing.assert_allclose(mu.numpy(), ho[:, :A].clamp(-5, 5).numpy(), rtol=2e-5, atol=2e-6)
            np.testing.assert_allclose(std.numpy(), torch.exp(torch.tanh(ho[:, A:2 * A])).numpy(), rtol=2e-5, atol=2e-6)
            np.testing.assert_allclose(v.numpy(), ho[:, -1:].numpy(), rtol=2e-5, atol=2e-6)
        elif name == "rainbow":
            np.testing.assert_allclose(agent.network(x, False).numpy(), exp["logits"], rtol=2e-5, atol=2e-5)
        else:
            np.testing.assert_allclose(agent.network(x).numpy(), exp["q"], rtol=2e-5, atol=2e-6)
    # the reference's greedy act() on the loaded weights picks the actions the GPU agent picked
    act = agent.act(exp["state"], training=False)["action"]
    if act.dtype.kind == "f":
        np.testing.assert_allclose(act, exp["action_eval"], rtol=0, atol=2e-6)
    else:
        np.testing.assert_array_equal(act.reshape(-1), exp["action_eval"].reshape(-1))
    # optimizer state came along (one step taken before saving)
    st = agent.optimizer.state_dict()["state"]
    assert len(st) == len(list(agent.network.parameters()))


AC_CASES = {
    "ddpg": dict(state_size=3, action_size=2, hidden_size=64, buffer_size=64, batch_size=8),
    "td3": dict(state_size=3, action_size=2, hidden_size=64, buffer_size=64, batch_size=8),
    "sac": dict(state_size=3, action_size=2, hidden_size=64, buffer_size=64, batch_size=8, use_dynamic_alpha=True),
}


@pytest.mark.parametrize("tag", list(AC_CASES))
def test_reference_loads_b200_actor_critic_checkpoint(agent_mod, tag):
    """ddpg.py:186-197 / td3.py:232-246 / sac.py:321-339 load() on a checkpoint written by the GPU agent after two learns."""
    d = os.path.join(CKPT, tag)
    if not os.path.exists(os.path.join(d, "ckpt")):
        pytest.skip(f"no checkpoint fixture for {tag}")
    agent = agent_mod.Agent(tag, device="cpu", run_step=100, **AC_CASES[tag])
    agent.load(d)
    exp = dict(np.load(os.path.join(d, "outputs.npz")))
    x, a = torch.from_numpy(exp["state"]), torch.from_numpy(exp["action"])
    act = agent.act(exp["state"], training=False)["action"]
    np.testing.assert_allclose(act, exp["action_eval"], rtol=0, atol=2e-6)
    with torch.no_grad():
        if tag == "ddpg":
            np.testing.assert_allclose(agent.critic(x, a).numpy(), exp["q1"], rtol=2e-5, atol=2e-6)
        else:       # the reference's load() puts critic2's weights into critic1 and never loads critic2
            np.testing.assert_allclose(agent.critic1(x, a).numpy(), exp["q2"], rtol=2e-5, atol=2e-6)
    opts = [agent.actor_optimizer] + ([agent.critic_optimizer] if tag == "ddpg" else [agent.critic_optimizer1, agent.critic_optimizer2])
    for i, o in enumerate(opts):
        st = o.state_dict()["state"]
        steps = 1.0 if (tag == "td3" and i == 0) else 2.0          # TD3's actor steps on every second learn (td3.py:174)
        assert len(st) == len(o.param_groups[0]["params"]) and all(float(v["step"]) == steps for v in st.values())
    if tag == "sac":
        np.testing.assert_allclose(agent.log_alpha.detach().numpy(), exp["log_alpha"], rtol=0, atol=0)
        assert float(agent.alpha_optimizer.state_dict()["state"][0]["step"]) == 2.0
