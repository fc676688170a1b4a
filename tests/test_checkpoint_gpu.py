"""Checkpoint format parity (jorldy/core/agent/dqn.py:184-199, reinforce.py:128-142): torch.save of
{"network": state_dict, "optimizer": state_dict} at path/ckpt with the reference's state_dict keys, so the
reference's --eval can load GPU-trained weights and vice versa; sync_in / sync_out round trip."""
import os

import numpy as np
import pytest
import torch

import gen_inputs as G

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,kw", [("ppo", {}), ("dqn", {}), ("rainbow", {"n_step": 3}), ("ape_x", {"network": "dueling", "num_workers": 2})])
def test_save_load_roundtrip_and_keys(tmp_path, name, kw):
    from jorldy_b200.core import Agent
    a = Agent(name, state_size=4, action_size=3, hidden_size=32, device="cuda", run_step=100, buffer_size=64, batch_size=8, **kw) \
        if name != "ppo" else Agent(name, state_size=4, action_size=3, hidden_size=32, device="cuda", run_step=100, batch_size=32, n_step=8)
    # take one optimiser step so the optimizer state exists
    for g in a.network.g.values():          # named views only: the flat buffer's alignment padding stays zero
        g.normal_()
    a.optimizer.step(max_norm=1.0)
    a.save(str(tmp_path))
    ck = torch.load(os.path.join(str(tmp_path), "ckpt"), map_location="cpu", weights_only=False)
    assert set(ck.keys()) == {"network", "optimizer"}
    case = {"H": 32, "D": 4, "A": 3, "K": 51, "continuous": False, "agent": name,
            "net": {"ppo": None, "dqn": "discrete_q_network", "rainbow": "rainbow", "ape_x": "dueling"}[name]}
    expected = list(G.ppo_shapes(case).keys()) if name == "ppo" else list(G.q_shapes(case).keys())
    assert list(ck["network"].keys()) == expected                      # same keys, same order as the reference modules
    n_params = len(expected)
    assert sorted(ck["optimizer"]["state"].keys()) == list(range(n_params))
    b = Agent(name, state_size=4, action_size=3, hidden_size=32, device="cuda", run_step=100, buffer_size=64, batch_size=8, **kw) \
        if name != "ppo" else Agent(name, state_size=4, action_size=3, hidden_size=32, device="cuda", run_step=100, batch_size=32, n_step=8)
    b.load(str(tmp_path))
    assert torch.equal(a.network.flat, b.network.flat)
    if hasattr(b, "target_network"):
        assert torch.equal(b.target_network.flat, b.network.flat)      # load sets target := network (dqn.py:198)
    st_a, st_b = a.optimizer.state_dict(), b.optimizer.state_dict()
    for i in range(n_params):
        for k in st_a["state"][i]:
            assert torch.equal(torch.as_tensor(st_a["state"][i][k]).cpu(), torch.as_tensor(st_b["state"][i][k]).cpu())
    # sync_out / sync_in
    w = a.sync_out()["weights"]
    assert all(v.device.type == "cpu" for v in w.values())
    b.network.flat.zero_()
    b.sync_in(w)
    assert torch.equal(a.network.flat, b.network.flat)
