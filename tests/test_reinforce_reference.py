"""REINFORCE's float64 oracle (oracle/reinforce.py) against the UNMODIFIED reference `reinforce` agent (CPU).
tests/golden/make_golden_reinforce.py mints one reference learn() per case into a temporary directory; the oracle,
started from the same parameters and episode, must give the same result and post-learn parameters (fp32 reference vs
float64 oracle: rtol 1e-4, atol 1e-5 on results, atol 0.1 * lr on parameters).  A checkpoint written by this project's
agent on the GPU must load in the upstream class.  The assumptions listed in the golden maker hold only once this test
has run: parity with the upstream class is unpinned.  Needs an upstream JORLDY checkout (JORLDY_REFERENCE=<checkout>/jorldy,
tests/golden/refimport.py); skipped without one."""
import os

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def agent_mod():
    from refimport import REF_ROOT, import_reference
    if not REF_ROOT or not os.path.isdir(REF_ROOT):
        pytest.skip("reference not present (set JORLDY_REFERENCE to an upstream JORLDY checkout's jorldy/ directory)")
    return import_reference()[0]


@pytest.mark.parametrize("name", ["reinforce_discrete", "reinforce_continuous"])
def test_oracle_matches_reference_reinforce(agent_mod, tmp_path, name):
    import make_golden_reinforce as M
    from oracle import reinforce as orf
    case = M.CASES[name]
    gold = dict(np.load(M.gen(agent_mod, name, case, out_dir=str(tmp_path))))
    import gen_inputs as G
    params = {k: torch.from_numpy(v) for k, v in G.make_params(M.shapes(case), case["seed"]).items()}
    for k, v in params.items():
        np.testing.assert_array_equal(v.numpy(), gold[f"init.{k}"])
    state, action, reward, _ = M.episode(case)
    ret = orf.reference_returns(reward, case["gamma"], True)
    a = torch.as_tensor(action if case["continuous"] else action.reshape(-1))
    ref = orf.learn(params, torch.as_tensor(state), a, torch.as_tensor(ret), case["A"], case["continuous"], case["lr"])
    np.testing.assert_allclose(ref["loss"], float(gold["result.loss"]), rtol=1e-4, atol=1e-5)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"param.{k}"], rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)


@pytest.mark.parametrize("network, A", [("discrete_policy", 2), ("continuous_policy", 3)])
def test_gpu_checkpoint_loads_in_reference(agent_mod, tmp_path, network, A):
    if not torch.cuda.is_available():
        pytest.skip("writing the checkpoint needs the CUDA agent")
    from jorldy_b200.core.agent.reinforce import REINFORCE
    ours = REINFORCE(state_size=4, action_size=A, hidden_size=32, network=network, device="cuda")
    ours.save(str(tmp_path))
    ref = agent_mod.Agent("reinforce", state_size=4, action_size=A, hidden_size=32, network=network,
                          optim_config={"name": "adam", "lr": 1e-3}, device="cpu")
    ref.load(str(tmp_path))
    for k, v in ref.network.state_dict().items():
        np.testing.assert_array_equal(v.numpy(), ours.network.p[k].cpu().numpy(), err_msg=k)
