"""The Munchausen agents' float64 oracle (oracle/munchausen.py) against the UNMODIFIED reference M-DQN and M-IQN (CPU):
tests/golden/make_golden_munchausen.py mints one reference learn() of each into a temporary directory, and the oracle,
started from the same parameters, minibatch and fractions, must give the same loss, max_Q and post-step parameters
(fp32 reference vs float64 oracle: rtol 1e-4, atol 1e-5).  M-IQN's fractions are the reference's recorded draws, taken
in the order this project draws them: the online pass on s, the target pass on s', the target pass on s.  That order and
the constructor keys alpha / tau / l_0 are assumptions until this test has run: parity with the upstream classes is
unpinned.  Needs an upstream JORLDY checkout (JORLDY_REFERENCE=<checkout>/jorldy, tests/golden/refimport.py); skipped
without one."""
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


@pytest.mark.parametrize("name", ["m_dqn", "m_iqn"])
def test_oracle_matches_reference_munchausen_agents(agent_mod, tmp_path, name):
    import make_golden_munchausen as M
    from oracle import munchausen as om
    gold = dict(np.load(M.gen(agent_mod, out_dir=str(tmp_path))))
    case = M.CASE
    init = {n: {k[len(f"{name}.init.{n}."):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith(f"{name}.init.{n}.")}
            for n in ("network", "target_network")}
    batch = {k: torch.from_numpy(gold[f"batch.{k}"]) for k in ("state", "next_state", "action", "reward", "done")}
    hp = dict(gamma=case["gamma"], lr=case["lr"], alpha=case["alpha"], tau=case["tau"], l_0=case["l_0"])
    if name == "m_dqn":
        ref = om.mdqn_learn(init["network"], init["target_network"], batch, hp)
    else:
        taus = [torch.from_numpy(gold[f"m_iqn.tau{i}"]).reshape(case["B"], case["N"]) for i in (0, 1, 2)]
        ref = om.miqn_learn(init["network"], init["target_network"], batch, *taus, dict(hp, D_em=64))
    for k in ("loss", "max_Q"):
        np.testing.assert_allclose(ref["result"][k], float(gold[f"{name}.result.{k}"]), rtol=1e-4, atol=1e-5, err_msg=k)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"{name}.param.{k}"], rtol=1e-4, atol=1e-5, err_msg=k)
