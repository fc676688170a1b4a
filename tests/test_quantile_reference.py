"""The quantile agents' float64 oracle (oracle/quantile.py) against the UNMODIFIED reference QR-DQN and IQN (CPU):
tests/golden/make_golden_quantile.py mints one reference learn() of each into a temporary directory, and the oracle,
started from the same parameters, minibatch and fractions, must give the same loss, max_Q and post-step parameters
(fp32 reference vs float64 oracle: rtol 1e-4, atol 1e-5).  IQN's fractions are the reference's recorded draws: the
first for the online pass on s, the second for the target pass on s'.  Parity with the upstream classes is otherwise
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


@pytest.mark.parametrize("name", ["qrdqn", "iqn"])
def test_oracle_matches_reference_quantile_agents(agent_mod, tmp_path, name):
    import make_golden_quantile as M
    from oracle import quantile as oq
    gold = dict(np.load(M.gen(agent_mod, out_dir=str(tmp_path))))
    case = M.CASE
    init = {n: {k[len(f"{name}.init.{n}."):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith(f"{name}.init.{n}.")}
            for n in ("network", "target_network")}
    batch = {k: torch.from_numpy(gold[f"batch.{k}"]) for k in ("state", "next_state", "action", "reward", "done")}
    if name == "qrdqn":
        ref = oq.qrdqn_learn(init["network"], init["target_network"], batch,
                             dict(A=case["A"], K=case["K"], gamma=case["gamma"], lr=case["lr"]))
    else:
        tau, tau_n = (torch.from_numpy(gold[f"iqn.tau{i}"]).reshape(case["B"], case["N"]) for i in (0, 1))
        ref = oq.iqn_learn(init["network"], init["target_network"], batch, tau, tau_n,
                           dict(D_em=64, gamma=case["gamma"], lr=case["lr"]))
    for k in ("loss", "max_Q"):
        np.testing.assert_allclose(ref["result"][k], float(gold[f"{name}.result.{k}"]), rtol=1e-4, atol=1e-5, err_msg=k)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"{name}.param.{k}"], rtol=1e-4, atol=1e-5, err_msg=k)
