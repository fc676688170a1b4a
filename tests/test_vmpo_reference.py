"""V-MPO's float64 oracle (oracle/vmpo.py) against the UNMODIFIED reference `vmpo` agent (CPU).
tests/golden/make_golden_vmpo.py mints one reference learn() per case into a temporary directory; the oracle, started
from the same parameters, rollout and permutations, must give the same result dict and post-learn parameters (fp32
reference vs float64 oracle: rtol 1e-4, atol 1e-5 on results, atol 0.1 * lr on parameters).  The key names, the MSE
without 1/2 and the checkpoint's multiplier entries are assumptions until this test has run: parity with the upstream
class is unpinned.  Needs an upstream JORLDY checkout (JORLDY_REFERENCE=<checkout>/jorldy, tests/golden/refimport.py);
skipped without one."""
import os

import numpy as np
import pytest


@pytest.fixture(scope="module")
def agent_mod():
    from refimport import REF_ROOT, import_reference
    if not REF_ROOT or not os.path.isdir(REF_ROOT):
        pytest.skip("reference not present (set JORLDY_REFERENCE to an upstream JORLDY checkout's jorldy/ directory)")
    return import_reference()[0]


@pytest.mark.parametrize("name", ["vmpo_discrete", "vmpo_continuous"])
def test_oracle_matches_reference_vmpo(agent_mod, tmp_path, name):
    import make_golden_vmpo as M
    from helpers import ppo_oracle_inputs
    from oracle import vmpo as ov
    case = M.CASES[name]
    gold = dict(np.load(M.gen(agent_mod, name, case, out_dir=str(tmp_path))))
    params, batch, hp, perms = ppo_oracle_inputs(case)
    for k, v in params.items():
        np.testing.assert_array_equal(v.numpy(), gold[f"init.{k}"])
    hp = dict(hp, A=case["A"])
    ref = ov.learn(params, batch, hp, perms, case["lr"], (M.HP["eta"], M.HP["alpha_mu"], M.HP["alpha_sigma"]),
                   (M.HP["min_eta"], M.HP["min_alpha_mu"], M.HP["min_alpha_sigma"]),
                   (M.HP["eps_eta"], M.HP["eps_alpha_mu"], M.HP["eps_alpha_sigma"]))
    for k, v in ref["result"].items():
        np.testing.assert_allclose(v, float(gold[f"result.{k}"]), rtol=1e-4, atol=1e-5, err_msg=k)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"param.{k}"], rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)
