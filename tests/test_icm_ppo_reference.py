"""ICM-PPO's float64 oracle (oracle/icm_ppo.py) against the UNMODIFIED reference `icm_ppo` agent (CPU).
tests/golden/make_golden_icm_ppo.py mints one reference learn() per case into a temporary directory; the oracle, started
from the same policy and ICM parameters, rollout and permutations, must give the same result dict and post-learn
parameters (fp32 reference vs float64 oracle: rtol 1e-4, atol 1e-5 on results, atol 0.1 * lr on parameters).  The key
names, the module names and the pre-pass order are assumptions until this test has run: parity with the upstream class is
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


@pytest.mark.parametrize("name", ["icm_ppo_discrete", "icm_ppo_continuous"])
def test_oracle_matches_reference_icm_ppo(agent_mod, tmp_path, name):
    import make_golden_icm_ppo as M
    from helpers import ppo_oracle_inputs
    from oracle import icm_ppo as oi
    case = M.CASES[name]
    gold = dict(np.load(M.gen(agent_mod, name, case, out_dir=str(tmp_path))))
    params, batch, hp, perms = ppo_oracle_inputs(case)
    for k, v in params.items():
        np.testing.assert_array_equal(v.numpy(), gold[f"init.{k}"])
    icm = {k[len("icm_init."):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith("icm_init.")}
    bufs = {k: v for k, v in icm.items() if "running" in k or "num_batches" in k}
    icm = {k: v for k, v in icm.items() if k not in bufs}
    hp = dict(hp, A=case["A"])
    ref = oi.learn(params, icm, bufs, batch, hp, M.HP, perms, case["lr"], oi.new_state(case["D"], case["N"]))
    for k, v in ref["result"].items():
        np.testing.assert_allclose(v, float(gold[f"result.{k}"]), rtol=1e-4, atol=1e-5, err_msg=k)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"param.{k}"], rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)
    for k, v in ref["icm"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"icm.{k}"], rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)
