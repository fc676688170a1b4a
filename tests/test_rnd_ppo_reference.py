"""RND-PPO's float64 oracle (oracle/rnd_ppo.py) against the UNMODIFIED reference `rnd_ppo` agent (CPU).
tests/golden/make_golden_rnd_ppo.py mints one reference learn() per case into a temporary directory; the oracle, started
from the reference agent's own policy and RND parameters, rollout and permutations, must give the same result dict and
post-learn parameters (fp32 reference vs float64 oracle: rtol 1e-4, atol 1e-5 on results, atol 0.1 * lr on parameters).
The key names, the layer stack, BatchNorm on the predictor only, the advantage mix and the result keys are assumptions
until this test has run: parity with the upstream class is unpinned.  Needs an upstream JORLDY checkout
(JORLDY_REFERENCE=<checkout>/jorldy, tests/golden/refimport.py); skipped without one."""
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


@pytest.mark.parametrize("name", ["rnd_ppo_discrete", "rnd_ppo_continuous"])
def test_oracle_matches_reference_rnd_ppo(agent_mod, tmp_path, name):
    import make_golden_rnd_ppo as M
    from helpers import ppo_oracle_inputs
    from oracle import rnd_ppo as orr
    case = M.CASES[name]
    gold = dict(np.load(M.gen(agent_mod, name, case, out_dir=str(tmp_path))))
    _, batch, hp, perms = ppo_oracle_inputs(case)
    params = {k[len("init."):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith("init.")}
    rnd = {k[len("rnd_init."):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith("rnd_init.")}
    tgt = {k[len("target."):]: v for k, v in rnd.items() if k.startswith("target.")}
    pred = {k[len("predictor."):]: v for k, v in rnd.items() if k.startswith("predictor.")}
    bufs = {k: v for k, v in pred.items() if "running" in k or "num_batches" in k}
    pred = {k: v for k, v in pred.items() if k not in bufs}
    ref = orr.learn(params, tgt, pred, bufs, batch, dict(hp, A=case["A"]), M.HP, perms, case["lr"],
                    orr.new_state(case["D"], case["N"]))
    for k, v in ref["result"].items():
        np.testing.assert_allclose(v, float(gold[f"result.{k}"]), rtol=1e-4, atol=1e-5, err_msg=k)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"param.{k}"], rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)
    for k, v in ref["predictor"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"rnd.predictor.{k}"], rtol=1e-4, atol=0.1 * case["lr"], err_msg=k)
    for k, v in tgt.items():
        np.testing.assert_array_equal(v.numpy(), gold[f"rnd.target.{k}"], err_msg=k)
