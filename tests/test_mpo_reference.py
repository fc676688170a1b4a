"""MPO's float64 oracle (oracle/mpo.py) against the UNMODIFIED reference `mpo` agent (CPU).
tests/golden/make_golden_mpo.py mints one reference learn() on a fixed batch of discrete-action windows into a temporary
directory; the oracle, started from the same parameters and batch, must give the same result dict and post-learn
parameters (fp32 reference vs float64 oracle: rtol 1e-4, atol 1e-5 on results, atol 0.1 * lr on parameters).  The
assumptions listed in the maker hold until this test has run: parity with the upstream class is unpinned.  Needs an
upstream JORLDY checkout (JORLDY_REFERENCE=<checkout>/jorldy, tests/golden/refimport.py); skipped without one."""
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


def test_oracle_matches_reference_mpo(agent_mod, tmp_path):
    import make_golden_mpo as M
    from oracle import mpo as om
    case = M.CASES["mpo_discrete"]
    gold = dict(np.load(M.gen(agent_mod, "mpo_discrete", case, out_dir=str(tmp_path))))
    get = lambda prefix: {k[len(prefix):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith(prefix)}
    hp = dict(continuous=False, A=case["A"], gamma=case["gamma"], lr=case["lr"], clip_grad_norm=M.HP["clip_grad_norm"],
              target_update_period=M.HP["target_update_period"], critic_loss_type=M.HP["critic_loss_type"],
              eps=(M.HP["eps_eta"], M.HP["eps_alpha_mu"], M.HP["eps_alpha_sigma"]),
              mins=(M.HP["min_eta"], M.HP["min_alpha_mu"], M.HP["min_alpha_sigma"]))
    ref = om.Learner(get("init.actor."), get("init.critic."), (M.HP["eta"], M.HP["alpha_mu"], M.HP["alpha_sigma"]), hp)
    result, _ = ref.learn(get("batch."))
    for k, v in result.items():
        np.testing.assert_allclose(v, float(gold[f"result.{k}"]), rtol=1e-4, atol=1e-5, err_msg=k)
    for net, params in (("actor", ref.actor), ("critic", ref.critic)):
        for k, v in params.items():
            np.testing.assert_allclose(v.detach().numpy(), gold[f"param.{net}.{k}"], rtol=1e-4, atol=0.1 * case["lr"],
                                       err_msg=f"{net}.{k}")
