"""The discrete-action SAC's float64 oracle (oracle/sac_discrete.py) against the UNMODIFIED reference SAC with
`actor="discrete_policy"` (CPU): tests/golden/make_golden_sacd.py mints three reference learn() calls into a temporary
directory, and the oracle, started from the same parameters and fed the same minibatch and alpha bookkeeping, must give
the same result dicts and log_alpha (fp32 reference vs float64 oracle: rtol 1e-4, atol 1e-5).  Parity with the
upstream class is otherwise unpinned.  Needs an upstream JORLDY checkout (JORLDY_REFERENCE=<checkout>/jorldy,
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


def test_oracle_matches_reference_discrete_sac(agent_mod, tmp_path):
    import make_golden_sacd as M
    from oracle import sac_discrete as osd
    gold = dict(np.load(M.gen(agent_mod, out_dir=str(tmp_path))))
    case = M.CASE
    init = {n: {k[len(f"init.{n}."):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith(f"init.{n}.")}
            for n in M.NETS}
    batch = {k: torch.from_numpy(gold[f"batch.{k}"]) for k in ("state", "next_state", "action", "reward", "done")}
    hp = dict(gamma=case["gamma"], actor_lr=case["actor_lr"], critic_lr=case["critic_lr"], alpha_lr=case["alpha_lr"],
              use_dynamic_alpha=case["dynamic_alpha"], A=case["A"])
    nets, la = dict(init), torch.tensor([float(gold["init.log_alpha"])], dtype=torch.float64)
    alpha, opt = float(np.exp(gold["init.log_alpha"])), None
    for i in range(case["learns"]):
        ref = osd.learn(nets["actor"], nets["critic1"], nets["critic2"], nets["target_critic1"], nets["target_critic2"], la,
                        alpha, batch, hp, opt)
        for k, v in ref["result"].items():
            np.testing.assert_allclose(v, float(gold[f"result{i}.{k}"]), rtol=1e-4, atol=1e-5, err_msg=f"{k} (learn {i})")
        np.testing.assert_allclose(ref["log_alpha"].item(), float(gold[f"log_alpha{i}"]), rtol=1e-5, atol=1e-7)
        nets = dict(nets, actor=ref["actor"], critic1=ref["critic1"], critic2=ref["critic2"])   # learn() alone: targets stay
        la, alpha, opt = ref["log_alpha"], ref["alpha"], ref["opt_state"]
