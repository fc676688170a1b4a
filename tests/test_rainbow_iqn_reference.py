"""Rainbow-IQN's float64 oracle (oracle/rainbow_iqn.py) against the UNMODIFIED reference `rainbow_iqn` agent (CPU), and a
GPU-written checkpoint loaded by that class.  tests/golden/make_golden_rainbow_iqn.py mints one reference learn() into a
temporary directory; the oracle, started from the same parameters, minibatch, IS weights, fractions and noise, must give the
same loss, max_Q, max_logit, min_logit, priorities and post-step parameters (fp32 reference vs float64 oracle: rtol 1e-4,
atol 1e-5).  The recorded draws are mapped in the order this project draws them: fractions then the a1, v1, a2, v2 noise
(eps_i, eps_j) of the online pass on s, the online pass on s', the target pass on s'.  That order, the parameter names and
the priority L_b^alpha are assumptions until this test has run: parity with the upstream class is unpinned.  Needs an
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


def test_oracle_matches_reference_rainbow_iqn(agent_mod, tmp_path):
    import make_golden_rainbow_iqn as M
    from oracle import rainbow_iqn as ori
    gold = dict(np.load(M.gen(agent_mod, out_dir=str(tmp_path))))
    case = M.CASE
    B, N = case["B"], case["N"]
    init = {n: {k[len(f"init.{n}."):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith(f"init.{n}.")}
            for n in ("network", "target_network")}
    batch = {k: torch.from_numpy(gold[f"batch.{k}"]) for k in ("state", "next_state", "action", "reward", "done")}
    taus = [torch.from_numpy(gold[f"rand{i}"]).reshape(B, N) for i in range(3)]
    eps = [torch.from_numpy(gold[f"randn{i}"]).reshape(-1).to(torch.float64) for i in range(24)]
    noise = [[(eps[8 * f + 2 * k], eps[8 * f + 2 * k + 1]) for k in range(4)] for f in range(3)]
    ref = ori.learn(init["network"], init["target_network"], batch, torch.from_numpy(gold["weights"]), taus, noise,
                    dict(D_em=64, gamma=case["gamma"], alpha=case["alpha"], lr=case["lr"]))
    for k in ("loss", "max_Q", "max_logit", "min_logit"):
        np.testing.assert_allclose(ref["result"][k], float(gold[f"result.{k}"]), rtol=1e-4, atol=1e-5, err_msg=k)
    np.testing.assert_array_equal(gold["prio.index"], gold["indices"])
    np.testing.assert_allclose(ref["prio"].numpy(), gold["prio.p"], rtol=1e-4, atol=1e-5)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"param.{k}"], rtol=1e-4, atol=1e-5, err_msg=k)


@pytest.mark.gpu
def test_reference_loads_a_gpu_written_checkpoint(agent_mod, tmp_path):
    from jorldy_b200.core import Agent
    kw = dict(state_size=4, action_size=3, hidden_size=32, buffer_size=64, batch_size=8, n_step=3, num_sample=8,
              run_step=100)
    ours = Agent("rainbow_iqn", device="cuda", seed=4, **kw)
    ours.save(str(tmp_path))
    ref = agent_mod.Agent("rainbow_iqn", device="cpu", **kw)
    ref.load(str(tmp_path))                          # the reference's own load()
    sd = ref.network.state_dict()
    assert list(sd) == list(ours.network.p)
    for k, v in ours.network.state_dict().items():
        assert torch.equal(sd[k].cpu(), v.cpu()), k
