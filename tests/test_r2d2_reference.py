"""R2D2's float64 oracle (oracle/r2d2.py) against the UNMODIFIED reference `r2d2` agent (CPU), and a GPU-written
checkpoint loaded by that class.  tests/golden/make_golden_r2d2.py mints one reference learn() into a temporary directory;
the oracle, started from the same parameters, sequences and IS weights, must give the same loss, max_Q, priorities and
post-step parameters (fp32 reference vs float64 oracle: rtol 1e-4, atol 1e-5).  The upstream key names, the previous
action as an input, squared TD against Huber, and the reset at episode starts against zero padding are assumptions
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


def test_oracle_matches_reference_r2d2(agent_mod, tmp_path):
    import make_golden_r2d2 as M
    from oracle import r2d2 as orr
    gold = dict(np.load(M.gen(agent_mod, out_dir=str(tmp_path))))
    case = M.CASE
    init = {n: {k[len(f"init.{n}."):]: torch.from_numpy(v) for k, v in gold.items() if k.startswith(f"init.{n}.")}
            for n in ("network", "target_network")}
    batch = {k: torch.from_numpy(gold[f"batch.{k}"]) for k in
             ("state", "action", "prev_action", "reset", "reward", "done", "h0", "c0")}
    hp = dict(gamma=case["gamma"], n_step=case["n"], n_burn_in=case["Tb"], seq_len=case["T"], eta=case["eta"],
              alpha=case["alpha"], lr=case["lr"], eps=1e-8, clip=40.0, A=case["A"])
    ref = orr.learn(init["network"], init["target_network"], batch, torch.from_numpy(gold["weights"]), hp)
    for k in ("loss", "max_Q"):
        np.testing.assert_allclose(ref["result"][k], float(gold[f"result.{k}"]), rtol=1e-4, atol=1e-5, err_msg=k)
    np.testing.assert_array_equal(gold["prio.index"], gold["indices"])
    np.testing.assert_allclose(ref["prio"].numpy(), gold["prio.p"], rtol=1e-4, atol=1e-5)
    for k, v in ref["params"].items():
        np.testing.assert_allclose(v.numpy(), gold[f"param.{k}"], rtol=1e-4, atol=1e-5, err_msg=k)


@pytest.mark.gpu
def test_reference_loads_a_gpu_written_checkpoint(agent_mod, tmp_path):
    from jorldy_b200.core import Agent
    kw = dict(state_size=4, action_size=3, hidden_size=32, buffer_size=64, batch_size=8, n_step=2, seq_len=4, n_burn_in=2,
              run_step=100)
    ours = Agent("r2d2", device="cuda", seed=4, **kw)
    ours.save(str(tmp_path))
    ref = agent_mod.Agent("r2d2", device="cpu", **kw)
    ref.load(str(tmp_path))                          # the reference's own load()
    sd = ref.network.state_dict()
    assert list(sd) == list(ours.network.p)
    for k, v in ours.network.state_dict().items():
        assert torch.equal(sd[k].cpu(), v.cpu()), k
