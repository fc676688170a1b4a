"""MuZero's float64 oracle (oracle/muzero.py) and agent contract against the UNMODIFIED reference `muzero` agent (CPU).
tests/golden/make_golden_muzero.py mints the reference's value converter outputs and its constructor / act / checkpoint
behaviour into a temporary directory; the oracle's transforms must equal the converter's (fp32 or f64 reference vs
float64 oracle: atol 1e-5), and the reference must take this project's config keys and keep the checkpoint layout
{"network", "optimizer"}.  The assumptions listed in the golden maker hold only once this test has run: parity with
the upstream class is unpinned.  Needs an upstream JORLDY checkout (JORLDY_REFERENCE=<checkout>/jorldy,
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


def test_oracle_transforms_match_reference_converter(agent_mod, tmp_path):
    import make_golden_muzero as M
    from oracle import muzero as om
    case = M.CASES["muzero_transform"]
    gold = dict(np.load(M.gen(agent_mod, "muzero_transform", case, out_dir=str(tmp_path))))
    x, p = M.inputs(case)
    V = case["V"]
    np.testing.assert_allclose(om.scalar_to_support(torch.as_tensor(x), V).numpy(),
                               gold["scalar2vector"].reshape(len(x), 2 * V + 1), atol=1e-5)
    np.testing.assert_allclose(om.support_to_scalar(torch.log(torch.as_tensor(p)), V).numpy(),
                               gold["vector2scalar"].reshape(-1), rtol=1e-5, atol=1e-5)


def test_reference_takes_the_config_and_keeps_the_checkpoint_layout(agent_mod, tmp_path):
    import make_golden_muzero as M
    case = M.CASES["muzero_agent"]
    gold = dict(np.load(M.gen(agent_mod, "muzero_agent", case, out_dir=str(tmp_path))))
    a = gold["action"]
    assert a.shape == (1, 1) and 0 <= int(a[0, 0]) < case["A"]
    assert sorted(gold["ckpt_keys"].tolist()) == ["network", "optimizer"]
