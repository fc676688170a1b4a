"""Imports the UNMODIFIED reference (an upstream JORLDY checkout's `jorldy/` directory, named by the JORLDY_REFERENCE
environment variable) from a writable copy.

Used by the golden-vector makers and by tests/test_checkpoint_reference.py, which skips without it; no other test or
benchmark needs the reference.  A copy is needed because the reference's registries write `_*_dict.txt` next to
themselves at import (core/agent/__init__.py:24 etc.).
"""
import os
import shutil
import sys
import tempfile

REF_ROOT = os.environ.get("JORLDY_REFERENCE", "")


def import_reference():
    if not REF_ROOT or not os.path.isdir(REF_ROOT):
        raise RuntimeError("reference not present: set JORLDY_REFERENCE to an upstream JORLDY checkout's jorldy/ directory")
    dst = os.path.join(tempfile.gettempdir(), "jorldy_ref_copy")
    if not os.path.isdir(dst):
        shutil.copytree(REF_ROOT, dst, ignore=shutil.ignore_patterns("mlagents", "__pycache__"))
    if dst not in sys.path:
        sys.path.insert(0, dst)
    import core.agent as agent_mod      # noqa: E402
    import core.buffer as buffer_mod    # noqa: E402
    import core.network as network_mod  # noqa: E402
    return agent_mod, buffer_mod, network_mod
