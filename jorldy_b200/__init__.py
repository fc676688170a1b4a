"""jorldy_b200 — H100-native rollout-collect -> buffer -> learn() core behind JORLDY's plugin surface.

Only what the hot path needs lives here: `csrc/` (sm_90a CUDA kernels + C ABI), `_lib.py`
(ctypes binding generated from include/jorldy_b200.h) and `core/` + `manager/` + `run_mode.py`
(the host-side mirror of the reference's Agent / Env / Buffer / Network / Optimizer interface).
"""
__version__ = "0.1.0"
