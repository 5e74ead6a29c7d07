"""Drop-in overlay: `src.core.text_corruptor` of the reference, served by simple_tip_b200 (H100 / sm_90a).

Put this repository root before the reference on sys.path (`src` is a namespace package in the
reference, so `src.dnn_test_prio` and `src.plotters` still resolve to the reference).
"""
from simple_tip_b200.core.text_corruptor import *  # noqa: F401,F403
from simple_tip_b200.core import text_corruptor as _impl

globals().update({k: v for k, v in vars(_impl).items() if k.startswith("_") and not k.startswith("__")})
