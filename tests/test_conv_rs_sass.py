"""CPU: every conv_rs_kernel instantiation in the built library issues each tap step as one wgmma commit group (SASS check, see
tools/check_wgmma_groups.py)."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import check_wgmma_groups as cwg  # noqa: E402


def test_conv_rs_steps_are_single_wgmma_groups():
    from vtoonify_b200 import _lib
    if cwg.find_cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip(f"{_lib.LIB_PATH} not built")
    assert cwg.main(["--lib", _lib.LIB_PATH, "--kernel", "conv_rs_kernel"]) == 0
