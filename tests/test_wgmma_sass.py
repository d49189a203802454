"""CPU: every conv_tc_kernel instantiation in the built library issues each tap step as one wgmma commit group (SASS check).

A step split into several hardware groups still computes the right result, so no GPU test notices it; only the speed
drops, because waiting for the previous group then waits for the current one too (see tools/check_wgmma_groups.py)."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import check_wgmma_groups as cwg  # noqa: E402


def test_conv_tc_steps_are_single_wgmma_groups():
    from vtoonify_b200 import _lib
    if cwg.find_cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip(f"{_lib.LIB_PATH} not built")
    assert cwg.main(["--lib", _lib.LIB_PATH]) == 0


def test_checker_flags_split_groups_and_placeholders():
    # one bf16x3 step as ptxas emits it when the step holds runtime control flow, then the same step as a single group
    split = ["WARPGROUP.ARRIVE",
             "HGMMA.64x128x16.F32.BF16 R24, gdesc[UR8], R24, UP0",
             "HGMMA.64x128x16.F32.BF16 R24, gdesc[UR8], R24, gsb0",
             "WARPGROUP.ARRIVE",
             "HGMMA.64x128x16.F32.BF16 R24, gdesc[UR8], R24, gsb0",
             "WARPGROUP.ARRIVE",
             "HGMMA.64x8x16.F16 RZ, gdesc[URZ], RZ, !UPT, gsb0",
             "WARPGROUP.DEPBAR.LE gsb0, 0x1"]
    single = ["WARPGROUP.ARRIVE",
              "HGMMA.64x128x16.F32.BF16 R24, gdesc[UR8], R24, UP0",
              "HGMMA.64x128x16.F32.BF16 R24, gdesc[UR8], R24",
              "HGMMA.64x128x16.F32.BF16 R24, gdesc[UR8], R24, gsb0",
              "WARPGROUP.DEPBAR.LE gsb0, 0x1",
              "HGMMA.64x128x16.F32.BF16 R24, gdesc[UR8], R24, gsb0",
              "WARPGROUP.DEPBAR.LE gsb0, 0x0"]
    n_mma, n_groups, problems = cwg.check_groups(split)
    assert (n_mma, n_groups) == (4, 3)
    assert any("placeholder" in p for p in problems)
    assert sum("without a wait" in p for p in problems) == 2
    assert cwg.check_groups(single) == (4, 2, [])
    log = ("ptxas info    : (C7519) warpgroup.arrive is injected in around line 713 by compiler to allow use of registers in GMMA "
           "in function '_ZN43_GLOBAL__N__eb83ca3a_10_conv_tc_cu_23933d8f14conv_tc_kernelILi32EEEvNS_6TcArgsE'\n"
           "ptxas info    : Used 138 registers, used 1 barriers\n")
    assert len(cwg.check_log(log)) == 1
