"""CPU: the register-budget check of tools/check_wgmma_groups.py (setmaxnreg plan against the launch allocation, no spills).

setmaxnreg.inc waits until enough registers are free, so a plan above what the launch allocated hangs on the GPU instead of
failing; the check has to catch it from the SASS and `cuobjdump -res-usage`."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import check_wgmma_groups as cwg  # noqa: E402

WIDE = "conv_tc_kernel<256, 1, 1>"


def test_register_plan_check():
    insns = ["USETMAXREG.TRY_ALLOC.CTAPOOL UP0, 0xd0", "HGMMA.64x256x16.F32.BF16 R24, gdesc[UR24], R24, gsb0",
             "USETMAXREG.DEALLOC.CTAPOOL 0x58"]
    assert cwg.maxreg_plan(insns) == (88, 208)
    assert cwg.check_regs(insns, (168, 0, 0)) == []
    assert any("exceeds" in p for p in cwg.check_regs(insns, (160, 0, 0)))
    assert any("spills" in p for p in cwg.check_regs(insns, (168, 16, 0)))
    assert any("incomplete" in p for p in cwg.check_regs(insns[:2], (168, 0, 0)))
    assert cwg.check_regs(insns[1:2], None) == []   # no setmaxnreg: nothing to check
    usage = cwg.res_usage(" Function _Z3foov:\n  REG:168 STACK:8 SHARED:1024 LOCAL:4 CONSTANT[0]:2688 TEXTURE:0 SURFACE:0 SAMPLER:0\n")
    assert usage == {"_Z3foov": (168, 8, 4)}


def test_wide_instantiation_is_checked():
    from vtoonify_b200 import _lib
    tool = cwg.find_cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip(f"{_lib.LIB_PATH} not built")
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    usage = cwg.res_usage(subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout)
    funcs = {cwg.short_name(n): (n, insns) for n, insns in cwg.kernel_sass(sass).items()}
    assert WIDE in funcs, sorted(funcs)
    name, insns = funcs[WIDE]
    dec, inc = cwg.maxreg_plan(insns)
    assert dec is not None and inc is not None, "the wide instantiation no longer reallocates registers"
    assert cwg.check_regs(insns, usage.get(name)) == []
    # every other instantiation keeps the flat budget
    assert all(cwg.maxreg_plan(i) == (None, None) for s, (_, i) in funcs.items() if s != WIDE)
