"""CPU: the ping-pong instantiation conv_tc_pingpong_kernel<128, 1, 1> keeps one wgmma commit group per tap step (both 64-row
halves of the tile in it), and its setmaxnreg plan fits the launch allocation without spills (tools/check_wgmma_groups.py)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import check_wgmma_groups as cwg  # noqa: E402

KERNEL = "conv_tc_pingpong_kernel"


def _built():
    from vtoonify_b200 import _lib
    tool = cwg.find_cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip(f"{_lib.LIB_PATH} not built")
    return tool, _lib.LIB_PATH


def test_pingpong_steps_are_single_wgmma_groups_and_plan_fits():
    _, lib = _built()
    assert cwg.main(["--lib", lib, "--kernel", KERNEL]) == 0


def test_pingpong_instantiation_reallocates_registers():
    tool, lib = _built()
    sass = subprocess.run([tool, "-sass", lib], capture_output=True, text=True, check=True).stdout
    usage = cwg.res_usage(subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True, check=True).stdout)
    funcs = {cwg.short_name(n, KERNEL): (n, insns) for n, insns in cwg.kernel_sass(sass, KERNEL).items()}
    assert sorted(funcs) == [f"{KERNEL}<128, 1, 1>"]
    name, insns = funcs[f"{KERNEL}<128, 1, 1>"]
    assert cwg.maxreg_plan(insns) == (88, 208)
    assert cwg.check_regs(insns, usage.get(name)) == []
    n_mma, n_groups, problems = cwg.check_groups(insns)
    assert (n_mma, n_groups, problems) == (12, 1, [])   # 2 halves x 6 split-operand MMAs, one group per tap step
