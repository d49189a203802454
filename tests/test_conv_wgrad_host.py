"""CPU: the weight-gradient entry points of the C ABI — host-only planning, descriptor validation, struct layout, and the
one-wgmma-group-per-step property of the compiled kernel (SASS check)."""
import ctypes
import os
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import check_wgmma_groups as cwg  # noqa: E402


def _desc(B=2, M=64, N=64, H=128, W=128, k=3, stride=1, per_sample=0):
    """placeholder pointers: planning never dereferences them"""
    from vtoonify_b200 import _lib
    d = _lib.ConvWgradDesc()
    d.struct_size = ctypes.sizeof(_lib.ConvWgradDesc)
    d.B, d.per_sample, d.stride = B, per_sample, stride
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    d.a, d.a_h, d.a_w, d.M, d.a_cstride = 0x10000, Ho, Wo, M, (M + 31) // 32 * 32
    d.s, d.s_h, d.s_w, d.N, d.s_cstride = 0x20000, H, W, N, (N + 31) // 32 * 32
    d.taps = k * k
    for t in range(k * k):
        d.tap_dy[t], d.tap_dx[t] = t // k - k // 2, t % k - k // 2
    d.out = 0x30000
    return d


def test_workspace_plan_is_host_only_and_descriptor_determined():
    from vtoonify_b200 import _lib
    lib = _lib.load()
    # 64 -> 64, 3x3, B = 2 at 128 x 128: 9 output tiles, so the 1024 K steps of 32 pixels are split 15 ways (132 / 9 rounded up)
    assert lib.vt_conv2d_wgrad_ws_floats(ctypes.byref(_desc())) == 15 * 64 * 64 * 9
    # 512 -> 512 at 32 x 32: 9 taps x 8 M tiles x 2 N tiles = 144 work items, no split
    assert lib.vt_conv2d_wgrad_ws_floats(ctypes.byref(_desc(B=4, M=512, N=512, H=32, W=32))) == 0
    # per-sample results: one slice per sample
    assert lib.vt_conv2d_wgrad_ws_floats(ctypes.byref(_desc(B=4, M=512, N=512, H=32, W=32, per_sample=1))) == 0
    for kw in ({}, {"stride": 2}, {"k": 1, "M": 3, "N": 64, "per_sample": 1}, {"B": 1, "H": 512, "W": 512}):
        vals = {lib.vt_conv2d_wgrad_ws_floats(ctypes.byref(_desc(**kw))) for _ in range(3)}
        assert len(vals) == 1 and min(vals) >= 0, (kw, vals)


def test_rejected_descriptors():
    from vtoonify_b200 import _lib
    lib = _lib.load()
    cases = []
    d = _desc(); d.stride = 3; cases.append((d, b"stride"))
    d = _desc(); d.taps = 37; cases.append((d, b"taps"))
    d = _desc(); d.a_cstride = 48; cases.append((d, b"multiples of 32"))
    d = _desc(); d.s_cstride = 80; cases.append((d, b"multiples of 32"))
    d = _desc(); d.struct_size -= 8; cases.append((d, b"size mismatch"))
    for d, msg in cases:
        assert lib.vt_conv2d_wgrad_ws_floats(ctypes.byref(d)) == -1
        assert msg in lib.vt_last_error(), lib.vt_last_error()
        assert lib.vt_conv2d_wgrad(ctypes.byref(d), None) != 0       # rejected before any device work
        assert msg in lib.vt_last_error()


def test_wgrad_desc_layout_matches_header():
    from vtoonify_b200 import _lib
    fields = ["B", "a", "a_cstride", "s", "s_cstride", "taps", "tap_dy", "tap_dx", "out", "ws", "ws_floats"]
    prog = "#include <stdio.h>\n#include <stddef.h>\n#include \"vtoonify_b200.h\"\nint main(){ printf(\"%zu" + " %zu" * len(fields) + \
        "\\n\", sizeof(vt_conv_wgrad_desc)" + "".join(f", offsetof(vt_conv_wgrad_desc, {f})" for f in fields) + "); return 0; }\n"
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c")
        with open(c, "w") as f:
            f.write(prog)
        exe = os.path.join(td, "t")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        vals = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    D = _lib.ConvWgradDesc
    assert vals == [ctypes.sizeof(D)] + [getattr(D, f).offset for f in fields]


def test_wgrad_steps_are_single_wgmma_groups():
    from vtoonify_b200 import _lib
    if cwg.find_cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip(f"{_lib.LIB_PATH} not built")
    assert cwg.main(["--lib", _lib.LIB_PATH, "--kernel", "conv_wgrad_kernel"]) == 0
