"""CPU: the C-ABI library loads and exports exactly the symbols include/vtoonify_b200.h declares (no compute calls)."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vtoonify_b200.h")


def header_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vt_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from vtoonify_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    declared = header_symbols()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported by the .so"
    # the Python binding table covers the header exactly
    assert sorted(_lib.SYMBOLS.keys()) == declared
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = sorted(set(re.findall(r" T (vt_[a-z0-9_]+)$", out, flags=re.M)))
    assert set(declared) <= set(exported)


def test_load_binds_and_reports_abi_version():
    from vtoonify_b200 import _lib
    lib = _lib.load()
    assert lib.vt_abi_version() == _lib.ABI_VERSION == 7
    assert b"abi=7" in lib.vt_build_info()
    assert b"sm_90a" in lib.vt_build_info()
    assert ctypes.sizeof(_lib.ConvDesc) % 8 == 0


def test_struct_layout_matches_header():
    """sizeof/offsetof of the two descriptor structs as compiled by gcc == the ctypes mirror."""
    from vtoonify_b200 import _lib
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "vtoonify_b200.h"
int main(){ printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(vt_conv_desc), offsetof(vt_conv_desc, weight), offsetof(vt_conv_desc, out),
  offsetof(vt_conv_desc, res), sizeof(vt_smalln_desc), offsetof(vt_smalln_desc, weight), offsetof(vt_smalln_desc, mul_c)); return 0; }
'''
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(td, "t")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        vals = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    C, S = _lib.ConvDesc, _lib.SmallNDesc
    assert vals == [ctypes.sizeof(C), C.weight.offset, C.out.offset, C.res.offset, ctypes.sizeof(S), S.weight.offset, S.mul_c.offset]


def test_host_only_entry_points():
    """Entry points that do not touch the device work on the CPU box: out-size arithmetic and argument validation."""
    from vtoonify_b200 import _lib
    lib = _lib.load()
    oh, ow = ctypes.c_int(), ctypes.c_int()
    # Blur after up-conv: (2h+1) -> 2h ; Upsample: n -> 2n ; Downsample: n -> n/2 (SURVEY App. C)
    assert lib.vt_upfirdn2d_out_size(17, 33, 4, 4, 1, 1, 1, 1, 1, 1, 1, 1, oh, ow) == 0 and (oh.value, ow.value) == (16, 32)
    assert lib.vt_upfirdn2d_out_size(8, 10, 4, 4, 2, 2, 1, 1, 2, 1, 2, 1, oh, ow) == 0 and (oh.value, ow.value) == (16, 20)
    assert lib.vt_upfirdn2d_out_size(12, 16, 4, 4, 1, 1, 2, 2, 1, 1, 1, 1, oh, ow) == 0 and (oh.value, ow.value) == (6, 8)
    assert lib.vt_upfirdn2d_out_size(4, 4, 4, 4, 0, 1, 1, 1, 0, 0, 0, 0, oh, ow) != 0
    assert b"up/down" in lib.vt_last_error()
    assert lib.vt_instnorm_ws_bytes(4, 72 * 128, 512, 0) > 0
    assert lib.vt_instnorm_ws_bytes(4, 72 * 128, 6, 0) == -1
    # pivoted partials: (pivot, sum and square sum of x - pivot) per (chunk, b, c) plus one pixel count per chunk;
    # 72x128 at C = 512 plans 144 chunks of 64 pixels
    assert lib.vt_instnorm_partials_floats(144, 4, 512) == 144 * (4 * 512 * 3 + 1)
    assert lib.vt_instnorm_ws_bytes(4, 72 * 128, 512, 0) == 4 * lib.vt_instnorm_partials_floats(144, 4, 512)
    assert lib.vt_instnorm_ws_bytes(4, 72 * 128, 512, 1) == 4 * lib.vt_instnorm_partials_floats(144, 4, 1024)
    assert lib.vt_instnorm_partials_floats(0, 4, 512) == -1
    d = _lib.ConvDesc()
    assert lib.vt_conv2d_tc_supported(d) == 0          # wrong struct_size -> rejected without touching the GPU
    assert lib.vt_conv2d_direct_f32(d, None) != 0 and b"size mismatch" in lib.vt_last_error()


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from vtoonify_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.VtError, match="no CPU"):
        _lib.load()


def _plan_desc(B, Cin, Cout, H, W, k=3, dil=1):
    """A descriptor with placeholder (aligned, never dereferenced) pointers: planning calls launch nothing."""
    from vtoonify_b200 import _lib
    d = _lib.ConvDesc()
    d.struct_size = ctypes.sizeof(_lib.ConvDesc)
    d.n_src = 1
    d.src[0] = 0x10000
    d.src_c[0] = d.src_cstride[0] = Cin
    d.B, d.H, d.W, d.Ho, d.Wo = B, H, W, H, W
    d.stride, d.taps = 1, k * k
    for t in range(k * k):
        d.tap_dy[t], d.tap_dx[t], d.tap_w[t] = (t // k - k // 2) * dil, (t % k - k // 2) * dil, t
    d.n_phase, d.out_cpitch = 1, Cout
    d.weight, d.weight_bf16x3 = 0x20000, 0x40000
    d.wB, d.w_taps, d.w_cstride, d.Cout = 1, k * k, Cin, Cout
    d.out = 0x30000
    d.out_sb, d.out_sy, d.out_sx = H * W * Cout, W * Cout, Cout
    d.alpha = d.beta = 1.0
    return d


def test_output_statistics_plan_is_host_only_and_batch_independent():
    """vt_conv2d_tc_stats_chunks plans without touching the GPU: one chunk per (pixel tile of an image, M tile of the work item,
    consumer warp); the plan must not depend on the batch size (a frame's statistics may not depend on its batch)."""
    from vtoonify_b200 import _lib
    lib = _lib.load()
    # 72 x 128 maps are handed over transposed: 9 x 8 tiles of 8 x 16 pixels x 8 consumer warps of 16 pixels
    assert lib.vt_conv2d_tc_stats_chunks(ctypes.byref(_plan_desc(4, 512, 512, 72, 128))) == 576
    for shape in [(512, 512, 72, 128, 3, 1), (512, 512, 72, 128, 3, 4), (64, 128, 19, 45, 3, 1), (128, 32, 16, 24, 1, 1), (32, 64, 9, 7, 3, 1)]:
        n = [lib.vt_conv2d_tc_stats_chunks(ctypes.byref(_plan_desc(B, *shape))) for B in (1, 2, 4, 7)]
        assert n[0] > 0 and len(set(n)) == 1, (shape, n)
    d = _plan_desc(1, 64, 128, 16, 16)
    d.n_phase = 4                                   # folded up-conv phases cannot deliver statistics
    d.Cout = 32
    assert lib.vt_conv2d_tc_stats_chunks(ctypes.byref(d)) == -1 and lib.vt_last_error()
