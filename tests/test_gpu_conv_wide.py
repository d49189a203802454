"""GPU: the 128 x 256 work item of conv_tc_kernel (m64n256k16, bf16 split) against the 128-wide item and the fp32 FFMA kernel.

Option tc_wide: 0 = 128-wide N tiles only, 1 = automatic (wide items on stride-1 layers, with the whole rounds wide and the
last partial round as a second launch of 128-wide items), 2 = wide items in one launch, stride 2 included.  Each output element gets the same k16 products in the
same order whatever the N tile, so all three must be bit-identical."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

BF16X3_TOL = 3e-5     # max-abs error relative to max(1, |ref|max), as in test_gpu_conv.py
WIDE_MODES = (0, 1, 2)


@pytest.fixture(scope="module")
def lib():
    from vtoonify_b200 import _lib
    return _lib.load()


def maxerr(a, b):
    assert tuple(a.shape) == tuple(b.shape), f"shape {tuple(a.shape)} vs {tuple(b.shape)}"
    return (a.double() - b.double()).abs().max().item()


def per_mode(lib, fn, modes=WIDE_MODES, **opts):
    """fn() under each tc_wide mode (and the given options), with every option restored afterwards"""
    from vtoonify_b200 import ops
    old = {k: lib.vt_set_option(k.encode(), v) for k, v in opts.items()}
    old_wide = lib.vt_set_option(b"tc_wide", 1)
    outs = {}
    try:
        for m in modes:
            lib.vt_set_option(b"tc_wide", m)
            outs[m] = fn()
            torch.cuda.synchronize()
    finally:
        lib.vt_set_option(b"tc_wide", old_wide)
        for k, v in old.items():
            lib.vt_set_option(k.encode(), v)
        ops.set_precision(ops.DEFAULT_PRECISION)
    return outs


def assert_identical(outs):
    flat = {m: o if isinstance(o, tuple) else (o,) for m, o in outs.items()}
    for m, o in flat.items():
        for a, b in zip(o, flat[0]):
            assert torch.equal(a, b), f"tc_wide {m} differs from tc_wide 0 by {maxerr(a, b):.3e}"


def conv(x, w, b, k, stride, pad, dil, precision, **epi):
    from vtoonify_b200 import ops
    B, Cin, H, W = x.shape
    xn = ops.to_nhwc(x.cuda(), round_tf32=False)
    wp = ops.prep_weights(w.cuda(), cin_pad=Cin, round_tf32=False)
    Ho, Wo = ops.conv_out_size(H, k, stride, pad, dil), ops.conv_out_size(W, k, stride, pad, dil)
    return ops.to_nchw(ops.conv2d_nhwc([xn], wp, ops.conv_taps(k, pad, dil), stride, Ho, Wo, bias=b.cuda(),
                                       precision=precision, **epi)).cpu()


CASES = [
    # B, Cin, Cout, H, W, k, stride, pad, dil
    (2, 256, 256, 24, 40, 3, 1, 1, 1),
    (1, 128, 512, 16, 24, 3, 1, 1, 1),
    (1, 512, 256, 20, 24, 3, 1, 2, 2),    # dilation 2
    (2, 256, 512, 24, 16, 3, 1, 4, 4),    # dilation 4: the 48 KB halo box, 2 halo + 4 weight stages
    (2, 128, 256, 33, 29, 3, 2, 1, 1),    # stride 2: parity views, odd sizes
    (1, 256, 512, 32, 24, 3, 2, 1, 1),
    (2, 512, 256, 18, 22, 2, 1, 0, 1),    # k2
    (1, 256, 512, 17, 30, 4, 1, 1, 1),    # k4
    (2, 256, 512, 19, 13, 1, 1, 0, 1),    # 1x1 (per-tap staging)
    (1, 64, 256, 19, 45, 3, 1, 1, 1),     # ragged tiles in both directions
    (2, 512, 512, 24, 16, 3, 1, 1, 1),    # the transposed view is picked: 3 x 1 tiles per image instead of 2 x 2
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[1]}to{c[2]}_k{c[5]}s{c[6]}d{c[8]}_{c[3]}x{c[4]}" for c in CASES])
def test_wide_vs_narrow_and_fp32(lib, case):
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(sum(case) + 11)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    from vtoonify_b200 import _lib, ops
    Ho, Wo = ops.conv_out_size(H, k, stride, pad, dil), ops.conv_out_size(W, k, stride, pad, dil)
    res = torch.randn((B, Cout, Ho, Wo), generator=g)
    kw = dict(act=_lib.ACT_LRELU, slope=0.2, gain=1.25, alpha=0.5, beta=0.75)
    resn = ops.to_nhwc(res.cuda(), round_tf32=False)
    ref = conv(x, w, b, k, stride, pad, dil, "fp32", res=resn, **kw)
    outs = per_mode(lib, lambda: conv(x, w, b, k, stride, pad, dil, "bf16x3", res=resn, **kw))
    assert_identical(outs)
    assert maxerr(outs[1], ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item()), f"{maxerr(outs[1], ref):.3e}"


@pytest.mark.parametrize("transpose", [0, 2])
def test_wide_transposed_view(lib, transpose):
    B, Cin, Cout, H, W = 1, 128, 256, 21, 37
    g = torch.Generator().manual_seed(71 + transpose)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)
    b = torch.randn(Cout, generator=g)
    ref = conv(x, w, b, 3, 1, 1, 1, "fp32")
    outs = per_mode(lib, lambda: conv(x, w, b, 3, 1, 1, 1, "bf16x3"), tc_transpose=transpose)
    assert_identical(outs)
    assert maxerr(outs[1], ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("shape", [(2, 128, 64, 12, 20), (1, 256, 128, 9, 16)])
def test_wide_folded_upconv(lib, shape):
    """Blur o conv_transpose2d as one launch with the 4 output phases stacked along N (n_eff = 4 * Cout = 256 / 512)"""
    from vtoonify_b200 import ops
    from oracle import vt_oracle as O
    B, Cin, Cout, H, W = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)
    k4 = O.make_kernel([1, 3, 3, 1]) * 4
    bias = torch.randn(Cout, generator=g); noise = torch.randn((B, 1, 2 * H, 2 * W), generator=g); nw = torch.tensor([0.2])
    xn = ops.to_nhwc(x.cuda(), round_tf32=False)
    wf = ops.fold_upconv_weights(ops.prep_weights(w.cuda(), cin_pad=Cin, round_tf32=False), k4.cuda())
    kw = dict(bias=bias.cuda(), noise=noise.cuda(), noise_w=nw.cuda(), act=1, gain=1.4142135)
    ref = ops.to_nchw(ops.conv_up2_folded_nhwc(xn, wf, precision="fp32", **kw)).cpu()
    outs = per_mode(lib, lambda: ops.to_nchw(ops.conv_up2_folded_nhwc(xn, wf, precision="bf16x3", **kw)).cpu())
    assert_identical(outs)
    assert maxerr(outs[1], ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("transpose", [0, 2])
def test_wide_adain_affine_stats_residual(lib, transpose):
    """AdaIN affine on the source while it is split, the output's instance-norm statistics from the epilogue, and a residual"""
    from vtoonify_b200 import ops
    B, Cin, Cout, H, W = 2, 256, 512, 19, 26
    g = torch.Generator().manual_seed(97 + transpose)
    x = torch.randn((B, Cin, H, W), generator=g) * 2 + 0.5
    aff = torch.randn((B, Cin, 2), generator=g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)
    b = torch.randn(Cout, generator=g)
    res = torch.randn((B, Cout, H, W), generator=g)
    ref = F.conv2d(x * aff[:, :, 0, None, None] + aff[:, :, 1, None, None], w, b, padding=1) * 0.5 + 0.75 * res
    xn, wp, resn = ops.to_nhwc(x.cuda()), ops.prep_weights(w.cuda(), cin_pad=Cin), ops.to_nhwc(res.cuda(), round_tf32=False)

    def run():
        ops.set_precision("bf16x3")
        y, st = ops.conv2d_nhwc([xn], wp, ops.conv_taps(3, 1), 1, H, W, bias=b.cuda(), src_affine=[aff.cuda()], res=resn,
                                alpha=0.5, beta=0.75, want_stats=True)
        return ops.to_nchw(y).cpu(), st.cpu()

    outs = per_mode(lib, run, tc_transpose=transpose)
    assert_identical(outs)
    y, st = outs[1]
    assert maxerr(y, ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())
    st_ref = ops.instnorm_stats(ops.to_nhwc(y.cuda(), round_tf32=False)).cpu()
    assert maxerr(st, st_ref) <= 1e-4 * max(1.0, st_ref.abs().max().item())


def _split_case(sms):
    """a 3x3 256->256 layer whose 40 pixel tiles per image give more than one round of wide items with a remainder"""
    B = 1
    while 40 * B <= sms or (40 * B) % sms == 0:
        B += 1
    return B, 64, 256, 80, 64


def test_wide_remainder_split_writes_every_element(lib):
    from vtoonify_b200 import ops
    B, Cin, Cout, H, W = _split_case(torch.cuda.get_device_properties(0).multi_processor_count)
    g = torch.Generator().manual_seed(5)
    xn = ops.to_nhwc(torch.randn((B, Cin, H, W), generator=g).cuda(), round_tf32=False)
    wp = ops.prep_weights((torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)).cuda(), cin_pad=Cin, round_tf32=False)
    b = torch.randn(Cout, generator=g).cuda()

    def run():
        ops.set_precision("bf16x3")
        out = torch.full((B, H, W, Cout), float("nan"), device="cuda")
        y, st = ops.conv2d_nhwc([xn], wp, ops.conv_taps(3, 1), 1, H, W, out=out, bias=b, want_stats=True)
        return y.cpu(), st.cpu()

    outs = per_mode(lib, run)
    for m, (y, st) in outs.items():
        assert not torch.isnan(y).any(), f"tc_wide {m}: {int(torch.isnan(y).sum())} elements not written"
        assert not torch.isnan(st).any()
    assert_identical(outs)


def traced_kernels(lib):
    """{tc_wide mode: sorted conv_tc_kernel template arguments} of the split case, from torch.profiler traces"""
    from torch.profiler import ProfilerActivity, profile
    from vtoonify_b200 import ops
    B, Cin, Cout, H, W = _split_case(torch.cuda.get_device_properties(0).multi_processor_count)
    g = torch.Generator().manual_seed(6)
    xn = ops.to_nhwc(torch.randn((B, Cin, H, W), generator=g).cuda(), round_tf32=False)
    wp = ops.prep_weights((torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)).cuda(), cin_pad=Cin, round_tf32=False)

    def kernels():
        ops.set_precision("bf16x3")
        ops.conv2d_nhwc([xn], wp, ops.conv_taps(3, 1), 1, H, W)   # weight split and module load outside the trace
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ops.conv2d_nhwc([xn], wp, ops.conv_taps(3, 1), 1, H, W)
            torch.cuda.synchronize()
        names = [m.group(1) for e in prof.events() for m in [re.search(r"conv_tc_kernel<(\d+, \d+, \d+)>", e.name)] if m]
        return sorted(names)

    return per_mode(lib, kernels)


def test_wide_kernels_are_the_ones_that_run():
    """tc_wide 1 runs conv_tc_kernel<256, 1, 1> on the whole rounds and conv_tc_kernel<128, 1, 1> on the rest; 2 runs the
    wide kernel alone; 0 the 128-wide kernel alone.  Traced in a child process whose only profiler sessions are these: traces
    taken late in a long test process can come back without their kernels."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--trace-kernels"]
    r = subprocess.run(args, cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, f"kernel trace failed:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    line = [l for l in r.stdout.splitlines() if l.startswith("KERNELS ")][-1]
    got = {int(k): v for k, v in json.loads(line[len("KERNELS "):]).items()}
    assert got[0] == ["128, 1, 1"]
    assert got[1] == ["128, 1, 1", "256, 1, 1"]
    assert got[2] == ["256, 1, 1"]


if __name__ == "__main__" and sys.argv[1:] == ["--trace-kernels"]:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from vtoonify_b200 import _lib
    print("KERNELS " + json.dumps(traced_kernels(_lib.load())))
