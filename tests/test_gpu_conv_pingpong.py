"""GPU: the ping-pong form of the 128 x 128 bf16-split work item (conv_tc_pingpong_kernel<128, 1, 1>, each consumer warpgroup
owns whole items) against the cooperative kernel and the fp32 FFMA kernel.

Option tc_pingpong: 0 = cooperative only, 1 = automatic (launches with at least 3 items per CTA, without the fused ToRGB or
tanh), 2 = ping-pong wherever the instantiation exists, launches of 1 or 2 items per CTA included.  Each output element gets
the same k16 products in the same order and the same epilogue arithmetic in both forms, so all three must be bit-identical,
the instance-norm partial sums included."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

BF16X3_TOL = 3e-5     # max-abs error relative to max(1, |ref|max), as in test_gpu_conv.py
PP_MODES = (0, 1, 2)


@pytest.fixture(scope="module")
def lib():
    from vtoonify_b200 import _lib
    return _lib.load()


def maxerr(a, b):
    assert tuple(a.shape) == tuple(b.shape), f"shape {tuple(a.shape)} vs {tuple(b.shape)}"
    return (a.double() - b.double()).abs().max().item()


def per_mode(lib, fn, modes=PP_MODES, opt="tc_pingpong", **opts):
    """fn() under each mode of `opt` (and the given options), with every option restored afterwards"""
    from vtoonify_b200 import ops
    old = {k: lib.vt_set_option(k.encode(), v) for k, v in opts.items()}
    old_mode = lib.vt_set_option(opt.encode(), 1)
    outs = {}
    try:
        for m in modes:
            lib.vt_set_option(opt.encode(), m)
            outs[m] = fn()
            torch.cuda.synchronize()
    finally:
        lib.vt_set_option(opt.encode(), old_mode)
        for k, v in old.items():
            lib.vt_set_option(k.encode(), v)
        ops.set_precision(ops.DEFAULT_PRECISION)
    return outs


def assert_identical(outs):
    flat = {m: o if isinstance(o, tuple) else (o,) for m, o in outs.items()}
    for m, o in flat.items():
        for a, b in zip(o, flat[0]):
            assert torch.equal(a, b), f"tc_pingpong {m} differs from tc_pingpong 0 by {maxerr(a, b):.3e}"


def conv(x, w, b, k, stride, pad, dil, precision, **epi):
    from vtoonify_b200 import ops
    B, Cin, H, W = x.shape
    xn = ops.to_nhwc(x.cuda(), round_tf32=False)
    wp = ops.prep_weights(w.cuda(), cin_pad=Cin, round_tf32=False)
    Ho, Wo = ops.conv_out_size(H, k, stride, pad, dil), ops.conv_out_size(W, k, stride, pad, dil)
    return ops.to_nchw(ops.conv2d_nhwc([xn], wp, ops.conv_taps(k, pad, dil), stride, Ho, Wo, bias=b.cuda(),
                                       precision=precision, **epi)).cpu()


def _grid_case(sms, items_per_cta):
    """B, H, W of a layer with exactly items_per_cta 8 x 16 pixel tiles per SM (one N tile): one 16-row strip of sms tiles per image"""
    return items_per_cta, 16, 8 * sms


CASES = [
    # B, Cin, Cout, H, W, k, stride, pad, dil
    (2, 128, 128, 24, 40, 3, 1, 1, 1),
    (1, 256, 128, 20, 24, 3, 1, 2, 2),    # dilation 2
    (2, 128, 128, 24, 16, 3, 1, 4, 4),    # dilation 4
    (2, 128, 128, 33, 29, 3, 2, 1, 1),    # stride 2: parity views, odd sizes
    (2, 256, 128, 18, 22, 2, 1, 0, 1),    # k2
    (1, 128, 128, 17, 30, 4, 1, 1, 1),    # k4
    (2, 256, 128, 19, 13, 1, 1, 0, 1),    # 1x1 (per-tap staging)
    (1, 64, 128, 19, 45, 3, 1, 1, 1),     # ragged tiles in both directions
    (1, 32, 256, 21, 37, 3, 1, 1, 1),     # two N tiles per pixel tile (tc_wide 0 below)
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[1]}to{c[2]}_k{c[5]}s{c[6]}d{c[8]}_{c[3]}x{c[4]}" for c in CASES])
def test_pingpong_vs_cooperative_and_fp32(lib, case):
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(sum(case) + 13)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    from vtoonify_b200 import _lib, ops
    Ho, Wo = ops.conv_out_size(H, k, stride, pad, dil), ops.conv_out_size(W, k, stride, pad, dil)
    res = torch.randn((B, Cout, Ho, Wo), generator=g)
    kw = dict(act=_lib.ACT_LRELU, slope=0.2, gain=1.25, alpha=0.5, beta=0.75)
    resn = ops.to_nhwc(res.cuda(), round_tf32=False)
    ref = conv(x, w, b, k, stride, pad, dil, "fp32", res=resn, **kw)
    outs = per_mode(lib, lambda: conv(x, w, b, k, stride, pad, dil, "bf16x3", res=resn, **kw), tc_wide=0)
    assert_identical(outs)
    assert maxerr(outs[1], ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item()), f"{maxerr(outs[1], ref):.3e}"


@pytest.mark.parametrize("items_per_cta", [1, 2, 3])
def test_pingpong_item_counts(lib, items_per_cta):
    """a CTA with one item (only warpgroup 0 works), two, and an odd count (warpgroup 0 owns the last item alone); and a grid with
    fewer items than SMs"""
    B, H, W = _grid_case(torch.cuda.get_device_properties(0).multi_processor_count, items_per_cta)
    for B, W in ((B, W), (1, 40)):
        g = torch.Generator().manual_seed(items_per_cta * 7 + W)
        x = torch.randn((B, 64, H, W), generator=g)
        w = torch.randn((128, 64, 3, 3), generator=g) / np.sqrt(64 * 9)
        b = torch.randn(128, generator=g)
        ref = conv(x, w, b, 3, 1, 1, 1, "fp32")
        outs = per_mode(lib, lambda: conv(x, w, b, 3, 1, 1, 1, "bf16x3"))
        assert_identical(outs)
        assert maxerr(outs[1], ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("shape", [(2, 128, 32, 12, 20), (1, 64, 32, 40, 72)])
def test_pingpong_folded_upconv(lib, shape):
    """Blur o conv_transpose2d as one launch with the 4 output phases stacked along N (n_eff = 4 * 32 = 128), noise and lrelu"""
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
def test_pingpong_two_sources_src_scale(lib, transpose):
    """two sources, the second multiplied by a per-pixel map while it is split (f_E * m_E of the model)"""
    from vtoonify_b200 import ops
    B, C1, Cout, H, W = 2, 96, 128, 23, 30
    g = torch.Generator().manual_seed(31 + transpose)
    a = torch.randn((B, C1, H, W), generator=g); c = torch.randn((B, 32, H, W), generator=g)
    m = torch.rand((B, 1, H, W), generator=g)
    w = torch.randn((Cout, C1 + 32, 3, 3), generator=g) / np.sqrt((C1 + 32) * 9)
    b = torch.randn(Cout, generator=g)
    ref = F.conv2d(torch.cat([a, c * m], 1), w, b, padding=1)
    an, cn, wp = ops.to_nhwc(a.cuda()), ops.to_nhwc(c.cuda()), ops.prep_weights(w.cuda(), cin_pad=C1 + 32)

    def run():
        ops.set_precision("bf16x3")
        y = ops.conv2d_nhwc([an, cn], wp, ops.conv_taps(3, 1), 1, H, W, bias=b.cuda(), src_scale=[None, m.cuda()])
        return ops.to_nchw(y).cpu()

    outs = per_mode(lib, run, tc_transpose=transpose)
    assert_identical(outs)
    assert maxerr(outs[1], ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("transpose", [0, 2])
def test_pingpong_adain_affine_stats_residual(lib, transpose):
    """AdaIN affine on the source while it is split, the output's instance-norm statistics from the epilogue, and a residual"""
    from vtoonify_b200 import ops
    B, Cin, Cout, H, W = 2, 256, 128, 19, 26
    g = torch.Generator().manual_seed(101 + transpose)
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


def test_pingpong_wide_remainder_writes_every_element(lib):
    """the 128-wide remainder launch of a wide layer (first pixel tile m_first > 0) in ping-pong form"""
    from vtoonify_b200 import ops
    B, Cin, Cout, H, W = _split_case(torch.cuda.get_device_properties(0).multi_processor_count)
    g = torch.Generator().manual_seed(9)
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
        assert not torch.isnan(y).any(), f"tc_pingpong {m}: {int(torch.isnan(y).sum())} elements not written"
        assert not torch.isnan(st).any()
    assert_identical(outs)


def _kernel_names(prof):
    return sorted(m.group(1) for e in prof.events() for m in [re.search(r"(conv_tc(?:_pingpong)?_kernel<\d+, \d+, \d+>)", e.name)] if m)


def test_pingpong_on_wide_layer_launches(lib):
    """the 128-wide launches of a wide layer (all of it with tc_wide 0, the remainder with tc_wide 1) run the ping-pong kernel
    with tc_pingpong 2; the automatic plan keeps them cooperative, at 2.4 and 0.4 items per CTA"""
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
        return _kernel_names(prof)

    for pp, narrow in ((1, "conv_tc_kernel<128, 1, 1>"), (2, "conv_tc_pingpong_kernel<128, 1, 1>")):
        got = per_mode(lib, kernels, modes=(0, 1, 2), opt="tc_wide", tc_pingpong=pp)
        assert got[0] == [narrow]
        assert got[1] == sorted([narrow, "conv_tc_kernel<256, 1, 1>"])
        assert got[2] == ["conv_tc_kernel<256, 1, 1>"]


def test_pingpong_kernel_selection(lib):
    """which launches the automatic plan moves: bf16-split 128-wide items, stride 1 and 2, with at least 3 items per CTA;
    not a launch of 2 items per CTA or fewer, tanh or the fp16 split"""
    from torch.profiler import ProfilerActivity, profile
    from vtoonify_b200 import _lib, ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    H, W = 96, 16 * sms    # stride 1: 12 items per SM, stride 2: 3
    g = torch.Generator().manual_seed(3)
    x = ops.to_nhwc(torch.randn((1, 64, H, W), generator=g).cuda(), round_tf32=False)
    x_small = ops.to_nhwc(torch.randn((1, 64, 20, 24), generator=g).cuda(), round_tf32=False)
    x_two = ops.to_nhwc(torch.randn((1, 64, 16, 16 * sms), generator=g).cuda(), round_tf32=False)   # 2 items per SM
    wp = ops.prep_weights((torch.randn((128, 64, 3, 3), generator=g) / 24).cuda(), cin_pad=64, round_tf32=False)

    def names(stride=1, act=0, fmt="bf16", src=x):
        ops.set_precision("bf16x3")
        ops.set_option("rs_fmt", fmt)
        Ho, Wo = src.shape[1] // stride, src.shape[2] // stride
        try:
            ops.conv2d_nhwc([src], wp, ops.conv_taps(3, 1), stride, Ho, Wo, act=act)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ops.conv2d_nhwc([src], wp, ops.conv_taps(3, 1), stride, Ho, Wo, act=act)
                torch.cuda.synchronize()
        finally:
            ops.set_option("rs_fmt", "bf16")
        return _kernel_names(prof)

    coop, pp = ["conv_tc_kernel<128, 1, 1>"], ["conv_tc_pingpong_kernel<128, 1, 1>"]
    assert per_mode(lib, names) == {0: coop, 1: pp, 2: pp}
    assert per_mode(lib, lambda: names(stride=2)) == {0: coop, 1: pp, 2: pp}
    assert per_mode(lib, lambda: names(src=x_small)) == {0: coop, 1: coop, 2: pp}
    assert per_mode(lib, lambda: names(src=x_two)) == {0: coop, 1: coop, 2: pp}
    assert per_mode(lib, lambda: names(act=_lib.ACT_RELU_TANH)) == {0: coop, 1: coop, 2: coop}
    assert per_mode(lib, lambda: names(fmt="f16")) == {m: ["conv_tc_kernel<128, 1, 2>"] for m in PP_MODES}
