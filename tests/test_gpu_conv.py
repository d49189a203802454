"""GPU parity of the convolution kernels: fp32 FFMA kernel vs the oracle's F.conv2d; wgmma kernel vs the FFMA kernel
on TF32-representable data (where both must agree to fp32 accumulation-order noise), for every staging mode."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def maxerr(a, b):
    assert tuple(a.shape) == tuple(b.shape), f"shape {tuple(a.shape)} vs {tuple(b.shape)}"
    return (a.double() - b.double()).abs().max().item()


def set_knob(lib, key, value):
    """vt_set_option for a key the library must know (it returns -1 for an unknown key and changes nothing) -> old value"""
    old = lib.vt_set_option(key, value)
    assert old != -1, f"vt_set_option: the library has no option {key.decode()!r}"
    return old


def tf32_exact(shape, g, scale=1.0):
    """values with <= 8 significant bits: exactly representable in TF32 (10-bit mantissa)"""
    return (torch.randint(-64, 65, shape, generator=g).float() / 32.0) * scale


CASES = [
    # B, Cin, Cout, H, W, k, stride, pad, dil
    (1, 32, 32, 16, 8, 1, 1, 0, 1),      # exactly one tile, 1x1 == plain GEMM
    (2, 32, 64, 16, 16, 3, 1, 1, 1),
    (2, 64, 32, 19, 13, 3, 1, 1, 1),     # partial tiles
    (1, 128, 256, 20, 12, 3, 1, 1, 1),
    (1, 512, 512, 9, 16, 3, 1, 1, 1),    # two N tiles, 16 k-chunks
    (2, 64, 64, 12, 20, 3, 1, 2, 2),     # dilation 2
    (1, 64, 64, 24, 16, 3, 1, 4, 4),     # dilation 4
    (2, 32, 64, 17, 21, 3, 2, 1, 1),     # stride 2 (parity views), odd sizes
    (1, 64, 128, 32, 32, 3, 2, 1, 1),
    (3, 32, 32, 4, 4, 3, 1, 1, 1),       # tiny maps (4x4 features of a 32x32 frame)
]


def _run(ops, x, w, bias, k, stride, pad, dil, precision, **epi):
    xn = ops.to_nhwc(x.cuda(), round_tf32=False)
    wp = ops.prep_weights(w.cuda(), cin_pad=xn.shape[3])
    Ho = ops.conv_out_size(x.shape[2], k, stride, pad, dil)
    Wo = ops.conv_out_size(x.shape[3], k, stride, pad, dil)
    y = ops.conv2d_nhwc([xn], wp, ops.conv_taps(k, pad, dil), stride, Ho, Wo, bias=None if bias is None else bias.cuda(),
                        precision=precision, **epi)
    return ops.to_nchw(y).cpu()


@pytest.mark.parametrize("case", CASES)
def test_direct_vs_torch(case):
    from vtoonify_b200 import ops
    ops.set_precision("fp32")
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    ref = F.conv2d(x, w, b, stride=stride, padding=pad, dilation=dil)
    y = _run(ops, x, w, b, k, stride, pad, dil, "fp32")
    assert maxerr(y, ref) <= 5e-5, maxerr(y, ref)
    ops.set_precision(ops.DEFAULT_PRECISION)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("case", CASES)
def test_tc_vs_direct_exact_data(case, mode):
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007)
    x = tf32_exact((B, Cin, H, W), g)
    w = tf32_exact((Cout, Cin, k, k), g, 1.0 / 8)
    b = torch.randn(Cout, generator=g)
    ops.set_precision("fp32")
    ref = _run(ops, x, w, b, k, stride, pad, dil, "fp32")
    old = set_knob(_lib.load(), b"tc_mode", mode)
    try:
        y = _run(ops, x, w, b, k, stride, pad, dil, "tf32")
    finally:
        _lib.load().vt_set_option(b"tc_mode", old)
        ops.set_precision(ops.DEFAULT_PRECISION)
    scale = ref.abs().max().item()
    assert maxerr(y, ref) <= 2e-5 * max(1.0, scale), f"mode {mode}: err {maxerr(y, ref):.3e} (scale {scale:.1f})"


def test_tc_epilogue_variants():
    from vtoonify_b200 import _lib, ops
    g = torch.Generator().manual_seed(11)
    B, C, H, W = 2, 64, 18, 14
    x = tf32_exact((B, C, H, W), g); w = tf32_exact((C, C, 3, 3), g, 1 / 8)
    b = torch.randn(C, generator=g); res = torch.randn((B, C, H, W), generator=g)
    noise = torch.randn((B, 1, H, W), generator=g); nw = torch.tensor([0.25])
    ref = F.leaky_relu(F.conv2d(x, w, None, padding=1) + nw * noise + b.view(1, -1, 1, 1), 0.2) * 1.5
    ref = ref * 0.7 + 0.3 * res
    for prec in ("fp32", "tf32"):
        ops.set_precision("fp32")  # no output rounding for this check
        y = _run(ops, x, w, b, 3, 1, 1, 1, prec, noise=noise.cuda(), noise_w=nw.cuda(), act=_lib.ACT_LRELU, slope=0.2,
                 gain=1.5, res=ops.to_nhwc(res.cuda(), round_tf32=False), alpha=0.7, beta=0.3)
        assert maxerr(y, ref) <= 1e-4, (prec, maxerr(y, ref))
    ops.set_precision(ops.DEFAULT_PRECISION)


def test_virtual_concat_two_sources():
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(12)
    a = tf32_exact((2, 64, 10, 9), g); c = tf32_exact((2, 32, 10, 9), g)
    w = tf32_exact((64, 96, 3, 3), g, 1 / 8)
    ref = F.conv2d(torch.cat([a, c], 1), w, padding=1)
    for prec in ("fp32", "tf32"):
        ops.set_precision("fp32")
        wp = ops.prep_weights(w.cuda(), cin_pad=96)
        y = ops.conv2d_nhwc([ops.to_nhwc(a.cuda(), round_tf32=False), ops.to_nhwc(c.cuda(), round_tf32=False)], wp,
                            ops.conv_taps(3, 1), 1, 10, 9, precision=prec)
        assert maxerr(ops.to_nchw(y).cpu(), ref) <= 1e-4, prec
    ops.set_precision(ops.DEFAULT_PRECISION)


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
def test_conv_transpose_polyphase(prec):
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(13)
    x = tf32_exact((2, 64, 7, 9), g); w = tf32_exact((32, 64, 3, 3), g, 1 / 8)   # [Cout, Cin, k, k]
    ref = F.conv_transpose2d(x, w.transpose(0, 1), stride=2, padding=0)
    ops.set_precision("fp32")
    wp = ops.prep_weights(w.cuda(), cin_pad=64)
    y = ops.conv_transpose2d_s2_k3_nhwc(ops.to_nhwc(x.cuda(), round_tf32=False), wp, precision=prec)
    ops.set_precision(ops.DEFAULT_PRECISION)
    assert y.shape == (2, 15, 19, 32)
    assert maxerr(ops.to_nchw(y).cpu(), ref) <= 1e-4


def test_tf32_random_data_error_budget():
    """Random (non-representable) data: TF32 error stays within the analytic budget 2^-11-ish relative to output rms."""
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(14)
    x = torch.randn((2, 256, 24, 16), generator=g); w = torch.randn((256, 256, 3, 3), generator=g) / 48
    ref = F.conv2d(x, w, padding=1)
    ops.set_precision("tf32")
    xn = ops.to_nhwc(x.cuda())
    y = ops.conv2d_nhwc([xn], ops.prep_weights(w.cuda(), cin_pad=256), ops.conv_taps(3, 1), 1, 24, 16)
    err = maxerr(ops.to_nchw(y).cpu(), ref)
    rms = ref.pow(2).mean().sqrt().item()
    print(f"tf32 conv 256->256: max err {err:.3e}, rms {rms:.3f}, rel {err / rms:.3e}")
    ops.set_precision(ops.DEFAULT_PRECISION)
    assert err <= 4e-3 * rms


def test_smalln_conv_variants():
    from vtoonify_b200 import _lib, ops
    from oracle import vt_oracle as O
    ops.set_precision("fp32")
    g = torch.Generator().manual_seed(15)
    B, C, H, W = 2, 64, 10, 12
    x = torch.randn((B, C, H, W), generator=g); skip3 = torch.randn((B, 3, H, W), generator=g)
    w = torch.randn((3, C + 3, 3, 3), generator=g) / 24; b = torch.randn(3, generator=g)
    ref = F.conv2d(torch.cat([skip3, x], 1), w, b, padding=1)
    xn = ops.to_nhwc(x.cuda())
    wp = ops.prep_weights(w[:, 3:].contiguous().cuda(), cin_pad=C)
    wpl = w[:, :3].permute(2, 3, 0, 1).reshape(9, 3, 3).contiguous().cuda()
    y = ops.smalln_conv(xn, wp, ops.conv_taps(3, 1), 3, B, H, W, planar=skip3.cuda(), planar_weight=wpl, bias=b.cuda())
    assert maxerr(y.cpu(), ref) <= 2e-5
    # mask head: tanh(relu(conv)) and fused f_E * m
    w1 = torch.randn((1, C, 3, 3), generator=g) / 24; b1 = torch.randn(1, generator=g)
    fe = torch.randn((B, 32, H, W), generator=g)
    m_ref = torch.tanh(F.relu(F.conv2d(x, w1, b1, padding=1)))
    m, fem = ops.smalln_conv(xn, ops.prep_weights(w1.cuda(), cin_pad=C), ops.conv_taps(3, 1), 1, B, H, W, bias=b1.cuda(),
                             act=_lib.ACT_RELU_TANH, mul_src=ops.to_nhwc(fe.cuda()))
    assert maxerr(m.cpu(), m_ref) <= 2e-5
    assert maxerr(ops.to_nchw(fem).cpu(), fe * m_ref) <= 2e-5
    # 1x1 + skip upsample (ToRGB tail)
    w2 = torch.randn((3, C, 1, 1), generator=g) / 8
    sk = torch.randn((B, 3, H // 2, W // 2), generator=g)
    k4 = O.make_kernel([1, 3, 3, 1]) * 4
    ref2 = F.conv2d(x, w2, b) + O.upfirdn2d(sk, k4, up=2, pad=(2, 1))
    y2 = ops.smalln_conv(xn, ops.prep_weights(w2.cuda(), cin_pad=C), [(0, 0, 0)], 3, B, H, W, bias=b.cuda(),
                         skip=sk.cuda(), skip_kernel=k4.cuda())
    assert maxerr(y2.cpu(), ref2) <= 2e-5
    ops.set_precision(ops.DEFAULT_PRECISION)


@pytest.mark.parametrize("mt", [1, 2, 4])
@pytest.mark.parametrize("case", [CASES[1], CASES[2], CASES[3], CASES[5], CASES[9]])
def test_tc_m_tiles_per_work_item(case, mt):
    """Work items of 1/2/4 M tiles sharing each weight tile must give the same result as the FFMA kernel."""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007)
    x = tf32_exact((B, Cin, H, W), g)
    w = tf32_exact((Cout, Cin, k, k), g, 1.0 / 8)
    b = torch.randn(Cout, generator=g)
    ops.set_precision("fp32")
    ref = _run(ops, x, w, b, k, stride, pad, dil, "fp32")
    old = set_knob(_lib.load(), b"tc_mt", mt)
    try:
        y = _run(ops, x, w, b, k, stride, pad, dil, "tf32")
    finally:
        _lib.load().vt_set_option(b"tc_mt", old)
        ops.set_precision(ops.DEFAULT_PRECISION)
    scale = ref.abs().max().item()
    assert maxerr(y, ref) <= 2e-5 * max(1.0, scale), f"mt {mt}: err {maxerr(y, ref):.3e} (scale {scale:.1f})"


@pytest.mark.parametrize("shape", [(2, 64, 32, 7, 9), (1, 128, 64, 16, 24), (2, 32, 32, 33, 20), (1, 512, 256, 8, 8)])
def test_folded_upconv(shape):
    """Blur o conv_transpose2d folded into 4 phase kernels (one launch) vs the two-step reference formulation."""
    from vtoonify_b200 import ops
    from oracle import vt_oracle as O
    B, Cin, Cout, H, W = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = tf32_exact((B, Cin, H, W), g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)
    k4 = O.make_kernel([1, 3, 3, 1]) * 4
    bias = torch.randn(Cout, generator=g); noise = torch.randn((B, 1, 2 * H, 2 * W), generator=g); nw = torch.tensor([0.2])
    ref = O.upfirdn2d(F.conv_transpose2d(x, w.transpose(0, 1), stride=2), k4, pad=(1, 1))
    ref = F.leaky_relu(ref + nw * noise + bias.view(1, -1, 1, 1), 0.2) * 1.4142135
    xn = ops.to_nhwc(x.cuda(), round_tf32=False)
    # fp32: FFMA kernel on un-rounded folded weights == the reference to fp32 noise
    ops.set_precision("fp32")
    wf = ops.fold_upconv_weights(ops.prep_weights(w.cuda(), cin_pad=Cin), k4.cuda())
    y32 = ops.conv_up2_folded_nhwc(xn, wf, bias=bias.cuda(), noise=noise.cuda(), noise_w=nw.cuda(), act=1, gain=1.4142135)
    assert maxerr(ops.to_nchw(y32).cpu(), ref) <= 2e-5 * max(1.0, ref.abs().max().item())
    # tf32: tensor-core kernel vs FFMA kernel on the SAME TF32-rounded folded weights
    ops.set_precision("tf32")
    wfr = ops.fold_upconv_weights(ops.prep_weights(w.cuda(), cin_pad=Cin, round_tf32=False), k4.cuda())
    ops.set_precision("fp32")   # no output rounding in either run
    a = ops.conv_up2_folded_nhwc(xn, wfr, bias=bias.cuda(), noise=noise.cuda(), noise_w=nw.cuda(), act=1, gain=1.4142135, precision="fp32")
    t = ops.conv_up2_folded_nhwc(xn, wfr, bias=bias.cuda(), noise=noise.cuda(), noise_w=nw.cuda(), act=1, gain=1.4142135, precision="tf32")
    ops.set_precision(ops.DEFAULT_PRECISION)
    assert maxerr(ops.to_nchw(t).cpu(), ops.to_nchw(a).cpu()) <= 2e-5 * max(1.0, ref.abs().max().item())
    assert maxerr(ops.to_nchw(t).cpu(), ref) <= 5e-3 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("mt", [0, 1, 2])
@pytest.mark.parametrize("case", [CASES[1], CASES[2], CASES[3], CASES[4], CASES[5], (2, 256, 256, 40, 24, 3, 1, 1, 1), (1, 512, 512, 16, 16, 3, 1, 4, 4),
                                  (2, 64, 256, 17, 9, 3, 1, 1, 1), (2, 32, 32, 33, 70, 3, 1, 1, 1)])
def test_tc_m_tiles_with_epilogue(case, mt):
    """The tensor-core kernel vs the FFMA kernel on the Cout-256 layers and their neighbours, with the full epilogue (leaky ReLU,
    gain, residual with alpha / beta), for the automatic, one and two M tiles per work item (tc_mt)."""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007)
    x = tf32_exact((B, Cin, H, W), g)
    w = tf32_exact((Cout, Cin, k, k), g, 1.0 / 8)
    b = torch.randn(Cout, generator=g)
    res = torch.randn((B, Cout, H, W), generator=g)
    ops.set_precision("fp32")
    kw = dict(act=_lib.ACT_LRELU, slope=0.2, gain=1.25, alpha=0.5, beta=0.75)
    ref = _run(ops, x, w, b, k, stride, pad, dil, "fp32", res=ops.to_nhwc(res.cuda(), round_tf32=False), **kw)
    old = set_knob(_lib.load(), b"tc_mt", mt)
    try:
        y = _run(ops, x, w, b, k, stride, pad, dil, "tf32", res=ops.to_nhwc(res.cuda(), round_tf32=False), **kw)
    finally:
        _lib.load().vt_set_option(b"tc_mt", old)
        ops.set_precision(ops.DEFAULT_PRECISION)
    scale = ref.abs().max().item()
    assert maxerr(y, ref) <= 2e-5 * max(1.0, scale), f"mt {mt}: err {maxerr(y, ref):.3e} (scale {scale:.1f})"


# ---- bf16x3: split-operand tensor-core mode on arbitrary fp32 data ------------------------------------------------------
BF16X3_TOL = 3e-5     # max-abs error relative to max(1, |ref|max): three bf16 products drop only the a_lo*w_lo term (~2^-17)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("case", CASES + [(2, 256, 256, 40, 24, 3, 1, 1, 1)])
def test_bf16x3_vs_direct_random_data(case, mode):
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007 + 1)
    x = torch.randn((B, Cin, H, W), generator=g) * 3.0
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    ops.set_precision("fp32")
    ref = _run(ops, x, w, b, k, stride, pad, dil, "fp32")
    old = set_knob(_lib.load(), b"tc_mode", mode)
    try:
        y = _run(ops, x, w, b, k, stride, pad, dil, "bf16x3")
    finally:
        _lib.load().vt_set_option(b"tc_mode", old)
        ops.set_precision(ops.DEFAULT_PRECISION)
    scale = max(1.0, ref.abs().max().item())
    err = maxerr(y, ref)
    print(f"bf16x3 {case} mode {mode}: err {err:.3e} scale {scale:.2f}")
    assert err <= BF16X3_TOL * scale


@pytest.mark.parametrize("mt,m_major", [(1, 0), (1, 1), (2, 0), (4, 0)])
@pytest.mark.parametrize("case", [CASES[2], CASES[3], CASES[5], (2, 256, 256, 40, 24, 3, 1, 1, 1), (2, 64, 256, 17, 9, 3, 1, 1, 1)])
def test_bf16x3_work_item_shapes(case, mt, m_major):
    """M tiles per work item (tc_mt) and work-item order (tc_m_major: the N tiles of a pixel tile side by side, or N-tile-major)"""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007 + 2)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    res = torch.randn((B, Cout, H, W), generator=g)
    kw = dict(act=_lib.ACT_LRELU, slope=0.2, gain=1.25, alpha=0.5, beta=0.75)
    ops.set_precision("fp32")
    ref = _run(ops, x, w, b, k, stride, pad, dil, "fp32", res=ops.to_nhwc(res.cuda(), round_tf32=False), **kw)
    lib = _lib.load()
    old = (set_knob(lib, b"tc_mt", mt), set_knob(lib, b"tc_m_major", m_major))
    try:
        y = _run(ops, x, w, b, k, stride, pad, dil, "bf16x3", res=ops.to_nhwc(res.cuda(), round_tf32=False), **kw)
    finally:
        lib.vt_set_option(b"tc_mt", old[0]); lib.vt_set_option(b"tc_m_major", old[1])
        ops.set_precision(ops.DEFAULT_PRECISION)
    scale = max(1.0, ref.abs().max().item())
    assert maxerr(y, ref) <= BF16X3_TOL * scale, f"mt {mt} m_major {m_major}: {maxerr(y, ref):.3e} (scale {scale:.1f})"


@pytest.mark.parametrize("shape", [(2, 64, 32, 7, 9), (1, 128, 64, 16, 24), (1, 512, 256, 8, 8)])
def test_bf16x3_folded_upconv_and_concat(shape):
    from vtoonify_b200 import ops
    from oracle import vt_oracle as O
    B, Cin, Cout, H, W = shape
    g = torch.Generator().manual_seed(sum(shape) + 3)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)
    k4 = O.make_kernel([1, 3, 3, 1]) * 4
    bias = torch.randn(Cout, generator=g); noise = torch.randn((B, 1, 2 * H, 2 * W), generator=g); nw = torch.tensor([0.2])
    ref = O.upfirdn2d(F.conv_transpose2d(x, w.transpose(0, 1), stride=2), k4, pad=(1, 1))
    ref = F.leaky_relu(ref + nw * noise + bias.view(1, -1, 1, 1), 0.2) * 1.4142135
    ops.set_precision("bf16x3")
    try:
        xn = ops.to_nhwc(x.cuda())
        wf = ops.fold_upconv_weights(ops.prep_weights(w.cuda(), cin_pad=Cin), k4.cuda())
        y = ops.conv_up2_folded_nhwc(xn, wf, bias=bias.cuda(), noise=noise.cuda(), noise_w=nw.cuda(), act=1, gain=1.4142135)
        assert maxerr(ops.to_nchw(y).cpu(), ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())
        # virtual concat of two sources
        x2 = torch.randn((B, 32, H, W), generator=g)
        w2 = torch.randn((Cout, Cin + 32, 3, 3), generator=g) / np.sqrt((Cin + 32) * 9)
        ref2 = F.conv2d(torch.cat([x, x2], 1), w2, padding=1)
        y2 = ops.conv2d_nhwc([xn, ops.to_nhwc(x2.cuda())], ops.prep_weights(w2.cuda(), cin_pad=Cin + 32), ops.conv_taps(3, 1), 1, H, W)
        assert maxerr(ops.to_nchw(y2).cpu(), ref2) <= BF16X3_TOL * max(1.0, ref2.abs().max().item())
    finally:
        ops.set_precision(ops.DEFAULT_PRECISION)


@pytest.mark.parametrize("transpose,m_major", [(0, 0), (0, 1), (2, 0), (2, 1)])
@pytest.mark.parametrize("case", [CASES[2], CASES[3], CASES[4], CASES[5], (2, 32, 32, 33, 20, 3, 1, 1, 1), (1, 64, 64, 9, 40, 1, 1, 0, 1),
                                  (1, 512, 512, 24, 16, 3, 1, 1, 1)])
def test_tc_transposed_view_and_item_order(case, transpose, m_major):
    """The planner may hand the problem to the kernel transposed (x <-> y), a pure re-indexing that must not change results (noise,
    residual and bias exercise every strided epilogue read), in either work-item order (tc_m_major)."""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007 + 5)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    res = torch.randn((B, Cout, H, W), generator=g)
    noise = torch.randn((B, 1, H, W), generator=g); nw = torch.tensor([0.3])
    kw = dict(act=_lib.ACT_LRELU, slope=0.2, gain=1.25, alpha=0.5, beta=0.75, noise=noise.cuda(), noise_w=nw.cuda())
    ops.set_precision("fp32")
    ref = _run(ops, x, w, b, k, stride, pad, dil, "fp32", res=ops.to_nhwc(res.cuda(), round_tf32=False), **kw)
    lib = _lib.load()
    old = (set_knob(lib, b"tc_transpose", transpose), set_knob(lib, b"tc_m_major", m_major))
    try:
        y = _run(ops, x, w, b, k, stride, pad, dil, "bf16x3", res=ops.to_nhwc(res.cuda(), round_tf32=False), **kw)
    finally:
        lib.vt_set_option(b"tc_transpose", old[0]); lib.vt_set_option(b"tc_m_major", old[1])
        ops.set_precision(ops.DEFAULT_PRECISION)
    scale = max(1.0, ref.abs().max().item())
    assert maxerr(y, ref) <= BF16X3_TOL * scale, f"T {transpose} m_major {m_major}: {maxerr(y, ref):.3e} (scale {scale:.1f})"


@pytest.mark.parametrize("transpose", [0, 2])
@pytest.mark.parametrize("shape", [(2, 64, 32, 7, 9), (1, 128, 64, 16, 24)])
def test_folded_upconv_transposed_view(shape, transpose):
    from vtoonify_b200 import _lib, ops
    from oracle import vt_oracle as O
    B, Cin, Cout, H, W = shape
    g = torch.Generator().manual_seed(sum(shape) + 9)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)
    k4 = O.make_kernel([1, 3, 3, 1]) * 4
    bias = torch.randn(Cout, generator=g); noise = torch.randn((B, 1, 2 * H, 2 * W), generator=g); nw = torch.tensor([0.2])
    ref = O.upfirdn2d(F.conv_transpose2d(x, w.transpose(0, 1), stride=2), k4, pad=(1, 1))
    ref = F.leaky_relu(ref + nw * noise + bias.view(1, -1, 1, 1), 0.2) * 1.4142135
    lib = _lib.load()
    old = set_knob(lib, b"tc_transpose", transpose)
    ops.set_precision("bf16x3")
    try:
        xn = ops.to_nhwc(x.cuda())
        wf = ops.fold_upconv_weights(ops.prep_weights(w.cuda(), cin_pad=Cin), k4.cuda())
        y = ops.conv_up2_folded_nhwc(xn, wf, bias=bias.cuda(), noise=noise.cuda(), noise_w=nw.cuda(), act=1, gain=1.4142135)
        assert maxerr(ops.to_nchw(y).cpu(), ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())
    finally:
        lib.vt_set_option(b"tc_transpose", old)
        ops.set_precision(ops.DEFAULT_PRECISION)


@pytest.mark.parametrize("shape", [(2, 64, 10, 12), (1, 128, 37, 70), (2, 32, 16, 32), (1, 256, 19, 33)])
@pytest.mark.parametrize("n_out", [1, 2, 3, 4])
def test_smalln_input_stationary_vs_gather_kernel(shape, n_out):
    """The input-stationary 3x3 kernel (each pixel read once, 9 partial dots in smem, shifted sum) against the gather kernel
    and torch: virtual concat [x | |x - x2|], per-tap constants, planar source, bias."""
    from vtoonify_b200 import _lib, ops
    ops.set_precision("fp32")
    B, C, H, W = shape
    g = torch.Generator().manual_seed(sum(shape) + n_out)
    x = torch.randn((B, C, H, W), generator=g); x2 = torch.randn((B, C, H, W), generator=g)
    pl = torch.randn((B, 3, H, W), generator=g)
    w = torch.randn((n_out, 2 * C, 3, 3), generator=g) / np.sqrt(18 * C); b = torch.randn(n_out, generator=g)
    wpl_t = torch.randn((n_out, 3, 3, 3), generator=g) / 5
    kc = torch.randn((1, 9, n_out), generator=g)          # per-tap constants (in-bounds taps only)
    ones = F.conv2d(torch.ones((1, 1, H, W)), torch.eye(9).view(9, 1, 3, 3), padding=1)      # [1,9,H,W] tap-in-bounds mask
    # conv taps are cross-correlation order (ky,kx) -> tap index ky*3+kx
    const = torch.einsum("othw,tn->onhw", ones, kc[0])
    ref = F.conv2d(torch.cat([x, (x - x2).abs()], 1), w, b, padding=1) + F.conv2d(pl, wpl_t, padding=1) + const
    xn, x2n = ops.to_nhwc(x.cuda()), ops.to_nhwc(x2.cuda())
    wp = ops.prep_weights(w.cuda(), cin_pad=2 * C)
    wpl = wpl_t.permute(2, 3, 0, 1).reshape(9, n_out, 3).contiguous().cuda()
    lib = _lib.load()
    outs = []
    for mode in (0, 2):
        old = set_knob(lib, b"smalln_is", mode)
        try:
            y = ops.smalln_conv(xn, wp, ops.conv_taps(3, 1), n_out, B, H, W, planar=pl.cuda(), planar_weight=wpl, bias=b.cuda(),
                                src2=x2n, tap_const=kc.cuda())
        finally:
            lib.vt_set_option(b"smalln_is", old)
        outs.append(y.cpu())
    ops.set_precision(ops.DEFAULT_PRECISION)
    scale = max(1.0, ref.abs().max().item())
    assert maxerr(outs[0], ref) <= 2e-5 * scale, f"gather kernel: {maxerr(outs[0], ref):.3e}"
    assert maxerr(outs[1], ref) <= 2e-5 * scale, f"input-stationary kernel: {maxerr(outs[1], ref):.3e}"


@pytest.mark.parametrize("transpose", [0, 2])
@pytest.mark.parametrize("case", [(2, 32, 64, 19, 13, 3, 1), (1, 128, 128, 24, 40, 3, 1), (2, 64, 32, 9, 16, 1, 0)])
def test_bf16x3_second_source_scaled_per_pixel(case, transpose):
    """conv(cat[a, c * m]) with the planar map m applied while the c tiles are split (Fusion: f_E * m_E never materialised)."""
    from vtoonify_b200 import _lib, ops
    B, C1, Cout, H, W, k, pad = case
    g = torch.Generator().manual_seed(sum(case) + 17)
    a = torch.randn((B, C1, H, W), generator=g); c = torch.randn((B, 32, H, W), generator=g)
    m = torch.rand((B, 1, H, W), generator=g)
    w = torch.randn((Cout, C1 + 32, k, k), generator=g) / np.sqrt((C1 + 32) * k * k)
    b = torch.randn(Cout, generator=g)
    ref = F.conv2d(torch.cat([a, c * m], 1), w, b, padding=pad)
    lib = _lib.load()
    old = set_knob(lib, b"tc_transpose", transpose)
    ops.set_precision("bf16x3")
    try:
        y = ops.conv2d_nhwc([ops.to_nhwc(a.cuda()), ops.to_nhwc(c.cuda())], ops.prep_weights(w.cuda(), cin_pad=C1 + 32),
                            ops.conv_taps(k, pad), 1, H, W, bias=b.cuda(), src_scale=[None, m.cuda()])
        assert maxerr(ops.to_nchw(y).cpu(), ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())
        with pytest.raises(_lib.VtError):   # the fp32 FFMA kernel does not implement it: must fail loudly, not ignore the map
            ops.conv2d_nhwc([ops.to_nhwc(a.cuda()), ops.to_nhwc(c.cuda())], ops.prep_weights(w.cuda(), cin_pad=C1 + 32),
                            ops.conv_taps(k, pad), 1, H, W, bias=b.cuda(), src_scale=[None, m.cuda()], precision="fp32")
    finally:
        lib.vt_set_option(b"tc_transpose", old)
        ops.set_precision(ops.DEFAULT_PRECISION)


@pytest.mark.parametrize("mode", [0, 2])
def test_smalln_masked_source(mode):
    from vtoonify_b200 import _lib, ops
    ops.set_precision("fp32")
    g = torch.Generator().manual_seed(23)
    B, C, H, W = 2, 64, 21, 37
    x = torch.randn((B, C, H, W), generator=g); m = torch.rand((B, 1, H, W), generator=g)
    pl = torch.randn((B, 3, H, W), generator=g)
    w = torch.randn((3, C + 3, 3, 3), generator=g) / 24; b = torch.randn(3, generator=g)
    ref = F.conv2d(torch.cat([pl, x * m], 1), w, b, padding=1)
    wp = ops.prep_weights(w[:, 3:].contiguous().cuda(), cin_pad=C)
    wpl = w[:, :3].permute(2, 3, 0, 1).reshape(9, 3, 3).contiguous().cuda()
    lib = _lib.load()
    old = set_knob(lib, b"smalln_is", mode)
    try:
        y = ops.smalln_conv(ops.to_nhwc(x.cuda()), wp, ops.conv_taps(3, 1), 3, B, H, W, planar=pl.cuda(), planar_weight=wpl,
                            bias=b.cuda(), src_mask=m.cuda())
    finally:
        lib.vt_set_option(b"smalln_is", old)
        ops.set_precision(ops.DEFAULT_PRECISION)
    assert maxerr(y.cpu(), ref) <= 2e-5


@pytest.mark.parametrize("with_planar,with_mask", [(True, True), (True, False), (False, False)])
def test_smalln_conv_via_tensor_core_tap_products(with_planar, with_mask):
    """Conv2d.forward_smalln in the bf16x3 mode: 1x1 tensor-core conv producing the 27 per-tap partial products + shifted sum,
    against torch and against the gather kernel."""
    from vtoonify_b200 import ops
    from vtoonify_b200.vtoonify import Conv2d
    g = torch.Generator().manual_seed(29)
    B, C, H, W = 2, 64, 21, 37
    npl = 3 if with_planar else 0
    conv = Conv2d(C + npl, 3, 3, 1, 1, bias=True)
    conv.weight.data = torch.randn(conv.weight.shape, generator=g) / 24
    conv.bias.data = torch.randn(3, generator=g)
    x = torch.randn((B, C, H, W), generator=g); m = torch.rand((B, 1, H, W), generator=g)
    pl = torch.randn((B, 3, H, W), generator=g) if with_planar else None
    xin = x * m if with_mask else x
    ref = F.conv2d(torch.cat([pl, xin], 1) if with_planar else xin, conv.weight.data, conv.bias.data, padding=1)
    conv.cuda()
    ops.set_precision("bf16x3")
    try:
        kw = dict(planar=pl.cuda() if with_planar else None, src_mask=m.cuda() if with_mask else None)
        y_tc = conv.forward_smalln(ops.to_nhwc(x.cuda()), **kw)
        ops.set_option("smalln_via_tc", False)
        y_g = conv.forward_smalln(ops.to_nhwc(x.cuda()), **kw)
    finally:
        ops.set_option("smalln_via_tc", True)
        ops.set_precision(ops.DEFAULT_PRECISION)
    assert maxerr(y_g.cpu(), ref) <= 2e-5
    assert maxerr(y_tc.cpu(), ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("nstack", [False, True])
@pytest.mark.parametrize("mt,m_major", [(0, 1), (1, 0), (2, 1), (4, 0)])
@pytest.mark.parametrize("case", [CASES[0], CASES[2], CASES[9], (2, 32, 32, 33, 70, 3, 1, 1, 1), (1, 128, 32, 24, 40, 3, 1, 2, 2)])
def test_bf16x3_n_stacked_weights(case, mt, m_major, nstack):
    """Cout == 32: weight rows stacked as [w_hi|w_hi] x32 + [w_lo|w_lo] x32 (N = 64, 4 MMAs per tap, halves summed in the
    epilogue) vs the 6-instruction form vs the FFMA kernel; with noise / bias / residual, M tiles per work item and work-item
    order."""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007 + 31)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    res = torch.randn((B, Cout, H, W), generator=g)
    noise = torch.randn((B, 1, H, W), generator=g); nw = torch.tensor([0.3])
    kw = dict(act=_lib.ACT_LRELU, slope=0.2, gain=1.25, alpha=0.5, beta=0.75, noise=noise.cuda(), noise_w=nw.cuda())
    ops.set_precision("fp32")
    ref = _run(ops, x, w, b, k, stride, pad, dil, "fp32", res=ops.to_nhwc(res.cuda(), round_tf32=False), **kw)
    lib = _lib.load()
    old = (set_knob(lib, b"tc_mt", mt), set_knob(lib, b"tc_m_major", m_major))
    ops.set_option("bf16x3_nstack", nstack)
    try:
        y = _run(ops, x, w, b, k, stride, pad, dil, "bf16x3", res=ops.to_nhwc(res.cuda(), round_tf32=False), **kw)
    finally:
        ops.set_option("bf16x3_nstack", False)
        lib.vt_set_option(b"tc_mt", old[0]); lib.vt_set_option(b"tc_m_major", old[1])
        ops.set_precision(ops.DEFAULT_PRECISION)
    scale = max(1.0, ref.abs().max().item())
    assert maxerr(y, ref) <= BF16X3_TOL * scale, f"nstack {nstack} mt {mt} m_major {m_major}: {maxerr(y, ref):.3e} (scale {scale:.1f})"


@pytest.mark.parametrize("transpose", [0, 2])
@pytest.mark.parametrize("case", [CASES[2], CASES[3], CASES[7], (2, 32, 32, 33, 70, 3, 1, 1, 1), "up"])
def test_tc_epilogue_direct_global_stores(case, transpose):
    """The epilogue writes each pixel's channel pairs straight from the accumulator registers to global memory: partial tiles,
    strided phase views (folded up-conv), transposed view, residual + noise."""
    from vtoonify_b200 import _lib, ops
    from oracle import vt_oracle as O
    lib = _lib.load()
    old = set_knob(lib, b"tc_transpose", transpose)
    ops.set_precision("bf16x3")
    try:
        g = torch.Generator().manual_seed(41)
        if case == "up":
            B, Cin, Cout, H, W = 2, 64, 32, 7, 9
            x = torch.randn((B, Cin, H, W), generator=g)
            w = torch.randn((Cout, Cin, 3, 3), generator=g) / np.sqrt(Cin * 9)
            k4 = O.make_kernel([1, 3, 3, 1]) * 4
            bias = torch.randn(Cout, generator=g); noise = torch.randn((B, 1, 2 * H, 2 * W), generator=g); nw = torch.tensor([0.2])
            ref = O.upfirdn2d(F.conv_transpose2d(x, w.transpose(0, 1), stride=2), k4, pad=(1, 1))
            ref = F.leaky_relu(ref + nw * noise + bias.view(1, -1, 1, 1), 0.2) * 1.4142135
            wf = ops.fold_upconv_weights(ops.prep_weights(w.cuda(), cin_pad=Cin), k4.cuda())
            y = ops.to_nchw(ops.conv_up2_folded_nhwc(ops.to_nhwc(x.cuda()), wf, bias=bias.cuda(), noise=noise.cuda(), noise_w=nw.cuda(),
                                                     act=1, gain=1.4142135)).cpu()
        else:
            B, Cin, Cout, H, W, k, stride, pad, dil = case
            x = torch.randn((B, Cin, H, W), generator=g)
            w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
            b = torch.randn(Cout, generator=g)
            Ho, Wo = ops.conv_out_size(H, k, stride, pad, dil), ops.conv_out_size(W, k, stride, pad, dil)
            res = torch.randn((B, Cout, Ho, Wo), generator=g)
            ref = F.conv2d(x, w, b, stride=stride, padding=pad, dilation=dil) * 0.5 + 0.75 * res
            y = _run(ops, x, w, b, k, stride, pad, dil, "bf16x3", res=ops.to_nhwc(res.cuda()), alpha=0.5, beta=0.75)
    finally:
        lib.vt_set_option(b"tc_transpose", old)
        ops.set_precision(ops.DEFAULT_PRECISION)
    assert maxerr(y, ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item()), f"{maxerr(y, ref):.3e}"


@pytest.mark.parametrize("transpose", [0, 2])
@pytest.mark.parametrize("case", [(2, 64, 64, 19, 13, 3, 1, 1), (1, 512, 512, 9, 16, 3, 4, 4), (2, 128, 32, 24, 40, 3, 2, 2), (2, 64, 64, 9, 8, 1, 0, 1)])
def test_bf16x3_per_channel_affine_on_source(case, transpose):
    """conv(pad0(x*scale[b,c] + shift[b,c])) with the affine applied while tiles are split (AdaIN inside the consuming conv):
    the zero padding must stay zero (the reference pads the normalised tensor), incl. dilated taps and the transposed view."""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, pad, dil = case
    g = torch.Generator().manual_seed(sum(case) + 43)
    x = torch.randn((B, Cin, H, W), generator=g) * 2 + 0.5
    aff = torch.randn((B, Cin, 2), generator=g)
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    xn = x * aff[:, :, 0, None, None] + aff[:, :, 1, None, None]
    ref = F.conv2d(xn, w, b, padding=pad, dilation=dil)
    lib = _lib.load()
    old = set_knob(lib, b"tc_transpose", transpose)
    ops.set_precision("bf16x3")
    try:
        y = ops.conv2d_nhwc([ops.to_nhwc(x.cuda())], ops.prep_weights(w.cuda(), cin_pad=Cin), ops.conv_taps(k, pad, dil), 1, H, W,
                            bias=b.cuda(), src_affine=[aff.cuda()])
        assert maxerr(ops.to_nchw(y).cpu(), ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())
        with pytest.raises(_lib.VtError):
            ops.conv2d_nhwc([ops.to_nhwc(x.cuda())], ops.prep_weights(w.cuda(), cin_pad=Cin), ops.conv_taps(k, pad, dil), 1, H, W,
                            bias=b.cuda(), src_affine=[aff.cuda()], precision="fp32")
    finally:
        lib.vt_set_option(b"tc_transpose", old)
        ops.set_precision(ops.DEFAULT_PRECISION)


def test_adain_affine_table_vs_adain_apply():
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(47)
    x = torch.randn((2, 64, 11, 9), generator=g) * 1.5 + 0.3
    gb = torch.randn((2, 128), generator=g)
    xn = ops.to_nhwc(x.cuda())
    st = ops.instnorm_stats(xn)
    ref = ops.adain_apply(xn, st, gb.cuda())
    aff = ops.adain_affine(st, gb.cuda())
    y = xn * aff[:, None, None, :, 0] + aff[:, None, None, :, 1]
    assert (y - ref).abs().max().item() <= 1e-5


# ---- round-2b scheduling options: same results whichever way they are set ---------------------------------------------
@pytest.mark.parametrize("opt,values", [(b"tc_tgroup", (0, 1, 48)), (b"tc_stage_policy", (0, 1)), (b"tc_halo_pct", (50, 60, 100))])
@pytest.mark.parametrize("case", [(2, 512, 512, 24, 40, 3, 1, 4, 4),     # dilation 4: the big-halo stage plan
                                  (1, 256, 256, 33, 20, 3, 1, 2, 2),
                                  (2, 64, 128, 19, 45, 3, 1, 1, 1),      # partial tiles in both directions
                                  (1, 128, 32, 16, 24, 1, 1, 0, 1)])     # 1x1, small N
def test_tc_scheduling_options_do_not_change_results(case, opt, values):
    """Taps per weight box (automatic, one, a 48 KB budget), the pipeline-stage plan of big halo boxes and the halo-staging
    threshold only change WHEN data moves, never what is summed in which order: bit-identical outputs (csrc/conv_tc.cu)."""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007 + 5)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    lib = _lib.load()
    ops.set_precision("fp32")
    ref = _run(ops, x, w, b, k, stride, pad, dil, "fp32")
    outs = []
    old = set_knob(lib, opt, values[0])
    try:
        for v in values:
            set_knob(lib, opt, v)
            outs.append(_run(ops, x, w, b, k, stride, pad, dil, "bf16x3"))
    finally:
        lib.vt_set_option(opt, old)
        ops.set_precision(ops.DEFAULT_PRECISION)
    assert maxerr(outs[0], ref) <= BF16X3_TOL * max(1.0, ref.abs().max().item())
    for o in outs[1:]:
        assert torch.equal(o, outs[0]), f"{opt.decode()} changed the result"


@pytest.mark.parametrize("shape", [(2, 128, 150, 201), (1, 512, 37, 64), (2, 32, 300, 310)])
def test_instnorm_chunk_plans_agree(shape):
    """Small chunks vs ~296 chunks per sample: the same statistics (different partial-sum grouping, double-precision finalize);
    a sample's statistics do not depend on the batch it is in under either plan (csrc/norm_fir.cu)."""
    from vtoonify_b200 import _lib, ops
    B, C, H, W = shape
    g = torch.Generator().manual_seed(B * 1000 + C)
    x = ops.to_nhwc((torch.randn((B, C, H, W), generator=g) * 2.0 + 0.5).cuda())
    x2 = ops.to_nhwc(torch.randn((B, C, H, W), generator=g).cuda())
    lib = _lib.load()
    res = {}
    old = set_knob(lib, b"instnorm_chunks", 0)
    try:
        for plan in (0, 296, 7):
            lib.vt_set_option(b"instnorm_chunks", plan)
            res[plan] = (ops.instnorm_stats(x), ops.instnorm_stats(x, x2))
            one = ops.instnorm_stats(x[:1].contiguous(), x2[:1].contiguous())
            assert torch.equal(one, res[plan][1][:1]), "statistics of a sample depend on its batch"
    finally:
        lib.vt_set_option(b"instnorm_chunks", old)
    xc = ops.to_nchw(x).double()
    mean = xc.mean(dim=(2, 3)); rstd = 1.0 / torch.sqrt(xc.var(dim=(2, 3), unbiased=False) + 1e-5)
    for plan, (s0, s1) in res.items():
        assert (s0[:, :, 0].double() - mean).abs().max().item() <= 1e-5, plan
        assert ((s0[:, :, 1].double() - rstd) / rstd).abs().max().item() <= 1e-5, plan
        assert (s1 - res[0][1]).abs().max().item() <= 2e-6 * max(1.0, res[0][1].abs().max().item()), plan


@pytest.mark.parametrize("case", [(4, 512, 512, 72, 128, 3, 1, 1, 1),    # the res-block layer (transposed view, 2 N tiles)
                                  (2, 512, 512, 24, 40, 3, 1, 4, 4),     # dilation 4
                                  (2, 64, 128, 19, 45, 3, 1, 1, 1),      # 2 M tiles per work item, partial tiles
                                  (1, 128, 32, 16, 24, 1, 1, 0, 1),      # 1x1, N = 32 (4 M tiles per work item)
                                  (3, 32, 64, 9, 7, 3, 1, 1, 1)])        # smaller than one tile
@pytest.mark.parametrize("m_major", [0, 1])
def test_tc_fused_output_statistics(case, m_major):
    """conv2d_nhwc(want_stats=True): per-tile partial sums written by the epilogue warps + finalize == the separate statistics
    pass over the stored output (AdaptiveInstanceNorm, model/dualstylegan.py:10-21); a sample's statistics do not depend on its
    batch; the output itself is untouched."""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 10007 + 9)
    x = ops.to_nhwc((torch.randn((B, Cin, H, W), generator=g) * 1.5).cuda(), round_tf32=False)
    w = ops.prep_weights((torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)).cuda(), cin_pad=Cin)
    b = torch.randn(Cout, generator=g).cuda()
    res = ops.to_nhwc(torch.randn((B, Cout, H, W), generator=g).cuda(), round_tf32=False)
    lib = _lib.load()
    old = set_knob(lib, b"tc_m_major", m_major)
    ops.set_precision("bf16x3")
    try:
        kw = dict(bias=b, act=_lib.ACT_LRELU, slope=0.2, gain=1.0, res=res, alpha=0.7, beta=0.7)
        y0 = ops.conv2d_nhwc([x], w, ops.conv_taps(k, pad, dil), 1, H, W, **kw)
        y, st = ops.conv2d_nhwc([x], w, ops.conv_taps(k, pad, dil), 1, H, W, want_stats=True, **kw)
        assert torch.equal(y, y0)
        ref = ops.instnorm_stats(y)
        assert tuple(st.shape) == (B, Cout, 2)
        assert (st[:, :, 0] - ref[:, :, 0]).abs().max().item() <= 2e-6 * max(1.0, ref[:, :, 0].abs().max().item())
        assert ((st[:, :, 1] - ref[:, :, 1]) / ref[:, :, 1]).abs().max().item() <= 1e-5
        yc = ops.to_nchw(y).double()
        assert (st[:, :, 0].double() - yc.mean(dim=(2, 3))).abs().max().item() <= 1e-5
        _, st1 = ops.conv2d_nhwc([x[:1].contiguous()], w, ops.conv_taps(k, pad, dil), 1, H, W, want_stats=True,
                                 **{**kw, "res": res[:1].contiguous()})
        assert torch.equal(st1, st[:1]), "statistics of a sample depend on its batch"
        ops.set_option("fuse_stats", False)
        _, st2 = ops.conv2d_nhwc([x], w, ops.conv_taps(k, pad, dil), 1, H, W, want_stats=True, **kw)
        assert torch.equal(st2, ref)
    finally:
        ops.set_option("fuse_stats", True)
        lib.vt_set_option(b"tc_m_major", old)
        ops.set_precision(ops.DEFAULT_PRECISION)
