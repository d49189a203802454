"""conv2d_gradfix gradients at their edges, element by element against float64 with the bars of tests/wgrad_bounds.py: the
input gradient (the transposed op on the forward kernels, through strided per-phase views with zero fill) where stride-2
geometries leave trailing rows and columns without a tap, with per-axis padding, rectangular kernels, dilation and
groups = batch, in the default bf16x3 mode and in fp32; the weight gradient of the same layers; the bias gradient over channel
counts that are not multiples of 4.  Then gradients through the reference's whole ModulatedConv2d.forward (x, weight,
modulation linear, style through the demodulation) on the drop-in ops, against float64 CPU autograd of the same statements."""
import math
import types

import pytest
import torch
import torch.nn.functional as F

from tests import wgrad_bounds as WB
from tests.test_gpu_gradfix import _reference_modconv_forward

pytestmark = pytest.mark.gpu


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


EDGE_CASES = [
    # B, Cin, Cout, H, W, kh, kw, stride, padding, dilation
    (2, 22, 48, 16, 16, 3, 3, 2, 0, 1),          # 3x3 p0 on an even map: row and column 15 get no tap
    (1, 48, 22, 16, 16, 5, 5, 2, 0, 1),          # 5x5 p0: row and column 15 get no tap
    (2, 3, 22, 15, 18, 3, 3, 2, (1, 0), 1),      # per-axis padding
    (1, 22, 3, 16, 17, 1, 3, 2, (0, 1), 1),      # 1x3, Cout = 3
    (2, 48, 48, 17, 16, 3, 1, 2, (1, 0), 1),     # 3x1
    (1, 22, 48, 20, 19, 3, 3, 2, 2, 2),          # dilation 2
    (2, 3, 3, 16, 16, 3, 3, 2, 0, 1),            # Cin = Cout = 3
    (2, 48, 22, 14, 15, 3, 3, 1, (0, 2), (1, 2)),  # stride 1, per-axis padding and dilation
]


def _pair(v):
    return (v, v) if isinstance(v, int) else v


def _conv_grads(B, Cin, Cout, H, W, kh, kw, s, p, d, groups, bias, seed):
    """(gpu grads, float64 (y, E, R) per gradient) of <conv2d(x, w, b), u>"""
    from vtoonify_b200.op import conv2d_gradfix
    G = groups
    x = _rand((B, G * Cin, H, W), seed)
    w = _rand((G * Cout, Cin, kh, kw), seed + 1, 1 / math.sqrt(Cin * kh * kw))
    b = _rand((G * Cout,), seed + 2, 0.1) if bias else None
    (py, px), (dy, dx) = _pair(p), _pair(d)
    Ho, Wo = (H + 2 * py - dy * (kh - 1) - 1) // s + 1, (W + 2 * px - dx * (kw - 1) - 1) // s + 1
    u = _rand((B, G * Cout, Ho, Wo), seed + 3)
    with torch.enable_grad():
        leaves = [t.cuda().requires_grad_(True) for t in (x, w) + ((b,) if bias else ())]
        y = conv2d_gradfix.conv2d(*leaves, stride=s, padding=p, dilation=d, groups=G)
        assert tuple(y.shape) == tuple(u.shape)
        grads = torch.autograd.grad((y * u.cuda()).sum(), leaves)
    kw_ = dict(stride=s, padding=p, dilation=d, groups=G)
    refs = [WB.bounds(lambda w_, u_: torch.nn.grad.conv2d_input(x.shape, w_, u_, **kw_), w, u),
            WB.bounds(lambda x_, u_: torch.nn.grad.conv2d_weight(x_, w.shape, u_, **kw_), x, u)]
    if bias:
        refs.append(WB.bounds(lambda one, u_: (one * u_).sum((0, 2, 3)), torch.ones(()), u))
    return grads, refs


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("c", EDGE_CASES, ids=[f"e{i}" for i in range(len(EDGE_CASES))])
def test_conv2d_gradients_at_edges(c, precision):
    from vtoonify_b200 import ops
    B, Cin, Cout, H, W, kh, kw, s, p, d = c
    old = ops.set_precision(precision)
    try:
        grads, refs = _conv_grads(B, Cin, Cout, H, W, kh, kw, s, p, d, 1, True, 10)
    finally:
        ops.set_precision(old)
    for name, g, (y64, E, R) in zip(("grad_input", "grad_weight", "grad_bias"), grads, refs):
        WB.check(g, y64, E, R, f"{c} [{precision}] {name}")
    if s == 2 and p == 0 and H == W == 16:
        E = refs[0][1]                                              # row and column 15 get no tap: checked to be exactly 0
        assert (E[:, :, 15] == 0).all() and (E[:, :, :, 15] == 0).all()


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("Cin,Cout,k,s,p", [(22, 48, 3, 2, 0), (48, 3, 3, 2, 1), (3, 22, 1, 2, 0), (48, 48, 3, 1, 1)])
def test_groups_is_batch_gradients_at_batch_8(Cin, Cout, k, s, p, precision):
    """the per-sample form of ModulatedConv2d with 8 samples: input [1, 8 Cin, H, W], weight [8 Cout, Cin, k, k]"""
    from vtoonify_b200 import ops
    old = ops.set_precision(precision)
    try:
        grads, refs = _conv_grads(1, Cin, Cout, 16, 15, k, k, s, p, 1, 8, False, 20)
    finally:
        ops.set_precision(old)
    for name, g, (y64, E, R) in zip(("grad_input", "grad_weight"), grads, refs):
        WB.check(g, y64, E, R, f"groups=8 {Cin}->{Cout} k{k} s{s} p{p} [{precision}] {name}")


@pytest.mark.parametrize("B,C,H,W", [(2, 22, 7, 9), (3, 3, 16, 16), (1, 517, 5, 3), (4, 6, 33, 31)])
def test_channel_sum(B, C, H, W):
    """grad_bias = ops.channel_sum(grad_output) over channel counts that are not multiples of 4"""
    from vtoonify_b200 import ops
    u = _rand((B, C, H, W), 30) + 3.0                               # a mean that dominates: a cancelling sum would hide errors
    y64, E, R = WB.bounds(lambda one, u_: (one * u_).sum((0, 2, 3)), torch.ones(()), u)
    WB.check(ops.channel_sum(u.cuda()), y64, E, R, f"channel_sum {B}x{C}x{H}x{W}")


# ---------------------------------------------------------------------------------------------------------------------------
# whole modulated convolutions
# ---------------------------------------------------------------------------------------------------------------------------
# the bar of every gradient tensor, relative to its max|ref|: the worst error measured on an H100 is 7.9e-6 max|ref| (torgb d/dx;
# every other tensor 3.3e-6 to 6.7e-6), so this leaves at least 5x headroom, and it is 5x tighter than the 2e-4 of
# test_gpu_conv_grad.py
MODCONV_TOL = 4e-5

MODCONV_CASES = [("plain", 4, 12, 10), ("up", 4, 12, 10), ("down", 4, 12, 10), ("torgb", 4, 12, 10), ("plain", 8, 32, 32)]


@pytest.mark.parametrize("mode,B,H,W", MODCONV_CASES, ids=[f"{m}-B{b}-{h}x{w}" for m, b, h, w in MODCONV_CASES])
def test_modulated_conv_backward(mode, B, H, W):
    """gradients of <ModulatedConv2d.forward(x, style), u> w.r.t. x, the weight, modulation.weight / .bias and the style, the
    reference's statements on vtoonify_b200.op against the same statements on F.conv2d / F.conv_transpose2d / the oracle's
    upfirdn2d in float64 on the CPU"""
    import vtoonify_b200.op as vop
    from oracle import vt_oracle as O
    from vtoonify_b200.stylegan import ModulatedConv2d
    from vtoonify_b200.weights import det_state_dict
    Cin = 64
    Cout, k = (3, 1) if mode == "torgb" else (32, 3)
    up, down, demod = mode == "up", mode == "down", mode != "torgb"
    m = ModulatedConv2d(Cin, Cout, k, 512, demodulate=demod, upsample=up, downsample=down)
    sd = {"c." + kk: v for kk, v in det_state_dict(m, seed=11).items()}
    x, style = _rand((B, Cin, H, W), 8), _rand((B, 512), 9)
    blur_pad = tuple(m.blur.pad) if hasattr(m, "blur") else None
    names = ["x", "style", "c.weight", "c.modulation.weight", "c.modulation.bias"]
    cpu_op = types.SimpleNamespace(upfirdn2d=O.upfirdn2d,
                                   conv2d_gradfix=types.SimpleNamespace(conv2d=F.conv2d, conv_transpose2d=F.conv_transpose2d))
    results = []
    with torch.enable_grad():
        for op, dev, dt in ((vop, "cuda", torch.float32), (cpu_op, "cpu", torch.float64)):
            sd_d = {kk: v.to(dev, dt) for kk, v in sd.items()}
            leaves = {"x": x.to(dev, dt), "style": style.to(dev, dt)}
            leaves.update({n: sd_d[n] for n in names[2:]})
            for t in leaves.values():
                t.requires_grad_(True)
            sd_d.update({n: leaves[n] for n in names[2:]})
            y = _reference_modconv_forward(op, leaves["x"], leaves["style"], sd_d, "c.", m.scale, demod, up, down,
                                           sd_d.get("c.blur.kernel"), blur_pad, m.padding)
            u = _rand(tuple(y.shape), 12).to(dev, dt)
            results.append(torch.autograd.grad((y * u).sum(), [leaves[n] for n in names]))
    worst = 0.0
    for n, g, ref in zip(names, *results):
        assert tuple(g.shape) == tuple(ref.shape), n
        err = (g.detach().cpu().double() - ref).abs().max().item()
        scale = ref.abs().max().item()
        rel = err / scale
        worst = max(worst, rel)
        print(f"ModulatedConv2d [{mode}] B={B} {H}x{W} d/d{n}: max|err| {err:.3e} = {rel:.3g} max|ref| (bar {MODCONV_TOL:.3g})")
        assert rel <= MODCONV_TOL, f"[{mode}] d/d{n}: {rel:.3g} > {MODCONV_TOL:.3g}"
