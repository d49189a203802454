"""conv2d_gradfix under autograd (model/stylegan/op/conv2d_gradfix.py:104-227): first and second derivatives of ``conv2d`` /
``conv_transpose2d`` on the GPU against float64 CPU autograd through F.conv2d / F.conv_transpose2d, ``no_weight_gradients()``
and the R1 penalty pattern (util.py:75-80), bit-identical forwards and reproducible gradients."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_gradfix import CONV_CASES

pytestmark = pytest.mark.gpu

TOL = 2e-4     # the TOL of test_gpu_gradfix.py, relative to max|ref|


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


def _close(y, ref, what, tol=TOL):
    assert y is not None, f"{what}: no gradient"
    assert tuple(y.shape) == tuple(ref.shape), f"{what}: shape {tuple(y.shape)} vs {tuple(ref.shape)}"
    err = (y.detach().cpu().double() - ref.detach().double()).abs().max().item()
    scale = max(1e-6, ref.abs().max().item())
    print(f"{what}: max|err| {err:.3e} (max|ref| {scale:.3f})")
    assert err <= tol * scale, f"{what}: {err:.3e} > {tol} * {scale:.3f}"


def _grads(fn, ins, u, device):
    """(output, grads of <fn(*ins), u> w.r.t. every non-None input): float64 on the CPU, float32 on the GPU"""
    if device == "cpu":
        leaves = [None if t is None else t.double().requires_grad_(True) for t in ins]
        u = u.double()
    else:
        leaves = [None if t is None else t.cuda().requires_grad_(True) for t in ins]
        u = u.cuda()
    y = fn(*leaves)
    grads = torch.autograd.grad((y * u).sum(), [t for t in leaves if t is not None])
    return y, grads


def _check_first_backward(gpu_fn, cpu_fn, ins, what):
    with torch.enable_grad():
        y_c = cpu_fn(*[None if t is None else t.double() for t in ins])
        u = _rand(tuple(y_c.shape), 99)
        _, g_c = _grads(cpu_fn, ins, u, "cpu")
        y_g, g_g = _grads(gpu_fn, ins, u, "cuda")
    assert y_g.requires_grad
    names = [n for n, t in zip(("grad_input", "grad_weight", "grad_bias"), ins) if t is not None]
    for n, a, b in zip(names, g_g, g_c):
        _close(a, b, f"{what} {n}")
        if n == "grad_input":
            assert a.is_contiguous()


EXTRA_CASES = [
    # B, Cin, Cout, H, W, kh, kw, stride, padding, dilation, bias
    (2, 32, 64, 17, 15, 3, 3, 2, 0, 1, True),          # 3x3 stride 2, padding 0, odd input
    (2, 64, 32, 16, 13, 1, 1, 2, 0, 1, True),          # 1x1 stride 2: the odd input positions get no gradient taps
    (1, 32, 32, 24, 24, 3, 3, 1, 4, 4, False),         # dilation 4
    (2, 512, 512, 32, 32, 3, 3, 1, 1, 1, True),        # many N and M tiles
    (2, 64, 64, 128, 128, 3, 3, 1, 1, 1, False),       # K = 32768 pixels: the pixel reduction is split across CTAs
]


@pytest.mark.parametrize("case", CONV_CASES + EXTRA_CASES, ids=[f"c{i}" for i in range(len(CONV_CASES))] + [f"x{i}" for i in range(len(EXTRA_CASES))])
def test_conv2d_first_backward(case):
    from vtoonify_b200.op import conv2d_gradfix
    B, Cin, Cout, H, W, kh, kw, s, p, d, has_bias = case
    x = _rand((B, Cin, H, W), 1)
    w = _rand((Cout, Cin, kh, kw), 2, 1 / math.sqrt(Cin * kh * kw))
    b = _rand((Cout,), 3, 0.1) if has_bias else None
    _check_first_backward(lambda x_, w_, b_=None: conv2d_gradfix.conv2d(x_, w_, b_, stride=s, padding=p, dilation=d),
                          lambda x_, w_, b_=None: F.conv2d(x_, w_, b_, stride=s, padding=p, dilation=d),
                          [x, w, b], f"conv2d {case}")


@pytest.mark.parametrize("G,Cin,Cout,k,stride,pad", [(2, 32, 64, 3, 1, 1), (3, 64, 3, 1, 1, 0), (4, 32, 32, 3, 2, 0), (3, 64, 64, 3, 1, 1)])
def test_conv2d_groups_is_batch_backward(G, Cin, Cout, k, stride, pad):
    """the per-sample form of ModulatedConv2d (model.py:291-301): input [1, G*Cin, H, W], weight [G*Cout, Cin, k, k]"""
    from vtoonify_b200.op import conv2d_gradfix
    H, W = 13, 18
    x = _rand((1, G * Cin, H, W), 4)
    w = _rand((G * Cout, Cin, k, k), 5, 1 / math.sqrt(Cin * k * k))
    _check_first_backward(lambda x_, w_: conv2d_gradfix.conv2d(x_, w_, padding=pad, stride=stride, groups=G),
                          lambda x_, w_: F.conv2d(x_, w_, padding=pad, stride=stride, groups=G),
                          [x, w], f"conv2d groups={G} {Cin}->{Cout} k{k} s{stride}")


@pytest.mark.parametrize("G,Cin,Cout", [(1, 64, 32), (3, 32, 64), (2, 64, 48)])
def test_conv_transpose2d_backward(G, Cin, Cout):
    from vtoonify_b200.op import conv2d_gradfix
    H, W = 9, 12
    x = _rand((1, G * Cin, H, W), 6)
    w = _rand((G * Cin, Cout, 3, 3), 7, 1 / math.sqrt(Cin * 9))
    b = _rand((G * Cout,), 8, 0.1) if G == 1 else None
    ins = [x, w] + ([b] if b is not None else [])
    _check_first_backward(lambda x_, w_, b_=None: conv2d_gradfix.conv_transpose2d(x_, w_, b_, padding=0, stride=2, groups=G),
                          lambda x_, w_, b_=None: F.conv_transpose2d(x_, w_, b_, padding=0, stride=2, groups=G),
                          ins, f"conv_transpose2d groups={G} {Cin}->{Cout}")


@pytest.mark.parametrize("kind", ["s1p1", "s2p0", "transpose"])
def test_double_backward(kind):
    """d/d(x, w, u) of <grad_x, v> and of <grad_w, V>, where grad_x, grad_w are the gradients of <conv(x, w), u> taken with
    create_graph=True (the second derivatives R1-style penalties need)"""
    from vtoonify_b200.op import conv2d_gradfix
    if kind == "transpose":
        x, w = _rand((1, 32, 7, 9), 10), _rand((32, 64, 3, 3), 11, 1 / math.sqrt(32 * 9))
        ops_ = (lambda x_, w_: conv2d_gradfix.conv_transpose2d(x_, w_, stride=2, padding=0),
                lambda x_, w_: F.conv_transpose2d(x_, w_, stride=2, padding=0))
    else:
        s, p = (1, 1) if kind == "s1p1" else (2, 0)
        x, w = _rand((2, 32, 15, 13), 10), _rand((64, 32, 3, 3), 11, 1 / math.sqrt(32 * 9))
        ops_ = (lambda x_, w_: conv2d_gradfix.conv2d(x_, w_, stride=s, padding=p),
                lambda x_, w_: F.conv2d(x_, w_, stride=s, padding=p))
    results = []
    with torch.enable_grad():
        for fn, dev, dt in ((ops_[0], "cuda", torch.float32), (ops_[1], "cpu", torch.float64)):
            xl = x.to(dev, dt).requires_grad_(True)
            wl = w.to(dev, dt).requires_grad_(True)
            y = fn(xl, wl)
            ul = _rand(tuple(y.shape), 12).to(dev, dt).requires_grad_(True)
            gx, gw = torch.autograd.grad((y * ul).sum(), [xl, wl], create_graph=True)
            v, V = _rand(tuple(gx.shape), 13).to(dev, dt), _rand(tuple(gw.shape), 14).to(dev, dt)
            r = torch.autograd.grad((gx * v).sum(), [xl, wl, ul], allow_unused=True, retain_graph=True)
            r2 = torch.autograd.grad((gw * V).sum(), [xl, wl, ul], allow_unused=True)
            results.append([torch.zeros_like(t) if g is None else g for g, t in zip(r + r2, [xl, wl, ul] * 2)])
    for name, a, b in zip(["d<gx,v>/dx", "d<gx,v>/dw", "d<gx,v>/du", "d<gw,V>/dx", "d<gw,V>/dw", "d<gw,V>/du"], *results):
        if b.abs().max().item() == 0:
            assert a.abs().max().item() == 0, f"{kind} {name}: expected zero"
        else:
            _close(a, b, f"{kind} {name}")


def _discriminator(conv2d, upfirdn2d, flrelu, x, P, K):
    """Two blocks of the reference Discriminator (model/stylegan/model.py): ConvLayer(3, C, 1), then ResBlock(C, 2C):
    conv1 3x3, conv2 = Blur(pad (2, 2)) + EqualConv2d 3x3 stride 2 padding 0, skip = Blur(pad (1, 1)) + 1x1 stride 2 without
    bias or activation; EqualConv2d scales its weight by 1/sqrt(fan_in), FusedLeakyReLU carries the bias."""
    def eq(w):
        return w * (1 / math.sqrt(w.shape[1] * w.shape[2] * w.shape[3]))
    h = flrelu(conv2d(x, eq(P["w0"]), None, stride=1, padding=0), P["b0"])
    o = flrelu(conv2d(h, eq(P["w1"]), None, stride=1, padding=1), P["b1"])
    o = flrelu(conv2d(upfirdn2d(o, K, pad=(2, 2)), eq(P["w2"]), None, stride=2, padding=0), P["b2"])
    sk = conv2d(upfirdn2d(h, K, pad=(1, 1)), eq(P["w3"]), None, stride=2, padding=0)
    return (o + sk) / math.sqrt(2)


def test_r1_penalty_pattern():
    """util.py:75-80: grad of D(x).sum() w.r.t. x with create_graph=True inside no_weight_gradients(), then backward of the
    squared gradient norm: the discriminator weights' gradients go through the double backward of every convolution."""
    from oracle import vt_oracle as O
    from vtoonify_b200.op import conv2d_gradfix, fused_leaky_relu, upfirdn2d
    C = 32
    shapes = {"w0": (C, 3, 1, 1), "b0": (C,), "w1": (C, C, 3, 3), "b1": (C,), "w2": (2 * C, C, 3, 3), "b2": (2 * C,), "w3": (2 * C, C, 1, 1)}
    P0 = {k: _rand(s, 20 + i, 0.1 if k[0] == "b" else 1.0) for i, (k, s) in enumerate(shapes.items())}
    x0 = _rand((2, 3, 16, 16), 30)
    K = O.make_kernel([1, 3, 3, 1])
    grads = []
    with torch.enable_grad():
        for dev, dt in (("cuda", torch.float32), ("cpu", torch.float64)):
            P = {k: v.to(dev, dt).requires_grad_(True) for k, v in P0.items()}
            x = x0.to(dev, dt).requires_grad_(True)
            if dev == "cuda":
                with conv2d_gradfix.no_weight_gradients():
                    out = _discriminator(conv2d_gradfix.conv2d, upfirdn2d, fused_leaky_relu, x, P, K.cuda())
                    gx, = torch.autograd.grad(out.sum(), x, create_graph=True)
            else:
                out = _discriminator(F.conv2d, O.upfirdn2d, O.fused_leaky_relu, x, P, K.double())
                gx, = torch.autograd.grad(out.sum(), x, create_graph=True)
            penalty = gx.pow(2).reshape(gx.shape[0], -1).sum(1).mean()
            penalty.backward()
            grads.append({k: v.grad for k, v in P.items()})
    for k in shapes:
        _close(grads[0][k], grads[1][k], f"R1 penalty d/d{k}")


def test_no_weight_gradients():
    from vtoonify_b200.op import conv2d_gradfix
    x0, w0 = _rand((2, 32, 12, 11), 40), _rand((64, 32, 3, 3), 41, 1 / math.sqrt(32 * 9))
    u = _rand((2, 64, 12, 11), 42)
    with torch.enable_grad():
        x, w = x0.cuda().requires_grad_(True), w0.cuda().requires_grad_(True)
        with conv2d_gradfix.no_weight_gradients():
            (conv2d_gradfix.conv2d(x, w, padding=1) * u.cuda()).sum().backward()
        assert w.grad is None
        xc, wc = x0.double().requires_grad_(True), w0.double().requires_grad_(True)
        (F.conv2d(xc, wc, padding=1) * u.double()).sum().backward()
    _close(x.grad, xc.grad, "x.grad inside no_weight_gradients()")
    assert not conv2d_gradfix.weight_gradients_disabled


def test_conv_contributes_to_input_gradient():
    """the convolution's share of x.grad is not dropped when x also reaches the loss another way"""
    from vtoonify_b200.op import conv2d_gradfix
    x0, w0 = _rand((1, 32, 10, 10), 50), _rand((32, 32, 3, 3), 51, 1 / math.sqrt(32 * 9))
    u = _rand((1, 32, 10, 10), 52)
    with torch.enable_grad():
        x = x0.cuda().requires_grad_(True)
        y = conv2d_gradfix.conv2d(x, w0.cuda(), padding=1)
        assert y.requires_grad
        ((y * u.cuda()).sum() + x.sum()).backward()
        xc = x0.double().requires_grad_(True)
        ((F.conv2d(xc, w0.double(), padding=1) * u.double()).sum() + xc.sum()).backward()
    _close(x.grad, xc.grad, "x.grad with a second path")


@pytest.mark.parametrize("form", ["plain", "stride2", "groups", "transpose"])
def test_forward_bit_identical_under_autograd(form):
    from vtoonify_b200.op import conv2d_gradfix
    if form == "transpose":
        x, w = _rand((1, 3 * 32, 9, 10), 60).cuda(), _rand((3 * 32, 64, 3, 3), 61).cuda()
        fn = lambda x_, w_: conv2d_gradfix.conv_transpose2d(x_, w_, stride=2, padding=0, groups=3)   # noqa: E731
    elif form == "groups":
        x, w = _rand((1, 2 * 64, 13, 12), 60).cuda(), _rand((2 * 32, 64, 3, 3), 61).cuda()
        fn = lambda x_, w_: conv2d_gradfix.conv2d(x_, w_, padding=1, groups=2)   # noqa: E731
    else:
        s = 2 if form == "stride2" else 1
        x, w = _rand((2, 64, 17, 16), 60).cuda(), _rand((48, 64, 3, 3), 61).cuda()
        fn = lambda x_, w_: conv2d_gradfix.conv2d(x_, w_, stride=s, padding=1)   # noqa: E731
    with torch.no_grad():
        y0 = fn(x, w)
    with torch.enable_grad():
        y1 = fn(x.clone().requires_grad_(True), w.clone().requires_grad_(True))
    assert y1.requires_grad
    assert torch.equal(y0, y1.detach())


@pytest.mark.parametrize("shape", [(2, 64, 64, 128, 128, 3), (2, 64, 32, 17, 20, 3), (1, 96, 160, 12, 12, 1)])
def test_gradients_are_reproducible(shape):
    from vtoonify_b200.op import conv2d_gradfix
    B, Cin, Cout, H, W, k = shape
    x0, w0 = _rand((B, Cin, H, W), 70).cuda(), _rand((Cout, Cin, k, k), 71).cuda()
    b0, u = _rand((Cout,), 72).cuda(), _rand((B, Cout, H, W), 73).cuda()
    runs = []
    with torch.enable_grad():
        for _ in range(2):
            x, w, b = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
            (conv2d_gradfix.conv2d(x, w, b, padding=k // 2) * u).sum().backward()
            runs.append((x.grad, w.grad, b.grad))
    for a, b in zip(*runs):
        assert torch.equal(a, b)
