"""GPU: the LPIPS kernels against torch and float64.  The 2x2 max-pool and its adjoint must be bit-identical to torch's (ties included:
equal values and all-zero windows, whose gradient goes to the first element in row-major order).  The head forms its per-pixel sums in
double from fp32 inputs and rounds once at the end, so its bars are a few u = 2^-24 times the float64 sum of the absolute terms (for the
forward, the loss itself: every term is non-negative).  Pixels with ||f|| = 0 and near-parallel f0, f1 are included."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
EPS = 1e-10


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2)


def within(got, ref, bound, name):
    err = (got.double() - ref).abs()
    worst = (err / bound.clamp_min(1e-300)).max().item()
    print(f"  {name}: max err / bar {worst:.3f}")
    assert bool((err <= bound).all()), f"{name}: max err / bar {worst:.3f}"


@pytest.mark.parametrize("shape", [(2, 64, 16, 16), (1, 128, 9, 11), (3, 256, 7, 6), (1, 512, 3, 2)])
def test_maxpool2x2_matches_torch_bit_for_bit(shape):
    from vtoonify_b200 import ops
    x = torch.randn(shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    got = nchw(ops.maxpool2x2(nhwc(x)))
    want = F.max_pool2d(x, 2, 2)
    assert got.shape == want.shape and torch.equal(got, want)


@pytest.mark.parametrize("shape,with_add", [((2, 64, 16, 16), False), ((1, 64, 9, 11), True), ((2, 128, 7, 6), True), ((1, 32, 5, 5), False)])
def test_maxpool2x2_grad_matches_torch_with_ties(shape, with_add):
    from vtoonify_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(2)
    # values in {0, 1, 2} make most windows tie, and relu(.) - 1 clamps a third of them to exact zeros (all-zero windows included)
    x = torch.relu(torch.randint(0, 3, shape, device="cuda", generator=gen).float() - 1.0)
    x[:, :, :4, :4] = 0.0
    B, C, H, W = shape
    g = torch.randn(B, C, H // 2, W // 2, device="cuda", generator=gen)
    add = torch.randn(shape, device="cuda", generator=gen) if with_add else None
    xr = x.clone().requires_grad_()
    with torch.enable_grad():
        F.max_pool2d(xr, 2, 2).backward(g)
    want = xr.grad if add is None else xr.grad + add
    got = nchw(ops.maxpool2x2_grad(nhwc(g), nhwc(x), None if add is None else nhwc(add)))
    assert torch.equal(got, want)


def _taps(B, shapes, seed):
    """taps [2B, h, w, C] with all-zero rows, near-parallel f0 / f1 rows and equal rows, plus lin weights"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    taps, ws = [], []
    for h, w, C in shapes:
        f = torch.relu(torch.randn(2 * B, h, w, C, device="cuda", generator=gen))
        f[:B, 0, 0] = 0.0                                                   # ||f0|| = 0
        f[B:, 0, -1] = 0.0                                                  # ||f1|| = 0
        f[:, -1, 0] = 0.0                                                   # both
        f[B:, h // 2, w // 2] = f[:B, h // 2, w // 2] * (1 + 1e-6)         # near-parallel
        f[B:, h // 2, 0] = f[:B, h // 2, 0]                                # equal
        taps.append(f.contiguous())
        ws.append(0.1 * torch.rand(C, device="cuda", generator=gen))
    return taps, ws


def _norm64(f):
    n = f.double().pow(2).sum(-1, keepdim=True).sqrt()
    return n, f.double() / (n + EPS)


SHAPES = [(16, 12, 64), (8, 6, 128), (4, 3, 256), (2, 2, 512), (1, 2, 512)]


@pytest.mark.parametrize("B", [1, 3])
def test_head_forward_against_float64(B):
    from vtoonify_b200 import ops
    taps, ws = _taps(B, SHAPES, 3 + B)
    got = ops.lpips_head(taps, ws)
    want = torch.zeros(B, dtype=torch.float64, device="cuda")
    for f, w in zip(taps, ws):
        _, u = _norm64(f)
        want += ((u[:B] - u[B:]) ** 2 * w.double()).sum(-1).mean((1, 2))
    within(got, want, 4 * U * want + 1e-30, f"head forward B={B}")
    again = ops.lpips_head(taps, ws)
    assert torch.equal(got, again)


def _head_grad64(f, w, g_b):
    """the gradient of sum_b g_b[b] * mean_p sum_c w (u0 - u1)^2 as the kernel states it, with the absolute terms of its bar"""
    B = f.shape[0] // 2
    HW = f.shape[1] * f.shape[2]
    n, u = _norm64(f)
    a = n + EPS
    t = u[:B] - u[B:]
    w = w.double()
    s = (g_b.double() / HW).reshape(B, 1, 1, 1)
    out, absb = [], []
    for side, sign in ((slice(0, B), 1.0), (slice(B, 2 * B), -1.0)):
        fs, ns, as_ = f[side].double(), n[side], a[side]
        A = sign * 2 * w * t
        Af = (A * fs).sum(-1, keepdim=True)
        k = torch.where(ns > 0, Af / (ns * as_).clamp_min(1e-300), torch.zeros_like(ns))
        g = s / as_ * (A - fs * k)
        g = torch.where(ns > 0, g, torch.zeros_like(g))
        bar = (s.abs() / as_) * (A.abs() + fs.abs() * ((A.abs() * fs.abs()).sum(-1, keepdim=True) / (ns * as_).clamp_min(1e-300)))
        out.append(g)
        absb.append(bar)
    return torch.cat(out), torch.cat(absb)


@pytest.mark.parametrize("target,pred", [(True, True), (False, True), (True, False)])
def test_head_backward_against_float64(target, pred):
    from vtoonify_b200 import ops
    B = 2
    taps, ws = _taps(B, SHAPES[:3] + [(3, 5, 64)], 11)
    g_b = torch.tensor([0.7, -1.3], device="cuda")
    for f, w in zip(taps, ws):
        got = ops.lpips_head_grad(f, w, g_b, target, pred)
        want, bar = _head_grad64(f, w, g_b)
        sel = slice(0 if target else B, 2 * B if pred else B)
        within(got, want[sel], 8 * U * bar[sel] + 1e-30, f"head backward {tuple(f.shape)} target={target} pred={pred}")
        # n == 0 gives 0 (autograd would give NaN there)
        zero_rows = f[sel].double().pow(2).sum(-1) == 0
        assert bool((got[zero_rows] == 0).all())
        assert torch.equal(got, ops.lpips_head_grad(f, w, g_b, target, pred))


def test_head_backward_is_the_derivative_of_the_forward():
    """away from ||f|| = 0 the stated formula is the autograd derivative of the float64 forward"""
    from vtoonify_b200 import ops
    B = 2
    gen = torch.Generator(device="cuda").manual_seed(5)
    f = (torch.rand(2 * B, 5, 4, 64, device="cuda", generator=gen) + 0.1).contiguous()
    w = 0.1 * torch.rand(64, device="cuda", generator=gen)
    g_b = torch.tensor([0.9, 1.7], device="cuda")
    f64 = f.double().requires_grad_()
    with torch.enable_grad():
        n = f64.pow(2).sum(-1, keepdim=True).sqrt()
        u = f64 / (n + EPS)
        val = ((u[:B] - u[B:]) ** 2 * w.double()).sum(-1).mean((1, 2))
        (val * g_b.double()).sum().backward()
    got = ops.lpips_head_grad(f, w, g_b, True, True)
    err = ((got.double() - f64.grad).norm() / f64.grad.norm()).item()
    print(f"  head backward vs autograd: rel L2 {err:.2e}")
    assert err < 1e-6
