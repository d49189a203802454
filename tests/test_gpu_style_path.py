"""GPU: the style path's small dense kernels of csrc/modulate.cu against float64: ``ops.linear`` (vt_linear_f32: every
EqualLinear, the mapping networks, the pSp / BiSeNet / discriminator heads), ``ops.pixelnorm`` (vt_pixelnorm_f32), the
``PixelNorm`` module at rank 2, 3 and 4, and the mapping networks ``Generator.style`` / ``get_latent`` / ``mean_latent`` and
``DualStyleGAN.style`` from a deterministic state_dict.

Bars (u = 2^-24), derived from the kernels' summation order:
  linear     lane i of the output's warp sums m = ceil(in_dim / 32) products x * fl(w * w_scale) serially, then 5 butterfly
             levels: |err(z)| <= (m + 7) u S + 2u |b|, S = sum |x w w_scale| (one u for fl(w * w_scale), one per product or
             fused add, one per tree level), with b = fl(bias * b_scale) and one more u for z + b.  The activation multiplies
             this by its Lipschitz constant (sqrt 2, 1, 1, 1/4) and adds its own roundings: 3u |out| for fused_lrelu (slope,
             the fp32 sqrt 2 and its product), u |out| for LeakyReLU, 4u |out| for the sigmoid (expf is within 2 ulp, then an
             add and a divide).
  pixelnorm  the sum of squares of m = ceil(dim / 32) terms per lane and 5 levels is off by <= (m + 5)u relatively, the mean and
             + 1e-8 add 2u, the sqrt halves all of it and adds u, 1/x and the product add 2u: |err| <= ((m + 7)/2 + 3) u |ref|.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

U = 2.0 ** -24
SQRT2 = math.sqrt(2.0)
LIP = {0: 1.0, 1: SQRT2, 2: 1.0, 3: 1.0, 4: 0.25}       # Lipschitz constant of each activation
OWN = {0: 0.0, 1: 3.0, 2: 1.0, 3: 0.0, 4: 4.0}          # the activation's own roundings (and fp32 sqrt 2), in u of |out|


def f32(v: float) -> float:
    return float(torch.tensor(v, dtype=torch.float32))


def act64(z, act):
    if act == 1:
        return torch.where(z > 0, z, 0.2 * z) * SQRT2
    if act == 2:
        return torch.where(z > 0, z, 0.2 * z)
    if act == 3:
        return z.clamp_min(0)
    if act == 4:
        return torch.sigmoid(z)
    return z


def linear64(x, w, b, w_scale, b_scale, act):
    """float64 of the kernel's operation on its fp32 inputs (scales rounded to fp32, as the kernel receives them); returns
    (out, bound on |err|) with the bound of the module docstring"""
    xd, wd = x.double().reshape(-1, x.shape[-1]), w.double()
    ws, bs = f32(w_scale), f32(b_scale)
    z = xd @ (wd * ws).t()
    S = xd.abs() @ (wd.abs() * ws).t()
    bb = torch.zeros(w.shape[0], dtype=torch.float64, device=x.device) if b is None else b.double() * bs
    z = z + bb
    out = act64(z, act)
    m = math.ceil(x.shape[-1] / 32)
    bar = LIP[act] * ((m + 7) * U * S + 2 * U * bb.abs()) + OWN[act] * U * out.abs()
    return out.reshape(*x.shape[:-1], w.shape[0]), bar.reshape(*x.shape[:-1], w.shape[0])


def check(got, ref, bar, what):
    err = (got.double() - ref).abs()
    ratio = (err / bar.clamp_min(1e-300)).max().item()
    print(f"{what}: max err {err.max().item():.2e}, max err/bar {ratio:.3f}")
    assert (err <= bar).all(), f"{what}: {ratio:.2f} x the bar"
    return ratio


# ---- linear --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_dim", [1, 3, 512])
@pytest.mark.parametrize("in_dim", [1, 31, 32, 33, 512, 8192])
@pytest.mark.parametrize("rows", [1, 2, 37, 144])
def test_linear_shapes_vs_float64(rows, in_dim, out_dim):
    """every (rows, in_dim, out_dim) of the grid with a bias and fused_lrelu; in_dim 8192 is the discriminator head's"""
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(rows * 10007 + in_dim * 13 + out_dim)
    x = torch.randn((rows, in_dim), generator=g).cuda()
    w = torch.randn((out_dim, in_dim), generator=g).cuda()
    b = torch.randn(out_dim, generator=g).cuda()
    ws = 1 / math.sqrt(in_dim)
    got = ops.linear(x, w, b, ws, 1.0, 1)
    ref, bar = linear64(x, w, b, ws, 1.0, 1)
    check(got, ref, bar, f"linear {rows}x{in_dim}->{out_dim}")


@pytest.mark.parametrize("act", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["equal", "mapping", "nobias", "rank3"])
def test_linear_params_vs_float64(kind, act):
    """EqualLinear's scales (w_scale = lr_mul / sqrt(in), b_scale = lr_mul), the mapping network's lr_mul = 0.01 with weights
    ~N(0,1)/0.01, no bias, and a rank-3 [B, L, in] input, under every activation"""
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(act * 31 + len(kind))
    lr_mul = 0.01 if kind == "mapping" else 1.0
    shape = (3, 18, 512) if kind == "rank3" else (37, 512)
    x = torch.randn(shape, generator=g).cuda()
    w = (torch.randn((512, 512), generator=g) / lr_mul).cuda()
    b = None if kind == "nobias" else (torch.randn(512, generator=g) * 0.5).cuda()
    ws, bs = lr_mul / math.sqrt(512), lr_mul
    got = ops.linear(x, w, b, ws, bs, act)
    assert tuple(got.shape) == shape[:-1] + (512,)
    ref, bar = linear64(x, w, b, ws, bs, act)
    check(got, ref, bar, f"linear {kind} act {act}")


# ---- pixelnorm -----------------------------------------------------------------------------------------------------------------
def pixelnorm_rows(dim, seed):
    """rows: unit, offset ~1e3, tiny ~1e-6 (mean of squares ~1e-12: the 1e-8 epsilon dominates), all zero, one-hot"""
    g = torch.Generator().manual_seed(seed)
    r = torch.randn((5, dim), generator=g)
    r[1] = 1e3 + r[1]
    r[2] = 1e-6 * r[2]
    r[3] = 0.0
    r[4] = 0.0
    r[4, dim // 2] = -3.0
    return r


def pixelnorm64(x, dim=-1):
    xd = x.double()
    return xd / torch.sqrt(xd.pow(2).mean(dim=dim, keepdim=True) + 1e-8)


@pytest.mark.parametrize("dim", [1, 7, 32, 512, 513, 4096])
def test_pixelnorm_vs_float64(dim):
    from vtoonify_b200 import ops
    x = pixelnorm_rows(dim, seed=dim).cuda()
    got = ops.pixelnorm(x)
    ref = pixelnorm64(x)
    bar = ((math.ceil(dim / 32) + 7) / 2 + 3) * U * ref.abs()
    check(got, ref, bar, f"pixelnorm dim {dim}")
    assert torch.equal(got[3], torch.zeros_like(got[3])), "an all-zero row must stay exactly zero"


@pytest.mark.parametrize("shape", [(3, 18, 512), (2, 512, 5, 7), (4, 512)])
def test_pixelnorm_module_normalises_dim1(shape):
    """PixelNorm (model/stylegan/model.py:13-18) takes mean(input ** 2, dim=1) whatever the rank"""
    from vtoonify_b200.stylegan import PixelNorm
    g = torch.Generator().manual_seed(len(shape))
    x = (torch.randn(shape, generator=g) + 0.5).cuda()
    got = PixelNorm()(x)
    assert tuple(got.shape) == shape
    ref = pixelnorm64(x, dim=1)
    bar = ((math.ceil(shape[1] / 32) + 7) / 2 + 3) * U * ref.abs()
    check(got, ref, bar, f"PixelNorm {shape}")


# ---- the mapping networks --------------------------------------------------------------------------------------------------------
def mapping64(seq, z):
    """float64 restatement of PixelNorm + EqualLinear(fused_lrelu) layers, from the module's own parameters; returns (out, bound
    on |err| per row in the 2-norm).  Each layer's own error (linear64's bar, 2-norm per row) is carried through the later
    layers by their Lipschitz constants sqrt 2 * ||scale W||_2 (fused_lrelu's slope is at most sqrt 2): a first-order bound
    of the whole chain against float64.  It is loose (the product of 8 Lipschitz constants); check_layers holds each layer to
    its own tight bar."""
    from vtoonify_b200.stylegan import EqualLinear, PixelNorm
    h = pixelnorm64(z)
    m = math.ceil(z.shape[-1] / 32)
    bound = (((m + 7) / 2 + 3) * U * h.abs()).norm(dim=-1)
    for layer in seq:
        if isinstance(layer, PixelNorm):
            continue
        assert isinstance(layer, EqualLinear) and layer.activation
        L = SQRT2 * torch.linalg.matrix_norm(layer.weight.double() * f32(layer.scale), ord=2).item()
        h_new, bar = linear64(h, layer.weight, layer.bias, layer.scale, layer.lr_mul, 1)
        bound = L * bound + bar.norm(dim=-1)
        h = h_new
    return h, bound


def check_layers(seq, z, what):
    """runs the mapping network layer by layer, checking each layer against float64 of its own fp32 input with the tight bars of
    the module docstring; returns the fp32 output"""
    from vtoonify_b200.stylegan import PixelNorm
    h = z
    for i, layer in enumerate(seq):
        out = layer(h)
        if isinstance(layer, PixelNorm):
            ref = pixelnorm64(h)
            bar = ((math.ceil(h.shape[-1] / 32) + 7) / 2 + 3) * U * ref.abs()
        else:
            ref, bar = linear64(h, layer.weight, layer.bias, layer.scale, layer.lr_mul, 1)
        check(out, ref, bar, f"{what} layer {i}")
        h = out
    return h


def check_mapping(got, ref, bound, what):
    err = (got.double() - ref)
    rel_l2 = (err.norm() / ref.norm()).item()
    row = err.norm(dim=-1)
    print(f"{what}: rel L2 err {rel_l2:.2e}, max err {err.abs().max().item():.2e}, "
          f"max row err/bound {(row / bound).max().item():.3f} (bound rel {(bound / ref.norm(dim=-1)).max().item():.2e})")
    assert (row <= bound).all(), "2-norm of a row's error above its bound"
    assert (err.abs().max(dim=-1).values <= bound).all()


def det_generator():
    from vtoonify_b200.stylegan import Generator
    from vtoonify_b200.weights import det_state_dict
    G = Generator(16, 512, 8)
    G.load_state_dict(det_state_dict(G, seed=2))
    return G.cuda().eval()


def test_generator_mapping_network_vs_float64():
    """Generator.style (PixelNorm + 8 EqualLinear(lr_mul 0.01)), get_latent and mean_latent"""
    G = det_generator()
    g = torch.Generator().manual_seed(17)
    z = torch.randn((37, 512), generator=g).cuda()
    ref, bound = mapping64(G.style, z)
    assert torch.equal(check_layers(G.style, z, "Generator.style"), G.style(z))
    check_mapping(G.style(z), ref, bound, "Generator.style")
    assert torch.equal(G.get_latent(z), G.style(z))
    torch.manual_seed(123)
    ml = G.mean_latent(1024)
    torch.manual_seed(123)
    zz = torch.randn(1024, 512, device="cuda")
    ref, bound = mapping64(G.style, zz)
    # the mean of 1024 rows, each within its bound: |mean err| <= mean of the row bounds, plus torch's fp32 mean over 1024 rows
    # (10 tree levels and the divide: 11u of mean |h| per element)
    bound_mean = bound.mean() + 11 * U * ref.abs().mean(0).norm()
    check_mapping(ml, ref.mean(0, keepdim=True), bound_mean.reshape(1), "Generator.mean_latent")


def test_dualstylegan_style_vs_float64():
    """DualStyleGAN.style: PixelNorm + 2 EqualLinear(lr_mul 0.01), on a [B, 18, 512] code reshaped as DualStyleGAN does"""
    from vtoonify_b200.dualstylegan import DualStyleGAN
    from vtoonify_b200.weights import det_state_dict
    D = DualStyleGAN(16, 512, 8)
    D.load_state_dict(det_state_dict(D, seed=4))
    D = D.cuda().eval()
    g = torch.Generator().manual_seed(19)
    s = torch.randn((2, 18, 512), generator=g).cuda()
    got = D.style(s.reshape(-1, 512)).reshape(s.shape)
    assert torch.equal(check_layers(D.style, s.reshape(-1, 512), "DualStyleGAN.style").reshape(s.shape), got)
    ref, bound = mapping64(D.style, s.reshape(-1, 512))
    check_mapping(got.reshape(-1, 512), ref, bound, "DualStyleGAN.style")
