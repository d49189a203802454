"""GPU: the G-step kernels (ops.torgb_gate_grad, fusion_mask_grad, fusion_adain_grad_stats, fusion_input_grad) against float64, with
bars derived from their summation order: every fp32 rounding step contributes at most u = 2^-24 of the magnitudes it combines, so each
bar is a small multiple of u times the float64 sum of absolute terms (computed alongside the reference).  Offset and near-constant
planes exercise the AdaIN sums, and f_G == f_E pixels the sign(0) = 0 split."""
import pytest
import torch
import torch.nn.functional as F

from tests.oracle_vtoonify_gstep import mask_head_backward

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2)


def within(got, ref, bound, name):
    err = (got.double() - ref).abs()
    worst = (err / bound.clamp_min(1e-300)).max().item()
    print(f"  {name}: max err / bar {worst:.3f}")
    assert bool((err <= bound).all()), f"{name}: max err / bar {worst:.3f}"


@pytest.mark.parametrize("wB,with_g", [(1, True), (2, True), (2, False)])
def test_torgb_gate_grad(wB, with_g):
    from vtoonify_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(11)
    B, C, H, W = 2, 96, 9, 13
    g = torch.randn(B, H, W, C, device="cuda", generator=gen) if with_g else None
    g_rgb = torch.randn(B, 3, H, W, device="cuda", generator=gen)
    w = torch.randn(wB, 1, 3, C + 32, device="cuda", generator=gen)
    ref = torch.randn(B, H, W, C, device="cuda", generator=gen)
    out = ops.torgb_gate_grad(g, g_rgb, w, ref, 0.2, 2 ** 0.5)
    w64 = w.double()[:, 0, :, :C].expand(B, 3, C)
    t = torch.einsum("bkc,bkhw->bhwc", w64, g_rgb.double())
    tabs = torch.einsum("bkc,bkhw->bhwc", w64.abs(), g_rgb.double().abs())
    if g is not None:
        t, tabs = t + g.double(), tabs + g.double().abs()
    gate = torch.where(ref > 0, 1.0, 0.2).double() * 2 ** 0.5
    within(out, gate * t, 6 * U * gate * tabs, "torgb_gate_grad")


def _mask_inputs(B, C, H, W, offset=0.0, spread=1.0, equal=False, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(100 + seed)
    f_g = offset + spread * torch.randn(B, C, H, W, device="cuda", generator=gen)
    f_e = offset + spread * torch.randn(B, C, H, W, device="cuda", generator=gen)
    if equal:
        f_e[:, :, ::2, ::3] = f_g[:, :, ::2, ::3]
    m = torch.tanh(torch.relu(torch.randn(B, 1, H, W, device="cuda", generator=gen)))
    g_p = torch.randn(B, C, H, W, device="cuda", generator=gen)
    g_m = torch.randn(B, 1, H, W, device="cuda", generator=gen)
    w2 = 0.05 * torch.randn(1, 2 * C, 3, 3, device="cuda", generator=gen)
    gb = torch.cat([1 + 0.3 * torch.randn(B, 2 * C, device="cuda", generator=gen), 0.3 * torch.randn(B, 2 * C, device="cuda", generator=gen)], 1)
    g_dir = torch.randn(B, C, H, W, device="cuda", generator=gen)
    a = torch.cat([f_g, (f_g - f_e).abs()], 1).double()
    stats = torch.stack([a.mean((2, 3)), torch.rsqrt(a.var((2, 3), unbiased=False) + 1e-5)], -1).float()
    return f_g, f_e, m, g_p, g_m, w2, gb, g_dir, stats


GEOMS = [(2, 64, 12, 10, 0.0, 1.0, False), (1, 128, 33, 7, 0.0, 1.0, True), (2, 32, 16, 16, 100.0, 1e-3, False),
         (1, 512, 8, 6, 0.0, 1.0, True), (2, 64, 9, 11, 5.0, 1e-6, True)]


@pytest.mark.parametrize("B,C,H,W,offset,spread,equal", GEOMS)
def test_fusion_mask_head_kernels(B, C, H, W, offset, spread, equal):
    from vtoonify_b200 import ops
    f_g, f_e, m, g_p, g_m, w2, gb, g_dir, stats = _mask_inputs(B, C, H, W, offset, spread, equal)
    d = lambda t: t.double()   # noqa: E731
    g_z_ref, db_ref = mask_head_backward(d(g_p), d(f_g), d(f_e), d(m), d(g_m), d(w2), d(stats), d(gb))[:2]
    w2t = w2.reshape(2 * C, 9).t().contiguous()
    # 1. g_z: the channel dot product in double, then three fp32 steps
    g_z, db = ops.fusion_mask_grad(nhwc(g_p), nhwc(f_e), m, g_m)
    sabs = (d(g_p) * d(f_e)).abs().sum(1, keepdim=True) + d(g_m).abs()
    mfac = (1 - d(m) ** 2) * (d(m) > 0)
    # 1 - m^2 in fp32 loses u * m^2 absolutely, a large relative error where m is close to 1
    zbar = 6 * U * sabs * (mfac + d(m) ** 2 * (d(m) > 0))
    within(g_z, g_z_ref, zbar + 1e-30, "g_z")
    within(db, db_ref, zbar.sum().reshape(1) + 1e-30, "conv2 bias grad")
    # 2. the AdaIN sums, against float64 sums built from the kernel's own g_z: u is a 9-term fp32 sum, ahat two fp32 steps, the sums
    # in double
    sums = ops.fusion_adain_grad_stats(g_z, w2t, nhwc(f_g), nhwc(f_e), stats)
    g_z_ref = d(g_z)
    u = F.conv_transpose2d(g_z_ref, d(w2), padding=1)
    uabs = F.conv_transpose2d(g_z_ref.abs(), d(w2).abs(), padding=1)
    a = torch.cat([d(f_g), (d(f_g) - d(f_e)).abs()], 1)
    mean, rstd = d(stats)[..., 0, None, None], d(stats)[..., 1, None, None]
    ahat = (a - mean) * rstd
    ahat_abs = ((a - mean).abs() + a.abs() * U) * rstd
    sums_ref = torch.stack([u.sum((2, 3)), (u * ahat).sum((2, 3))], -1)
    bar = torch.stack([(12 * U * uabs).sum((2, 3)), (12 * U * uabs * (ahat_abs + 1)).sum((2, 3))], -1)
    within(sums, sums_ref, bar + 1e-30, "AdaIN sums")
    # 3. the elementwise pass, from the kernel's own sums
    g_fg, g_fe = ops.fusion_input_grad(g_z, w2t, nhwc(f_g), nhwc(f_e), stats, gb, sums, nhwc(g_dir), nhwc(g_p), m)
    hw = H * W
    s64 = d(sums)
    coef = (d(gb)[:, :2 * C, None, None] * rstd).abs()
    t = d(gb)[:, :2 * C, None, None] * rstd * ((u - s64[..., 0, None, None] / hw) - ahat * s64[..., 1, None, None] / hw)
    sg = torch.sign(d(f_g) - d(f_e))
    tabs = coef * (uabs + (s64[..., 0, None, None] / hw).abs() + ahat_abs * (s64[..., 1, None, None] / hw).abs())
    within(g_fg, nhwc(t[:, :C] + sg * t[:, C:] + d(g_dir)),
           nhwc(12 * U * (tabs[:, :C] + tabs[:, C:] + d(g_dir).abs())) + 1e-30, "g_fG")
    within(g_fe, nhwc(d(g_p) * d(m) - sg * t[:, C:]), nhwc(12 * U * (tabs[:, C:] + (d(g_p) * d(m)).abs())) + 1e-30, "g_fE")
    if equal:   # sign(0) = 0: where f_G == f_E the |.| half sends nothing, g_fE is exactly g_p * m
        z = (f_g == f_e)
        assert bool(z.any())
        assert torch.equal(nchw(g_fe)[z], (g_p * m).expand_as(g_p)[z])


def test_mask_head_kernels_are_deterministic():
    from vtoonify_b200 import ops
    f_g, f_e, m, g_p, g_m, w2, gb, g_dir, stats = _mask_inputs(2, 128, 40, 36)
    w2t = w2.reshape(256, 9).t().contiguous()
    outs = []
    for _ in range(2):
        g_z, db = ops.fusion_mask_grad(nhwc(g_p), nhwc(f_e), m, g_m)
        sums = ops.fusion_adain_grad_stats(g_z, w2t, nhwc(f_g), nhwc(f_e), stats)
        outs.append((g_z, db, sums) + ops.fusion_input_grad(g_z, w2t, nhwc(f_g), nhwc(f_e), stats, gb, sums, None, nhwc(g_p), m))
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_channel_sum_nhwc():
    """The fusion convolutions' bias gradient: a per-channel sum with double partials, one rounding at the end."""
    from vtoonify_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(5)
    g = torch.randn(3, 37, 29, 64, device="cuda", generator=gen) + 10.0
    s = ops.channel_sum_nhwc(g)
    within(s, g.double().sum((0, 1, 2)), 2 * U * g.double().abs().sum((0, 1, 2)), "channel_sum_nhwc")
    assert torch.equal(s, ops.channel_sum_nhwc(g))
