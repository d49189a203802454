"""CPU: pin the float64 G-step oracle (tests/oracle_vtoonify_gstep.py) to the unmodified reference (tests/golden/gstep_*.npz), and
check in float64 the adjoint identities the library's G-step backward is built on (vtoonify_b200/vtoonify_grad.py)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import vt_oracle as O
from tests.oracle_vtoonify_gstep import CASES, GEOMS, WSTEP, inputs, loss_and_grads, mask_head_backward


def T(a):
    return torch.from_numpy(a)


def rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def g64(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("case", list(CASES))
def test_gstep_oracle_golden(golden, case, geom):
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict
    g = golden(f"gstep_{case}_{geom}")
    backbone, d_s = CASES[case]
    sd = det_state_dict(VToonify(backbone=backbone), seed=0)
    x, style = inputs(geom)
    r = loss_and_grads(sd, x, style, d_s, backbone)
    # both sides are float64 with the same operation order up to library kernels
    assert abs(r["loss"].item() - float(g["loss"])) <= 1e-12 * float(g["loss"])
    checks = [("img", r["img"][:, :, ::4, ::4], T(g["img_sub"])), ("x.grad", r["x_grad"][:, :, ::4, ::4], T(g["x_grad_sub"]))]
    checks += [(f"mask{i}", m, T(g[f"mask{i}"])) for i, m in enumerate(r["masks"])]
    assert len(r["masks"]) == sum(1 for n in g.files if n.startswith("mask"))
    for k, gr in r["grads"].items():
        if gr.dim() == 1:
            checks.append((k, gr, T(g["g:" + k])))
        else:
            checks.append((k, gr.flatten()[::WSTEP], T(g["gs:" + k])))
            assert abs(gr.norm().item() - float(g["gn:" + k])) <= 1e-10 * float(g["gn:" + k]), k
    assert len(r["grads"]) == sum(1 for n in g.files if n.startswith(("g:", "gs:")))
    for name, got, ref in checks:
        assert got.shape == ref.shape, name
        if ref.norm() == 0:
            assert got.norm() == 0, name
            continue
        assert rel(got, ref) <= 1e-10, f"{case} {geom} {name}: relative L2 {rel(got, ref):.2e}"


def test_upconv_adjoint_is_blur_pad2_then_stride2_conv_with_transposed_weights():
    """<Blur(conv_transpose(x, w, s2)), g> = <x, conv2d(Blur'(g, pad (2, 2)), w^T, s2)> with the up-conv's 4x4 blur (x4) and pad (1, 1)."""
    B, Ci, Co, H, W = 2, 5, 4, 6, 7
    x = torch.randn(B, Ci, H, W, generator=g64(1), dtype=torch.float64)
    w = torch.randn(Co, Ci, 3, 3, generator=g64(2), dtype=torch.float64)          # [Cout, Cin, 3, 3] as the library's slabs
    k = O.make_kernel([1, 3, 3, 1]).double() * 4
    y = O.upfirdn2d(F.conv_transpose2d(x, w.transpose(0, 1), stride=2), k, pad=(1, 1))
    g = torch.randn(y.shape, generator=g64(3), dtype=torch.float64)
    gt = O.upfirdn2d(g, torch.flip(k, [0, 1]), pad=(2, 2))                        # [B, Co, 2H+1, 2W+1]
    assert gt.shape[2:] == (2 * H + 1, 2 * W + 1)
    gx = F.conv2d(gt, w.transpose(0, 1), stride=2)                                # taps (ky, kx) unflipped, in/out swapped
    assert gx.shape == x.shape
    assert abs((y * g).sum().item() - (x * gx).sum().item()) <= 1e-12 * (y * g).abs().sum().item()


def test_torgb_and_skip_adjoints():
    """ToRGB's 1x1 modulated conv transposed is w_rgb[b]^T g_rgb per pixel; the skip Upsample(up 2, pad (2, 1)) transposed is
    upfirdn2d(down 2, pad (1, 2)) with the flipped kernel."""
    B, C, H, W = 2, 6, 5, 4
    a = torch.randn(B, C, 2 * H, 2 * W, generator=g64(4), dtype=torch.float64)
    wr = torch.randn(B, 3, C, generator=g64(5), dtype=torch.float64)
    s = torch.randn(B, 3, H, W, generator=g64(6), dtype=torch.float64)
    k = O.make_kernel([1, 3, 3, 1]).double() * 4
    rgb = torch.einsum("bkc,bchw->bkhw", wr, a) + O.upfirdn2d(s, k, up=2, pad=(2, 1))
    g = torch.randn(rgb.shape, generator=g64(7), dtype=torch.float64)
    ga = torch.einsum("bkc,bkhw->bchw", wr, g)
    gs = O.upfirdn2d(g, torch.flip(k, [0, 1]), down=2, pad=(1, 2))
    assert gs.shape == s.shape
    lhs = (rgb * g).sum().item()
    assert abs(lhs - (a * ga).sum().item() - (s * gs).sum().item()) <= 1e-12 * (rgb * g).abs().sum().item()


@pytest.mark.parametrize("equal_pixels", [False, True])
def test_mask_head_derivative(equal_pixels):
    """The formulas of the mask-head kernels (g_z, the AdaIN sums over the virtual concat, the |.| split with sign(0) = 0 and g_p * m)
    against torch autograd through AdaIN(cat(f_G, |f_G - f_E|)) -> conv2 -> tanh(relu) -> f_E * m, in float64."""
    B, C, H, W = 2, 8, 7, 6
    f_g = torch.randn(B, C, H, W, generator=g64(8), dtype=torch.float64)
    f_e = torch.randn(B, C, H, W, generator=g64(9), dtype=torch.float64)
    if equal_pixels:
        f_e[:, :, ::2, ::3] = f_g[:, :, ::2, ::3]
    w2 = 0.3 * torch.randn(1, 2 * C, 3, 3, generator=g64(10), dtype=torch.float64)
    b2 = torch.tensor([0.1], dtype=torch.float64)
    gb = torch.randn(B, 4 * C, generator=g64(11), dtype=torch.float64) * 0.5 + torch.cat([torch.ones(2 * C), torch.zeros(2 * C)])
    g_p = torch.randn(B, C, H, W, generator=g64(12), dtype=torch.float64)
    g_m = torch.randn(B, 1, H, W, generator=g64(13), dtype=torch.float64)
    fg, fe, gbl = f_g.clone().requires_grad_(), f_e.clone().requires_grad_(), gb.clone().requires_grad_()
    with torch.enable_grad():
        a = torch.cat([fg, (fg - fe).abs()], 1)
        an = F.instance_norm(a, eps=1e-5) * gbl[:, :2 * C, None, None] + gbl[:, 2 * C:, None, None]
        w2l, b2l = w2.clone().requires_grad_(), b2.clone().requires_grad_()
        m = torch.tanh(F.relu(F.conv2d(an, w2l, b2l, padding=1)))
        ((fe * m) * g_p).sum().backward(inputs=[fg, fe, gbl, w2l, b2l], retain_graph=True)
        (m * g_m).sum().backward(inputs=[fg, fe, gbl, w2l, b2l])
    ad = a.detach()
    mean = ad.mean((2, 3))
    rstd = torch.rsqrt(ad.var((2, 3), unbiased=False) + 1e-5)
    stats = torch.stack([mean, rstd], -1)
    g_z, db2, sums, g_fg, g_fe = mask_head_backward(g_p, f_g, f_e, m.detach(), g_m, w2, stats, gb)
    assert rel(db2, b2l.grad) <= 1e-12
    assert rel(torch.cat([sums[..., 1], sums[..., 0]], 1), gbl.grad) <= 1e-12           # (dgamma, dbeta)
    assert rel(g_fg, fg.grad) <= 1e-12 and rel(g_fe, fe.grad) <= 1e-12
    # conv2's weight gradient: the 1-output-channel weight gradient of g_z over the re-applied AdaIN
    assert rel(torch.nn.grad.conv2d_weight(an.detach(), w2.shape, g_z, padding=1), w2l.grad) <= 1e-12


@pytest.mark.parametrize("case", list(CASES))
def test_restated_reference_module_matches_the_oracle(case):
    """The reference module's own statements (grouped modulated convolutions, the benchmark's level (b) arm with the library's ops)
    compute, with torch's ops in float64, what the pinned oracle computes."""
    from tests.oracle_vtoonify_gstep import restated_forward
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict
    backbone, d_s = CASES[case]
    sd = {k: v.double() for k, v in det_state_dict(VToonify(backbone=backbone), seed=0).items()}
    x, style = inputs("ns")
    img, masks = restated_forward(sd, x.double(), style.double(), d_s, backbone)
    torch.set_default_dtype(torch.float64)       # the oracle builds Fusion's d_s label with torch.zeros
    try:
        r = O.vtoonify_forward(sd, x.double(), style.double(), d_s, backbone, return_mask=True)
    finally:
        torch.set_default_dtype(torch.float32)
    ref_img, ref_masks = r if backbone == "dualstylegan" else (r, [])
    assert rel(img, ref_img) <= 1e-12 and len(masks) == len(ref_masks)
    assert all(rel(a, b) <= 1e-12 for a, b in zip(masks, ref_masks))
