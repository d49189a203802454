"""Row-strip entry point (vt_conv2d_rs: the full-resolution 3x3 layers with Cin, Cout in {32, 64}): the default routing by row
width.  Every kernel instantiation, the fused ToRGB and the image-only launch are checked against float64 in
test_gpu_conv_rs_plans.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def _case(B, Cin, Cout, H, W, wB, seed, bias=True, noise=False, act=True):
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, H, W, Cin), generator=g).cuda()
    wt = (torch.randn((wB, Cout, Cin, 3, 3), generator=g) / (3 * Cin ** 0.5)).cuda()
    w = torch.cat([ops.prep_weights(wt[i], cin_pad=Cin, round_tf32=False) for i in range(wB)], dim=0).contiguous()
    kw = dict(bias=(torch.randn(Cout, generator=g) * 0.2).cuda() if bias else None, act=1 if act else 0, slope=0.2, gain=2 ** 0.5)
    if noise:
        kw["noise"] = torch.randn((B, 1, H, W), generator=g).cuda().contiguous()
        kw["noise_w"] = torch.tensor([0.3]).cuda()
    return x, w, kw


def _run(x, w, kw, H, W, rs):
    from vtoonify_b200 import ops
    ops.set_option("rs_conv", rs)
    return ops.conv2d_nhwc([x], w, ops.conv_taps(3, 1), 1, H, W, **kw)


def test_rs_default_routing():
    """by default only rows of >= 256 pixels go to the row-strip kernel; the results agree with the tap-by-tap kernel either way"""
    from vtoonify_b200 import ops
    assert ops.get_option("rs_conv") and ops.get_option("rs_min_width") == 256
    x, w, kw = _case(1, 32, 32, 48, 512, 1, seed=3)
    a = _run(x, w, kw, 48, 512, rs=True)
    b = _run(x, w, kw, 48, 512, rs=False)
    ops.set_option("rs_conv", True)
    assert (a - b).abs().max().item() <= 6e-5 * b.abs().max().item()
