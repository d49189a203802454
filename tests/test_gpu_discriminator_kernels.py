"""GPU: the minibatch standard deviation kernels (vt_mbstd_nhwc_f32, vt_mbstd_grad_nhwc_f32) against float64 autograd of the
reference expression (model/vtoonify.py:67-75), on ordinary planes and on planes whose mean is large next to their spread."""
import pytest
import torch

from tests.oracle_discriminator import mbstd as ref_mbstd

pytestmark = pytest.mark.gpu


def _planes(B, C, H, W, kind, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, C, H, W), generator=g)
    if kind == "offset":                 # mean 1e3 next to a spread of 1e-2 (the statistic is then ~1e-2)
        x = 1e3 + 1e-2 * x
    elif kind == "constant":             # zero variance: the statistic is sqrt(1e-8)
        x = torch.full((B, C, H, W), 0.3)
    return x


@pytest.mark.parametrize("B,C,H,W", [(8, 512, 4, 4), (4, 512, 4, 4), (2, 64, 3, 5), (1, 40, 4, 4), (12, 96, 2, 2), (3, 32, 4, 4)])
@pytest.mark.parametrize("kind", ["randn", "offset", "constant"])
def test_mbstd_forward_and_grad(B, C, H, W, kind):
    from vtoonify_b200 import ops
    x = _planes(B, C, H, W, kind, B * 100 + C)
    group = min(B, 4)
    xd = x.double().requires_grad_()
    with torch.enable_grad():
        ref = ref_mbstd(xd)                                    # [B, C + 1, H, W]
        u = torch.randn(ref.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
        (ref * u).sum().backward()
    xn = ops.to_nhwc(x.cuda())
    out = ops.mbstd(xn, group)
    Cp = out.shape[3]
    assert Cp == (C + 1 + 31) // 32 * 32
    got = out.permute(0, 3, 1, 2).double().cpu()
    assert torch.equal(got[:, :C], x.double())                 # the copied channels are exact
    assert (got[:, C + 1:] == 0).all()
    s_ref, s_got = ref[:, C].detach(), got[:, C]
    assert (s_got - s_ref).abs().max().item() <= 2e-6 * s_ref.abs().max().item()
    gin = torch.zeros((B, Cp, H, W), dtype=torch.float64)
    gin[:, :C + 1] = u
    gin[:, C + 1:] = 123.0                                     # the pad channels' gradient must be ignored
    gx = ops.mbstd_grad(ops.to_nhwc(gin.float().cuda()), xn, group)
    gx = gx.permute(0, 3, 1, 2).double().cpu()
    err = (gx - xd.grad).abs().max().item()
    assert err <= 2e-6 * xd.grad.abs().max().item() + 1e-6, f"{kind} B={B}: {err:.3e}"
    # deterministic
    assert torch.equal(ops.mbstd(xn, group), out)
    assert torch.equal(ops.mbstd_grad(ops.to_nhwc(gin.float().cuda()), xn, group).permute(0, 3, 1, 2).double().cpu(), gx)


def test_mbstd_rejects_uneven_batch():
    from vtoonify_b200 import _lib, ops
    x = torch.zeros((6, 4, 4, 512), device="cuda")
    with pytest.raises(_lib.VtError):
        ops.mbstd(x, 4)
    with pytest.raises(_lib.VtError):
        ops.mbstd_grad(torch.zeros((6, 4, 4, 544), device="cuda"), x, 4)
