"""The smoothing kernels (csrc/smooth.cu) on the GPU: the warp's mask against torch's CUDA grid_sample bit for bit, the warped values and
the window fusion against float64, the all-masked case, reruns, launches and guard regions."""
import pytest
import torch
import torch.nn.functional as F

from tests import oracle_smooth as O
from vtoonify_b200 import smooth_parsing as S
from vtoonify_b200._lib import check, launch_count, load

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _flows(B, H, W, seed, scale=12.0, quantum=None):
    g = torch.Generator().manual_seed(seed)
    f = (torch.rand((B, 2, H, W), generator=g) - 0.5) * scale
    f[:, :, : H // 6] = 0.0
    f[:, 0, H // 6: H // 5] = 4000.0                           # far outside
    if quantum:
        f = torch.round(f / quantum) * quantum
    return f


def _pixel_coords(flo):
    """the sample positions in pixels, in float32 exactly as the reference computes them (true division, then grid_sample's
    unnormalisation), as float64"""
    B, _, H, W = flo.shape
    g = O.sample_grid(flo.cpu().float())
    ix = ((g[..., 0] + 1.0) / 2) * (W - 1)
    iy = ((g[..., 1] + 1.0) / 2) * (H - 1)
    return ix.double(), iy.double()


def _bilinear64(x, ix, iy):
    """x [B, C, H, W] float64 sampled at pixel positions ix, iy [B, H, W] (zeros outside), per channel"""
    B, C, H, W = x.shape
    x0, y0 = torch.floor(ix), torch.floor(iy)
    out = torch.zeros_like(x)
    flat = x.reshape(B, C, H * W)
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        xi, yi = x0 + dx, y0 + dy
        w = (1 - (ix - xi).abs()) * (1 - (iy - yi).abs())
        ok = (xi >= 0) & (xi <= W - 1) & (yi >= 0) & (yi <= H - 1)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long().reshape(B, 1, H * W).expand(B, C, H * W)
        v = flat.gather(2, idx).reshape(B, C, H, W)
        out = out + torch.where(ok[:, None], v * w[:, None], torch.zeros_like(v))
    return out


@pytest.mark.parametrize("shape", [(2, 22, 31, 37), (1, 3, 45, 61), (3, 1, 128, 136)])
def test_warp_mask_bit_identical_to_grid_sample(shape):
    B, C, H, W = shape
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1)).to(DEV)
    flo = _flows(B, H, W, 2).to(DEV)
    out, mask = S.warp(x, flo)
    _, ref = O.warp(x, flo)                       # torch's CUDA grid_sample of ones, thresholded
    assert torch.equal(mask, ref)
    assert 0.1 < float(mask.mean()) < 0.95
    assert torch.equal(mask, mask[:, :1].expand_as(mask))


@pytest.mark.parametrize("C", [1, 3, 22])
@pytest.mark.parametrize("HW", [(31, 37), (64, 72), (127, 133)])
def test_warp_values_against_float64(C, HW):
    H, W = HW
    x = torch.randn((2, C, H, W), generator=torch.Generator().manual_seed(C)).to(DEV)
    flo = _flows(2, H, W, 3 + H).to(DEV)
    out, mask = S.warp(x, flo)
    ix, iy = _pixel_coords(flo)
    ref = _bilinear64(x.double().cpu(), ix, iy) * mask.double().cpu()
    err = float((out.double().cpu() - ref).abs().max())
    print(f"warp C={C} {H}x{W}: max |err| {err:.2e}")
    assert err <= 2e-6, err                       # measured worst 4.0e-7: a few ulps of values of magnitude ~4


def _fuse_inputs(window, C, H, W, seed, far=False):
    S_ = 2 * window + 1
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand((1, 3, 6, 7), generator=g), size=(H, W), mode="bilinear", align_corners=False) * 2 - 1
    imgs = (base + 0.15 * torch.randn((S_, 3, H, W), generator=g)).contiguous()
    pars = (4.0 * torch.randn((S_, C, H, W), generator=g)).contiguous()
    flows = _flows(S_, H, W, seed + 1, quantum=0.125)      # positions on a 1/8 grid: no mask sits near the 0.9999 threshold
    if far:
        flows.fill_(1e4)
    return imgs, pars, flows


@pytest.mark.parametrize("window", [0, 1, 5])
def test_fuse_against_float64(window):
    C, H, W = 19, 67, 83
    imgs, pars, flows = _fuse_inputs(window, C, H, W, 10 + window)
    wt = S.temporal_weights(window)
    d = [t.to(DEV) for t in (imgs, pars, flows)]
    n0 = launch_count()
    out = S.parsing_fuse(list(d[0]), list(d[1]), list(d[2]), wt.tolist())
    assert launch_count() - n0 == 1
    ref = O.fuse(imgs.double(), pars.double(), flows.double(), wt.double())
    err = float((out.double().cpu() - ref).norm() / ref.norm())
    mx = float((out.double().cpu() - ref).abs().max())
    print(f"fuse window={window}: relative L2 {err:.2e}, max |err| {mx:.2e}")
    assert err <= 5e-6 and mx <= 1.2e-4, (err, mx)       # measured worst 1.1e-6 and 3.1e-5
    again = S.parsing_fuse(list(d[0]), list(d[1]), list(d[2]), wt.tolist())
    assert torch.equal(out, again)


def test_fuse_all_masked_is_the_centre_map():
    window, C, H, W = 2, 5, 40, 48
    imgs, pars, flows = _fuse_inputs(window, C, H, W, 3, far=True)
    d = [t.to(DEV) for t in (imgs, pars, flows)]
    out = S.parsing_fuse(list(d[0]), list(d[1]), list(d[2]), S.temporal_weights(window).tolist())
    torch.testing.assert_close(out, d[1][window], rtol=1e-7, atol=0)


def test_warp_rerun_and_guard_regions():
    B, C, H, W = 2, 4, 33, 35
    x = torch.randn((B, C, H, W), generator=torch.Generator().manual_seed(4)).to(DEV)
    flo = _flows(B, H, W, 5).to(DEV)
    n = B * C * H * W
    G = 4096
    buf = torch.full((2 * n + 3 * G,), float("nan"), device=DEV)
    out, mask = buf[G:G + n], buf[2 * G + n:2 * G + 2 * n]
    n0 = launch_count()
    check(load().vt_flow_warp_f32(x.data_ptr(), flo.data_ptr(), out.data_ptr(), mask.data_ptr(), B, C, H, W,
                                  torch.cuda.current_stream().cuda_stream))
    assert launch_count() - n0 == 1
    torch.cuda.synchronize()
    for lo, hi in ((0, G), (G + n, 2 * G + n), (2 * G + 2 * n, 3 * G + 2 * n)):
        assert torch.isnan(buf[lo:hi]).all()
    ref_out, ref_mask = S.warp(x, flo)
    assert torch.equal(out.view(B, C, H, W), ref_out) and torch.equal(mask.view(B, C, H, W), ref_mask)


def test_fuse_guard_regions():
    window, C, H, W = 1, 3, 29, 31
    imgs, pars, flows = _fuse_inputs(window, C, H, W, 7)
    d = [t.to(DEV) for t in (imgs, pars, flows)]
    n, G = C * H * W, 2048
    buf = torch.full((n + 2 * G,), float("nan"), device=DEV)
    out = S.parsing_fuse(list(d[0]), list(d[1]), list(d[2]), S.temporal_weights(window).tolist(), out=buf[G:G + n].view(C, H, W))
    assert torch.isnan(buf[:G]).all() and torch.isnan(buf[G + n:]).all() and torch.isfinite(out).all()


def test_fuse_argument_errors():
    t3, t2 = torch.zeros((3, 16, 16), device=DEV), torch.zeros((2, 16, 16), device=DEV)
    with pytest.raises(ValueError):
        S.parsing_fuse([t3, t3], [t3, t3], [t2, t2], [1.0, 1.0])          # an even number of slots
    with pytest.raises(ValueError):
        S.parsing_fuse([t3] * 3, [t3] * 3, [t2, None, t2[:, :8]], [1.0] * 3)
