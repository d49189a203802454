"""The RAFT kernels of csrc/raft.cu against float64 (and torch bit for bit where the summation order allows it).
Bars: a few u = 2^-24 times the float64 sum of the absolute terms, as in tests/test_gpu_gstep_kernels.py."""
import pytest
import torch
import torch.nn.functional as F

from tests import oracle_raft as O
from vtoonify_b200 import ops
from vtoonify_b200._lib import c_int64, c_void_p, check, load

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
DEV = "cuda"


def _g(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _st():
    return ops._stream()


def test_input_s2d_against_float64():
    g = _g(0)
    B, H, W = 2, 16, 24
    i1, i2 = (torch.rand(B, 3, H, W, generator=g) * 255).to(DEV), (torch.rand(B, 3, H, W, generator=g) * 255).to(DEV)
    out = torch.full((2 * B, H // 2, W // 2, 32), float("nan"), device=DEV)
    check(load().vt_raft_input_s2d_f32(i1.data_ptr(), i2.data_ptr(), out.data_ptr(), B, H, W, 32, _st()))
    x = 2 * (torch.cat([i1, i2]).double() / 255.0) - 1.0
    ref = x.reshape(2 * B, 3, H // 2, 2, W // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(2 * B, H // 2, W // 2, 12)
    # one rounding of x / 255 (doubled exactly) and one of the subtraction; torch's CUDA scalar division multiplies by 1/255 instead,
    # so it is not a bit-exact yardstick (the reference runs the true division on the CPU, as the kernel does)
    assert (out[..., :12].double() - ref.double()).abs().max().item() <= 4 * U and not out[..., 12:].any()


@pytest.mark.parametrize("h,w,pad", [(16, 20, 0), (17, 13, 12), (5, 3, 1)])
def test_corr_pool_matches_torch(h, w, pad):
    """avg_pool2d(2, 2) with floor sizes, rows read at a padded stride: bit-identical to torch's CUDA kernel"""
    N = 37
    src = torch.randn(N, h * w + pad, generator=_g(h)).to(DEV)
    out = torch.empty(N, (h // 2) * (w // 2), device=DEV)
    check(load().vt_raft_corr_pool_f32(src.data_ptr(), out.data_ptr(), N, h, w, h * w + pad, _st()))
    ref = F.avg_pool2d(src[:, :h * w].reshape(N, 1, h, w), 2, stride=2).reshape(N, -1)
    assert torch.equal(out, ref)


def _lookup(levels, h2, w2, coords, cpitch=352):
    """levels: float32 [N, h_l*w_l] device tensors; coords [B, 2, h, w] -> [B, h, w, cpitch]"""
    B, _, h, w = coords.shape
    c = coords.permute(0, 2, 3, 1).contiguous()
    out = torch.full((B, h, w, cpitch), 7.0, device=DEV)
    lp = (c_void_p * 4)(*[t.data_ptr() for t in levels])
    ls = (c_int64 * 4)(*[t.shape[1] for t in levels])
    check(load().vt_raft_corr_lookup_f32(lp, ls, h2, w2, c.data_ptr(), out.data_ptr(), cpitch, B * h * w, _st()))
    return out


def test_corr_lookup_against_float64(golden):
    """fixture feature maps [1, 16, 17, 21] (level sizes 17x21, 8x10, 4x5, 2x2: odd sides); coordinates on pixel centres, fractional,
    on the border, just and far outside"""
    g = golden("raft_lookup")
    h2, w2 = g["fmap1"].shape[2:]
    pyr = O.pyramid(torch.from_numpy(g["fmap1"]).to(DEV), torch.from_numpy(g["fmap2"]).to(DEV))
    pyr = [p.reshape(p.shape[0], -1).contiguous() for p in pyr]
    fx = torch.from_numpy(g["coords"]).to(DEV)
    ref_fx = torch.from_numpy(g["corr"]).to(DEV).permute(0, 2, 3, 1)
    assert (_lookup(pyr, h2, w2, fx)[..., :324] - ref_fx).abs().max().item() <= 2e-5 * float(ref_fx.abs().max())
    coords = fx.clone()
    coords[0, :, 1, :6] = torch.tensor([[-1.0, -0.5, 20.5, 21.0, 1e4, -3e6], [-0.25, -1.0, 0.0, 16.0, 5.0, 2.0]], device=DEV)
    out = _lookup(pyr, h2, w2, coords)
    p64 = [p.double().reshape(-1, h2 >> i, w2 >> i) for i, p in enumerate(pyr)]
    ref = O.lookup(p64, coords.double()).permute(0, 2, 3, 1)
    amax = max(float(p.abs().max()) for p in pyr)
    # besides the 4-term sum (a few u of amax), the float32 sample coordinate coords / 2^l + offset is rounded once: its error of
    # u * |x| moves the sample along a slope of at most 2 * amax per pixel
    cmax = float(coords.clamp(-30, 30).abs().max()) + 4
    err = (out[..., :324].double() - ref).abs().max().item()
    assert err <= U * amax * (8 + 4 * cmax), err
    assert torch.equal(out[..., 324:], torch.full_like(out[..., 324:], 7.0))      # pad channels untouched


def test_gru_gates_saturated():
    g = _g(3)
    npix, C = 999, 128
    zr = (torch.randn(npix, 2 * C, generator=g) * 40).to(DEV)
    h = torch.randn(npix, C, generator=g).to(DEV)
    q = (torch.randn(npix, C, generator=g) * 30).to(DEV)
    rh = torch.empty_like(h)
    check(load().vt_raft_gru_reset_f32(zr.data_ptr(), h.data_ptr(), rh.data_ptr(), npix, C, _st()))
    ref = torch.sigmoid(zr[:, C:].double()) * h.double()
    assert (rh.double() - ref).abs().max().item() <= 4 * U * h.abs().max().item()
    hn = h.clone()
    check(load().vt_raft_gru_update_f32(zr.data_ptr(), q.data_ptr(), hn.data_ptr(), npix, C, _st()))
    z = torch.sigmoid(zr[:, :C].double())
    ref = (1 - z) * h.double() + z * torch.tanh(q.double())
    assert torch.isfinite(hn).all()
    assert (hn.double() - ref).abs().max().item() <= 8 * U * (h.abs().double() + 1).max().item()


def test_convf1_against_float64():
    g = _g(4)
    B, h, w = 2, 9, 14
    conv = torch.nn.Conv2d(2, 128, 7, padding=3)
    flow = (torch.randn(B, 2, h, w, generator=g) * 5).to(DEV)
    coords = torch.empty(B, h, w, 2, device=DEV)
    check(load().vt_raft_flow_f32(coords.data_ptr(), flow.data_ptr(), 1, None, 2, B, h, w, _st()))
    wt = conv.weight.detach().permute(2, 3, 1, 0).reshape(49, 2, 128).contiguous().to(DEV)
    b = conv.bias.detach().to(DEV)
    out = torch.empty(B, h, w, 128, device=DEV)
    check(load().vt_raft_convf1_f32(coords.data_ptr(), wt.data_ptr(), b.data_ptr(), out.data_ptr(), B, h, w, 128, _st()))
    grid = torch.stack(torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")[::-1], 0).to(DEV).double()
    f64 = coords.permute(0, 3, 1, 2).double() - grid
    ref = F.relu(F.conv2d(f64, conv.weight.double().to(DEV), conv.bias.double().to(DEV), padding=3)).permute(0, 2, 3, 1)
    terms = F.conv2d(f64.abs(), conv.weight.double().abs().to(DEV), conv.bias.double().abs().to(DEV), padding=3).permute(0, 2, 3, 1)
    assert ((out.double() - ref).abs() <= 4 * U * terms * 2 + 1e-30).all()
    assert (f64 - flow.double()).abs().max().item() <= 2 * U * 32          # coords = grid + flow, one rounding


def test_flow_init_update_and_store():
    B, h, w = 2, 5, 7
    coords = torch.empty(B, h, w, 2, device=DEV)
    check(load().vt_raft_flow_f32(coords.data_ptr(), None, 1, None, 2, B, h, w, _st()))
    assert torch.equal(coords[1, 3, 6], torch.tensor([6.0, 3.0], device=DEV))
    d = torch.randn(B, 2, h, w, generator=_g(5)).to(DEV)
    x = torch.zeros(B, h, w, 256, device=DEV)
    check(load().vt_raft_flow_f32(coords.data_ptr(), d.data_ptr(), 0, x[..., 254:].data_ptr(), 256, B, h, w, _st()))
    grid = torch.stack(torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")[::-1], -1).to(DEV).float()
    assert torch.equal(coords, grid + d.permute(0, 2, 3, 1))
    assert torch.equal(x[..., 254:], coords - grid) and not x[..., :254].any()


def test_upsample_large_logits():
    g = _g(6)
    B, h, w = 2, 6, 9
    mask = (torch.randn(B, h, w, 576, generator=g) * 60).to(DEV)
    flow = (torch.randn(B, 2, h, w, generator=g) * 4).to(DEV)
    coords = torch.empty(B, h, w, 2, device=DEV)
    check(load().vt_raft_flow_f32(coords.data_ptr(), flow.data_ptr(), 1, None, 2, B, h, w, _st()))
    up = torch.empty(B, 2, 8 * h, 8 * w, device=DEV)
    low = torch.empty(B, 2, h, w, device=DEV)
    check(load().vt_raft_upsample_f32(mask.data_ptr(), 576, coords.data_ptr(), up.data_ptr(), low.data_ptr(), B, h, w, _st()))
    grid = torch.stack(torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")[::-1], 0).to(DEV).double()
    f64 = coords.permute(0, 3, 1, 2).double() - grid
    assert torch.equal(low.double(), f64)
    ref = O.upsample(f64, mask.double().permute(0, 3, 1, 2))
    assert torch.isfinite(up).all()
    assert (up.double() - ref).abs().max().item() <= 16 * U * 8 * f64.abs().max().item()


def test_norm_relu_against_float64():
    g = _g(7)
    B, HW, C = 2, 300, 96
    x, r = torch.randn(B, HW, C, generator=g).to(DEV), torch.randn(B, HW, C, generator=g).to(DEV)
    st = torch.stack([torch.randn(B, C, generator=g), torch.rand(B, C, generator=g) + 0.5], -1).to(DEV).contiguous()
    sr = torch.stack([torch.randn(B, C, generator=g), torch.rand(B, C, generator=g) + 0.5], -1).to(DEV).contiguous()
    out = torch.empty_like(x)
    check(load().vt_raft_norm_relu_nhwc(x.data_ptr(), st.data_ptr(), r.data_ptr(), sr.data_ptr(), out.data_ptr(), B, HW, C, _st()))
    n = lambda t, s: (t.double() - s[:, None, :, 0].double()) * s[:, None, :, 1].double()
    ref = F.relu(F.relu(n(x, st)) + n(r, sr))
    assert (out.double() - ref).abs().max().item() <= 8 * U * (n(x, st).abs() + n(r, sr).abs()).max().item()
    check(load().vt_raft_norm_relu_nhwc(x.data_ptr(), st.data_ptr(), None, None, out.data_ptr(), B, HW, C, _st()))
    assert (out.double() - F.relu(n(x, st))).abs().max().item() <= 4 * U * n(x, st).abs().max().item()
