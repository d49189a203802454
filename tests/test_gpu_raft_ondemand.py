"""The on-demand RAFT correlation (ops.set_option("raft_corr", "on_demand")) on the GPU: the fmap pool and the on-demand lookup kernels
against float64 and the reference's alt_cuda_corr, whole RAFT and parsing-map smoothing against the float64 restatements at the existing
bars, the streaming FramePipeline against the two-step route under the option, and the memory of a smoothing batch at 576x1024.
Kernel bars: a few u = 2^-24 times the float64 sum of the absolute terms, as in tests/test_gpu_raft_kernels.py."""
import pytest
import torch
import torch.nn.functional as F

from tests import oracle_raft_ondemand as OD
from tests.golden.make_golden_raft import CASES, raft_args
from vtoonify_b200 import ops, set_precision
from vtoonify_b200._lib import c_void_p, check, load
from vtoonify_b200.raft import RAFT
from vtoonify_b200.weights import det_state_dict

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
DEV = "cuda"


def _st():
    return ops._stream()


@pytest.fixture(autouse=True)
def _restore_options():
    yield
    set_precision(ops.DEFAULT_PRECISION)
    ops.set_option("raft_corr", "volume")


@pytest.fixture(scope="module")
def model_sd():
    torch.manual_seed(0)
    m = RAFT(raft_args()).eval()
    sd = det_state_dict(m, seed=0)
    m.load_state_dict(sd, strict=True)
    m.requires_grad_(False)
    return m.to(DEV), {k: v.to(DEV) for k, v in sd.items()}


def _pool(x):
    """vt_raft_fmap_pool_f32 of an NHWC map"""
    B, h, w, C = x.shape
    out = torch.full((B, h // 2, w // 2, C), float("nan"), device=DEV)
    check(load().vt_raft_fmap_pool_f32(x.data_ptr(), out.data_ptr(), B, h, w, C, _st()))
    return out


@pytest.mark.parametrize("B,h,w,C", [(2, 16, 20, 256), (1, 17, 13, 256), (3, 5, 3, 8)])
def test_fmap_pool_matches_torch(B, h, w, C):
    """floor sizes, odd sides: bit-identical to torch's avg_pool2d, and within 2 u of float64"""
    x = torch.randn(B, h, w, C, generator=torch.Generator().manual_seed(h * w)).to(DEV)
    out = _pool(x)
    ref = F.avg_pool2d(x.permute(0, 3, 1, 2).contiguous(), 2, stride=2).permute(0, 2, 3, 1)
    assert torch.equal(out, ref)
    r64 = F.avg_pool2d(x.double().permute(0, 3, 1, 2), 2, stride=2).permute(0, 2, 3, 1)
    a64 = F.avg_pool2d(x.double().abs().permute(0, 3, 1, 2), 2, stride=2).permute(0, 2, 3, 1)
    assert ((out.double() - r64).abs() <= 3 * U * a64).all()


def _ondemand(f1, levels, coords, cpitch=352, bstride=None):
    """f1 NHWC [B or 1, h, w, 256] (bstride 0: one map for the whole batch), levels NHWC, coords [B, 2, h, w] -> [B, h, w, cpitch]"""
    B, _, h, w = coords.shape
    c = coords.permute(0, 2, 3, 1).contiguous()
    out = torch.full((B, h, w, cpitch), float("nan"), device=DEV)
    lp = (c_void_p * 4)(*[t.data_ptr() for t in levels])
    bs = f1.stride(0) if bstride is None else bstride
    check(load().vt_raft_corr_ondemand_f32(f1.data_ptr(), bs, lp, B, h, w, c.data_ptr(), out.data_ptr(), cpitch, _st()))
    return out


def _levels(f2):
    """NHWC fmap2 -> [fmap2, pooled x3] (torch's float32 pools: the kernel test does not depend on the pool kernel)"""
    lv = [f2]
    for _ in range(3):
        lv.append(F.avg_pool2d(lv[-1].permute(0, 3, 1, 2), 2, stride=2).permute(0, 2, 3, 1).contiguous())
    return lv


def _grid(B, h, w, spread, seed, integer=False):
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    d = spread * torch.randn(B, 2, h, w, generator=g)
    return torch.stack([xs, ys])[None] + (torch.round(d) if integer else d)


EDGE = [[-1.0, -0.5, 20.5, 21.0, 1e4, -3e6, -4.0, -9.5, -13.0, 0.0, float("nan"), 3.999999761581421],
        [-0.25, -1.0, 0.0, 16.0, 5.0, 2.0, -7.75, 30.0, -4.0, -41.0, 1.0, -1e-7]]


def _check_against_float64(f1, lv, coords, out, f1_full=None):
    """out against the float64 restatement on the same float32 inputs; bar: the 8-term FMA chains and 5-level lane tree of each dot
    and the 4-term tap sum (a few u of the absolute dot), plus the float32 rounding of coords / 2^l + offset, which moves a tap along a
    slope of at most 2 absolute dots per pixel (as in test_corr_lookup_against_float64)"""
    f1 = f1 if f1_full is None else f1_full
    B, h, w, C = f1.shape
    f1n = f1.double().permute(0, 3, 1, 2)
    pyr = [t.double().permute(0, 3, 1, 2) for t in lv]
    c64 = coords.double()
    finite = torch.isfinite(c64).all(1, keepdim=True)
    ref = OD.ondemand(f1n, pyr, torch.where(finite, c64, torch.full_like(c64, -1e9))).permute(0, 2, 3, 1)
    amax = max(float(torch.einsum("bchw,bcHW->bhwHW", f1n.abs(), p.abs()).max()) for p in pyr) / 16.0
    cmax = float(c64.nan_to_num(0).clamp(-30, 30).abs().max()) + 4
    err = (out[..., :324].double() - ref).abs().max().item()
    print(f"on-demand lookup: max |err| {err:.3e}, bar {U * amax * (24 + 4 * cmax):.3e}")
    assert err <= U * amax * (24 + 4 * cmax), err
    assert (out[..., 324:].view(torch.int32) == 0).all()          # pad channels exactly +0


@pytest.mark.parametrize("B,h,w,spread,integer", [(1, 17, 21, 0.0, False), (2, 16, 24, 0.0, True), (2, 19, 13, 2.5, False),
                                                  (3, 24, 32, 9.0, False), (1, 9, 8, 40.0, False)])
def test_ondemand_against_float64(B, h, w, spread, integer):
    """pixel centres, integer and fractional flows, far-reaching flows, odd h and w (odd level sizes), B > 1; the first row also holds
    border, just- and far-outside, negative, non-finite and just-below-integer coordinates"""
    g = torch.Generator().manual_seed(B * h + w)
    f1, f2 = torch.randn(B, h, w, 256, generator=g).to(DEV), torch.randn(B, h, w, 256, generator=g).to(DEV)
    coords = _grid(B, h, w, spread, h + w, integer)
    n = min(w, len(EDGE[0]))
    coords[0, :, 0, :n] = torch.tensor(EDGE)[:, :n]
    coords = coords.to(DEV)
    lv = _levels(f2)
    out = _ondemand(f1, lv, coords)
    _check_against_float64(f1, lv, coords, out)
    assert torch.equal(out, _ondemand(f1, lv, coords))                # reruns are bit-identical
    assert not out[0, 0, 4, :324].any() and (w <= 10 or not out[0, 0, 10, :324].any())   # far outside and NaN: zeros


def test_ondemand_fmap1_batch_stride_zero():
    """one fmap1 for every pair (batch stride 0, as expand gives) equals the materialised copies bit for bit"""
    B, h, w = 4, 16, 20
    g = torch.Generator().manual_seed(5)
    f1 = torch.randn(1, h, w, 256, generator=g).to(DEV)
    f2 = torch.randn(B, h, w, 256, generator=g).to(DEV)
    coords = _grid(B, h, w, 3.0, 6).to(DEV)
    lv = _levels(f2)
    out0 = _ondemand(f1, lv, coords, bstride=0)
    full = f1.expand(B, -1, -1, -1).contiguous()
    assert torch.equal(out0, _ondemand(full, lv, coords))
    _check_against_float64(f1, lv, coords, out0, f1_full=full)


def test_ondemand_against_reference_alt_cuda_corr():
    """the reference's alt_cuda_corr forward on each level (fmap1 with the pooled fmap2, coords / 2^l), / 16; h a multiple of 4 and w
    of 8, since its 4x8 blocks read unset shared coordinates past the map's edge"""
    from oracle.build_ref_alt_corr import load_alt_corr
    alt = load_alt_corr()
    if alt is None:
        pytest.skip("the reference's alt_cuda_corr is not built (oracle/build_ref_alt_corr.py)")
    B, h, w = 2, 16, 24
    g = torch.Generator().manual_seed(11)
    f1, f2 = torch.randn(B, h, w, 256, generator=g).to(DEV), torch.randn(B, h, w, 256, generator=g).to(DEV)
    coords = _grid(B, h, w, 4.0, 12)
    coords[0, :, 0, :6] = torch.tensor([[-1.0, -0.5, 23.5, 24.0, -30.0, 2.5], [-0.25, -1.0, 0.0, 16.0, 5.0, -12.0]])
    coords = coords.to(DEV)
    lv = _levels(f2)
    out = _ondemand(f1, lv, coords)
    cl = coords.permute(0, 2, 3, 1)
    amax = max(float(torch.einsum("bhwc,bHWc->bhwHW", f1.double().abs(), p.double().abs()).max()) for p in lv) / 16.0
    cmax = float(coords.clamp(-30, 30).abs().max()) + 4
    for l in range(4):
        corr, = alt.forward(f1.contiguous(), lv[l].contiguous(), (cl / 2 ** l).reshape(B, 1, h, w, 2).contiguous(), 4)
        ref = (corr[:, 0] / 16.0).permute(0, 2, 3, 1)
        err = (out[..., l * 81:(l + 1) * 81] - ref).abs().max().item()
        print(f"level {l}: max |on-demand - alt_cuda_corr| {err:.3e}")
        assert err <= U * amax * (64 + 4 * cmax), (l, err)


# ------------------------------------------------------------------------------------------------------------------ whole model
@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "tf32"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_forward_on_demand_against_float64(model_sd, name, prec):
    from tests.test_gpu_raft import BARS, _oracle64, _rel, _run
    m, sd = model_sd
    c = CASES[name]
    set_precision(prec)
    ops.set_option("raft_corr", "on_demand")
    out = _run(m, c)
    ref = _oracle64(sd, c)
    if c["test_mode"]:
        err = max(_rel(out[0], ref[0]), _rel(out[1], ref[1]))
    else:
        assert isinstance(out, list) and len(out) == c["iters"]
        err = max(_rel(o, r) for o, r in zip(out, ref))
    print(f"RAFT on demand {name} {prec}: worst relative L2 {err:.3e}")
    assert err <= BARS[prec], err


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "tf32"])
@pytest.mark.parametrize("name", ["w2", "w5"])
def test_smoothing_on_demand_against_float64(golden, model_sd, name, prec):
    from tests import oracle_smooth as OS
    from tests.test_gpu_smooth import BARS, _rel
    from tests.test_smooth_host import case
    from vtoonify_b200 import smooth_parsing as S
    m, sd = model_sd
    Is, Ps, window, ch, ref32 = case(golden, name)
    set_precision(prec)
    ops.set_option("raft_corr", "on_demand")
    with torch.no_grad():
        out = S.smooth_parsing_maps(Is, Ps, m, window=window, iters=20)
        sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
        ref = OS.smooth(sd64, Is.to(DEV).double(), Ps.to(DEV).double(), window, 20)
    err = _rel(out, ref.cpu())
    print(f"smoothing on demand {name} {prec}: relative L2 {err:.3e} against float64, {_rel(out[:, ch], ref32):.3e} against the fixture")
    assert err <= BARS[prec], err


def test_pipeline_on_demand_matches_two_step_route(model_sd):
    from tests.test_gpu_smooth_stream import _batches, _frames, _nets, _two_step
    from vtoonify_b200.frame_loop import FramePipeline
    from vtoonify_b200.weights import det_inputs
    raft = model_sd[0]
    m, p = _nets()
    set_precision("bf16x3")
    ops.set_option("raft_corr", "on_demand")
    B, N, window, iters, H, W = 3, 8, 2, 3, 64, 64
    style = det_inputs(1, 32, 32, seed=5)[1]
    frames = _frames(N, H, W, seed=77)
    outs = list(FramePipeline(m, style, d_s=0.5, parsing_net=p, smoothing=(raft, window, iters)).run(_batches(frames, B)))
    ref = _two_step(m, p, raft, style, frames, B, window, iters)
    assert len(outs) == len(ref) == (N + B - 1) // B
    for k, (o, r) in enumerate(zip(outs, ref)):
        assert o.shape == r.shape and torch.equal(o, r), k


def test_smoothing_batch_576x1024_memory(model_sd):
    """the 10-pair smoothing batch of 576x1024 frames (RAFT at 1152x2048: h, w = 144, 256) runs on demand, 2 iterations; its peak
    allocation above the inputs stays below every per-iteration activation held at once, twice over (2 x 2592 floats per pixel: the
    352-channel lookup, convc1/c2, convf1/f2, the GRU's z|r, q and r*h, the flow head, the mask head's 256 + 576) plus the pooled
    fmap2 levels (85 floats per pixel) and the up-sampled flow (128 per pixel): about 8 GB, where the volume's pyramid alone is 72 GB"""
    m = model_sd[0]
    set_precision("bf16x3")
    ops.set_option("raft_corr", "on_demand")
    B, h, w = 10, 144, 256
    g = torch.Generator(device=DEV).manual_seed(0)
    f1 = torch.randn(1, h, w, 256, device=DEV, generator=g)
    f2 = torch.randn(B, h, w, 256, device=DEV, generator=g)
    net = torch.tanh(torch.randn(B, h, w, 128, device=DEV, generator=g))
    x = torch.relu(torch.randn(B, h, w, 256, device=DEV, generator=g))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        low, up = m._iterate(f1.expand(B, -1, -1, -1), f2, net, x, 2)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    npix = B * h * w
    bound = 4 * npix * (2 * 2592 + 85 + 128)
    volume = 4 * B * (h * w) ** 2 * (1 + 1 / 4 + 1 / 16 + 1 / 64)
    print(f"576x1024 smoothing batch on demand: peak {peak / 1e9:.2f} GB above the inputs (bound {bound / 1e9:.2f} GB; "
          f"the volume's pyramid {volume / 1e9:.1f} GB)")
    assert up.shape == (B, 2, 8 * h, 8 * w) and torch.isfinite(up).all() and torch.isfinite(low).all()
    assert peak <= bound, (peak, bound)
