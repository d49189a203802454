"""conv_rs_kernel (the row-strip layers with output channels on the wgmma M and pixels on N) against the fp32 FFMA kernel and against
the conv_tc_kernel route of vt_conv2d_rs (option rs_kernel = 0), for every Cin / Cout in {32, 64}."""
import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture()
def lib():
    from vtoonify_b200 import _lib, ops
    lib = _lib.load()
    old = {k: ops.get_option(k) for k in ("rs_min_width", "rs_fmt", "rs_conv")}
    ops.set_option("rs_min_width", 1)
    ops.set_option("rs_conv", True)
    yield lib
    for k, v in old.items():
        ops.set_option(k, v)
    lib.vt_set_option(b"rs_kernel", 1)


def _case(B, Cin, Cout, H, W, wB, seed, bias=True, noise=True):
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, H, W, Cin), generator=g).cuda()
    wt = (torch.randn((wB, Cout, Cin, 3, 3), generator=g) / (3 * Cin ** 0.5)).cuda()
    w = torch.cat([ops.prep_weights(wt[i], cin_pad=Cin, round_tf32=False) for i in range(wB)], dim=0).contiguous()
    kw = dict(bias=(torch.randn(Cout, generator=g) * 0.2).cuda() if bias else None, act=1, slope=0.2, gain=2 ** 0.5)
    if noise:
        kw["noise"] = torch.randn((B, 1, H, W), generator=g).cuda().contiguous()
        kw["noise_w"] = torch.tensor([0.3]).cuda()
    return x, w, kw


def _run(lib, x, w, kw, H, W, route, precision=None, rgb=None, **extra):
    from vtoonify_b200 import ops
    lib.vt_set_option(b"rs_kernel", route)
    return ops.conv2d_nhwc([x], w, ops.conv_taps(3, 1), 1, H, W, precision=precision, rgb=rgb, **kw, **extra)


def _rel(a, b):
    return (a - b).abs().max().item() / b.abs().max().item()


CHANNELS = [(32, 32), (32, 64), (64, 32), (64, 64)]
SHAPES = [
    # B, H, W, wB, bias, noise
    (1, 37, 100, 1, True, True),      # ragged: neither H nor W a multiple of the 8 x 16 tile
    (3, 21, 420, 3, False, True),     # per-sample weights, no bias: 318 tiles, so CTAs cross sample boundaries and reload weights
    (2, 64, 256, 1, True, False),
]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"s{i}" for i in range(len(SHAPES))])
@pytest.mark.parametrize("cin,cout", CHANNELS, ids=[f"{a}to{b}" for a, b in CHANNELS])
def test_conv_rs_kernel_vs_fp32_and_conv_tc(lib, cin, cout, shape):
    B, H, W, wB, bias, noise = shape
    x, w, kw = _case(B, cin, cout, H, W, wB, seed=B * 100 + H + cin + cout, bias=bias, noise=noise)
    ref = _run(lib, x, w, kw, H, W, 1, precision="fp32")
    y = _run(lib, x, w, kw, H, W, 1)
    y2 = _run(lib, x, w, kw, H, W, 1)
    tc = _run(lib, x, w, kw, H, W, 0)
    torch.cuda.synchronize()
    assert torch.equal(y, y2), "conv_rs_kernel is not deterministic"
    e_ref, e_tc = _rel(y, ref), _rel(y, tc)
    print(f"conv_rs {cin}->{cout} {shape}: vs fp32 {e_ref:.2e}, vs conv_tc route {e_tc:.2e}")
    assert e_ref <= 4e-5 and e_tc <= 4e-5


@pytest.mark.parametrize("c", [32, 64])
def test_conv_rs_kernel_fused_torgb(lib, c):
    B, H, W, wB = 2, 40, 272, 2
    x, w, kw = _case(B, c, c, H, W, wB, seed=7 + c)
    g = torch.Generator().manual_seed(11)
    k1 = torch.tensor([1., 3., 3., 1.])
    rgb = {"w": (torch.randn((wB, 1, 3, c), generator=g) * 0.2).cuda(), "bias": (torch.randn(3, generator=g) * 0.1).cuda(),
           "skip": torch.randn((B, 3, H // 2, W // 2), generator=g).cuda(), "kernel": (k1[:, None] * k1[None, :] / 64 * 4).cuda()}
    ref = _run(lib, x, w, kw, H, W, 1, precision="fp32")   # the FFMA kernel has no fused ToRGB: the image is checked against conv_tc
    for r in (rgb, dict(rgb, skip=None, kernel=None)):
        tc, tc_rgb = _run(lib, x, w, kw, H, W, 0, rgb=r)
        y, y_rgb = _run(lib, x, w, kw, H, W, 1, rgb=r)
        none_out, only = _run(lib, x, w, kw, H, W, 1, rgb=dict(r, only=True))
        torch.cuda.synchronize()
        assert _rel(y, ref) <= 4e-5 and _rel(y, tc) <= 4e-5 and _rel(y_rgb, tc_rgb) <= 6e-5
        # the image-only launch (no activation written) gives the same image bit for bit
        assert none_out is None and torch.equal(only, y_rgb)


@pytest.mark.parametrize("cin,cout", CHANNELS, ids=[f"{a}to{b}" for a, b in CHANNELS])
def test_conv_rs_fallbacks(lib, cin, cout):
    """descriptors conv_rs_kernel does not take still give the right result through conv_tc_kernel: the fp16 split, and a launch
    that also writes the instance-norm statistics of its output"""
    from vtoonify_b200 import ops
    B, H, W = 2, 24, 136
    x, w, kw = _case(B, cin, cout, H, W, 1, seed=cin * 3 + cout)
    ref = _run(lib, x, w, kw, H, W, 1, precision="fp32")
    ops.set_option("rs_fmt", "f16")
    y16 = _run(lib, x, w, kw, H, W, 1)
    ops.set_option("rs_fmt", "bf16")
    y, stats = _run(lib, x, w, kw, H, W, 1, want_stats=True)
    torch.cuda.synchronize()
    assert _rel(y16, ref) <= 4e-6
    assert _rel(y, ref) <= 4e-5
    assert _rel(stats, ops.instnorm_stats(ref)) <= 1e-4


@pytest.mark.parametrize("cin,cout", CHANNELS, ids=[f"{a}to{b}" for a, b in CHANNELS])
def test_conv_rs_kernel_is_the_route(lib, cin, cout):
    """the launches above really run conv_rs_kernel with rs_kernel = 1, and conv_tc_kernel with rs_kernel = 0 or the fp16 split"""
    from torch.profiler import ProfilerActivity, profile
    from vtoonify_b200 import ops
    H, W = 16, 64
    x, w, kw = _case(1, cin, cout, H, W, 1, seed=1)

    def kernels(route, fmt="bf16"):
        ops.set_option("rs_fmt", fmt)
        _run(lib, x, w, kw, H, W, route)   # split weights and module load outside the trace
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _run(lib, x, w, kw, H, W, route)
            torch.cuda.synchronize()
        return " ".join(e.name for e in prof.events())

    new, old, f16 = kernels(1), kernels(0), kernels(1, "f16")
    ops.set_option("rs_fmt", "bf16")
    assert "conv_rs_kernel" in new and "conv_tc_kernel" not in new
    assert "conv_tc_kernel" in old and "conv_rs_kernel" not in old
    assert "conv_tc_kernel" in f16 and "conv_rs_kernel" not in f16
