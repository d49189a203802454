"""conv_rs_kernel (the row-strip layers with output channels on the wgmma M and pixels on N) is the kernel vt_conv2d_rs runs, and
option rs_kernel = 0 or the fp16 split sends the same launch to conv_tc_kernel, for every Cin / Cout in {32, 64}.  The results
of both kernels are checked against float64 in test_gpu_conv_rs_plans.py."""
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


CHANNELS = [(32, 32), (32, 64), (64, 32), (64, 64)]


@pytest.mark.parametrize("cin,cout", CHANNELS, ids=[f"{a}to{b}" for a, b in CHANNELS])
def test_conv_rs_kernel_is_the_route(lib, cin, cout):
    """a 16 x 64 launch really runs conv_rs_kernel with rs_kernel = 1, and conv_tc_kernel with rs_kernel = 0 or the fp16 split"""
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
