"""Row-strip up-convolution entry point (ops.conv_up2_rs_nhwc: Blur o conv_transpose2d as one convolution over the 4 output
phases) against the fp32 polyphase transposed conv + FIR pass and the folded route."""
import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture()
def knobs():
    from vtoonify_b200 import _lib, ops
    lib = _lib.load()
    old = {k: ops.get_option(k) for k in ("rs_min_width", "rs_fmt", "rsu_conv")}
    ops.set_option("rs_min_width", 1)
    old_t = lib.vt_set_option(b"tc_transpose", 1)
    assert old_t != -1
    yield lib
    for k, v in old.items():
        ops.set_option(k, v)
    lib.vt_set_option(b"tc_transpose", old_t)


def _blur():
    k1 = torch.tensor([1., 3., 3., 1.])
    return (k1[:, None] * k1[None, :] / 64 * 4).cuda()


def _case(B, Cin, Cout, H, W, wB, seed, noise):
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, H, W, Cin), generator=g).cuda()
    wt = (torch.randn((wB, Cout, Cin, 3, 3), generator=g) / (3 * Cin ** 0.5)).cuda()
    w9 = torch.cat([ops.prep_weights(wt[i], cin_pad=Cin, round_tf32=False) for i in range(wB)], dim=0).contiguous()
    kw = dict(bias=(torch.randn(Cout, generator=g) * 0.2).cuda(), act=1, slope=0.2, gain=2 ** 0.5)
    if noise:
        kw["noise"] = torch.randn((B, 1, 2 * H, 2 * W), generator=g).cuda().contiguous()
        kw["noise_w"] = torch.tensor([0.3]).cuda()
    return x, w9, kw


CASES = [
    # B, Cin, Cout, H, W, wB
    (1, 64, 32, 12, 128, 1),
    (1, 64, 32, 11, 100, 1),        # ragged in x and y
    (2, 64, 32, 9, 260, 2),         # per-sample weights
    (1, 128, 64, 10, 140, 1),       # N = 4 x 64 (two 128-wide N tiles, or one wide item), 4 K chunks
    (2, 128, 64, 7, 300, 1),
    (1, 32, 32, 5, 130, 1),
    (1, 64, 96, 6, 256, 1),         # N = 4 x 96: 128-wide N tiles across phase boundaries
]


@pytest.mark.parametrize("case", CASES, ids=[f"rsu{i}" for i in range(len(CASES))])
@pytest.mark.parametrize("fmt,tol", [("bf16", 5e-5), ("f16", 6e-6)])
@pytest.mark.parametrize("transpose", [0, 2], ids=["T0", "T2"])   # the kernel's view of the phase outputs as is / transposed (x <-> y)
def test_rsu_vs_fp32(knobs, case, fmt, tol, transpose):
    from vtoonify_b200 import ops
    B, Cin, Cout, H, W, wB = case
    lib = knobs
    assert lib.vt_set_option(b"tc_transpose", transpose) != -1
    ops.set_option("rs_fmt", fmt)
    K = _blur()
    x, w9, kw = _case(B, Cin, Cout, H, W, wB, seed=B * 100 + H, noise=(H % 2 == 1))
    t = ops.conv_transpose2d_s2_k3_nhwc(x, w9, precision="fp32")
    ref = ops.fir_nhwc(t, K, (1, 1), bias=kw["bias"], noise=kw.get("noise"), noise_w=kw.get("noise_w"), act=True, slope=0.2, gain=2 ** 0.5)
    y = ops.conv_up2_rs_nhwc(x, w9, K, **kw)
    torch.cuda.synchronize()
    assert tuple(y.shape) == (B, 2 * H, 2 * W, Cout)
    scale = ref.abs().max().item()
    err = (y - ref).abs().max().item()
    print(f"conv_rsu {case} [{fmt}, T {transpose}]: max|err| {err:.3e} (max|ref| {scale:.2f})")
    assert err <= tol * scale, f"{err:.3e} > {tol} * {scale:.2f}"


def test_rsu_module_routing_and_batch_independence(knobs):
    """StyledConv(upsample=True) takes the row-strip kernel when eligible; same result as the folded kernel; frames independent"""
    from vtoonify_b200 import ops
    from vtoonify_b200.stylegan import StyledConv
    from vtoonify_b200.weights import det_state_dict
    m = StyledConv(64, 32, 3, 512, upsample=True).eval()
    m.load_state_dict(det_state_dict(m, seed=4), strict=True)
    m.cuda()
    g = torch.Generator().manual_seed(2)
    x = torch.randn((3, 10, 264, 64), generator=g).cuda()
    style = torch.randn((3, 512), generator=g).cuda()
    noise = torch.randn((3, 1, 20, 528), generator=g).cuda()
    ops.set_option("rsu_conv", True)
    a = m.forward_nhwc(x, style, noise=noise)
    a1 = m.forward_nhwc(x[1:2].contiguous(), style[1:2], noise=noise[1:2].contiguous())
    ops.set_option("rsu_conv", False)
    b = m.forward_nhwc(x, style, noise=noise)
    assert (a - b).abs().max().item() <= 8e-5 * b.abs().max().item()
    assert torch.equal(a[1:2], a1), "a frame's result must not depend on the batch it travels in"
