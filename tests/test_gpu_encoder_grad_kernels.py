"""GPU: the two kernels of the encoder backward (ops.adain_grad_stats + ops.act_grad) against float64 autograd of
F.instance_norm + affine on the plane families of test_gpu_norm_stats.py, the fused bias-gradient sums against float64 channel
sums, and bit-identical reruns."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (mean, spread) of the planes; None: a constant plane with one outlier
FAMILIES = {"unit": (0.0, 1.0), "offset": (1e4, 1.0), "near_const": (12.1, 1e-3), "outlier": None}
SHAPES = [(1, 32, 32, 512), (8, 32, 32, 512), (8, 64, 64, 32), (1, 256, 256, 32)]   # (B, H, W, C)
# relative L2 / max|err| over max|ref| bars of the AdaIN backward against exact float64.  The kernels work from the fp32 (mean,
# rstd) table the forward applied; on the offset and near-constant planes that mean is off by up to half an ulp of the plane's
# level (5e-4 of the spread), which moves xhat by that much and the gradient by about that over sqrt(HW)
BARS = {"unit": (1e-5, 1e-4), "offset": (1e-4, 1e-3), "near_const": (1e-4, 1e-3), "outlier": (1e-5, 1e-4)}


def planes(kind, B, H, W, C, g):
    if FAMILIES[kind] is None:
        x = torch.full((B, H, W, C), 3.0, device="cuda")
        x[:, H // 2, W // 3, :] = 7.0
        return x
    mean, spread = FAMILIES[kind]
    return (mean + spread * torch.randn((B, H, W, C), generator=g, device="cuda")).float()


def errs(got, ref):
    d = (got.double() - ref).flatten()
    return (d.norm() / ref.norm()).item(), (d.abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize("kind", list(FAMILIES))
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_adain_backward_vs_float64(kind, shape):
    from vtoonify_b200 import ops
    B, H, W, C = shape
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H + C)
    x = planes(kind, B, H, W, C, g)
    gr = torch.randn((B, H, W, C), generator=g, device="cuda")
    ref_act = torch.randn((B, H, W, C), generator=g, device="cuda")
    res = torch.randn((B, H, W, C), generator=g, device="cuda")
    gb = torch.cat([1.0 + 0.3 * torch.randn((B, C), generator=g, device="cuda"),
                    0.1 * torch.randn((B, C), generator=g, device="cuda")], 1).contiguous()
    stats = ops.instnorm_stats(x)
    sums = ops.adain_grad_stats(gr, x, stats)
    # float64 autograd of gamma * instance_norm(x) + beta, NCHW
    x64 = x.double().permute(0, 3, 1, 2).requires_grad_()
    with torch.enable_grad():
        y = gb[:, :C, None, None].double() * F.instance_norm(x64, eps=1e-5) + gb[:, C:, None, None].double()
        y.backward(gr.double().permute(0, 3, 1, 2))
    t_ref = x64.grad.permute(0, 2, 3, 1)
    # the sums are those of the function the forward applied: xhat from the saved statistics, in float64
    st = stats.double()
    xh = (x.double() - st[:, None, None, :, 0]) * st[:, None, None, :, 1]
    sums_ref = torch.stack([gr.double().sum((1, 2)), (gr.double() * xh).sum((1, 2))], -1)
    e_s = errs(sums, sums_ref)
    print(f"\n{kind} {shape}: sums (dbeta, dgamma) rel L2 {e_s[0]:.2e} max {e_s[1]:.2e}")
    assert e_s[0] <= 1e-6 and e_s[1] <= 1e-5
    for gate in (False, True):
        for with_res in (False, True):
            out = ops.act_grad(gr, ref=ref_act if gate else None, slope=0.2, gain=1.5, res=res if with_res else None, beta=0.7,
                               adain=(x, stats, gb, sums))
            want = t_ref * 1.5
            if gate:
                want = torch.where(ref_act > 0, want, want * 0.2)
            if with_res:
                want = want + 0.7 * res.double()
            e = errs(out, want)
            print(f"  gate={gate} res={with_res}: rel L2 {e[0]:.2e}, max|err|/max|ref| {e[1]:.2e}")
            assert e[0] <= BARS[kind][0] and e[1] <= BARS[kind][1]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_act_grad_bias_sums_and_reruns(shape):
    from vtoonify_b200 import ops
    B, H, W, C = shape
    g = torch.Generator(device="cuda").manual_seed(7 + C)
    gr = torch.randn((B, H, W, C), generator=g, device="cuda")
    ref_act = torch.randn((B, H, W, C), generator=g, device="cuda")
    out, bg = ops.act_grad(gr, ref=ref_act, slope=0.2, gain=0.5, bias_grad=True)
    want = torch.where(ref_act > 0, gr, gr * 0.2) * 0.5
    assert torch.equal(out, want.float()) or (out - want).abs().max().item() <= 1e-7
    bg_ref = out.double().sum((0, 1, 2))
    e = ((bg.double() - bg_ref).abs() / out.double().abs().sum((0, 1, 2))).max().item()
    print(f"\n{shape}: bias-gradient sum error / sum of |terms| {e:.2e}")
    assert e <= 1e-7
    out2, bg2 = ops.act_grad(gr, ref=ref_act, slope=0.2, gain=0.5, bias_grad=True)
    assert torch.equal(out, out2) and torch.equal(bg, bg2)
    x = planes("offset", B, H, W, C, g)
    stats = ops.instnorm_stats(x)
    s1, s2 = ops.adain_grad_stats(gr, x, stats), ops.adain_grad_stats(gr, x, stats)
    assert torch.equal(s1, s2)


def test_act_grad_rejects_bad_shapes():
    from vtoonify_b200 import ops
    from vtoonify_b200._lib import VtError
    g = torch.zeros((1, 4, 4, 6), device="cuda")
    with pytest.raises(VtError):
        ops.act_grad(g)
    with pytest.raises(VtError):
        ops.act_grad(torch.zeros((1, 4, 4, 8), device="cuda"), ref=torch.zeros((1, 4, 4, 4), device="cuda"))
