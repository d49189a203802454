"""CPU: calibration of the error bars in tests/wgrad_bounds.py.  The float64 weight-gradient reduction agrees with PyTorch's
own; a float32 emulation of the weight-gradient kernel's arithmetic passes both bars with at least 4x headroom at the largest K
of the GPU suite; the statistical bar rejects each of six ways of breaking that emulation; and the GPU case list reaches every
choice of the kernel's planner."""
import pytest
import torch
import torch.nn.functional as F

from tests import wgrad_bounds as WB
from tests.test_gpu_conv_wgrad import CASES, assert_plan_coverage, case, case_data, host_ws_floats, k, largest_k_case, plan_of

HEADROOM = 4.0


def _small(c, M=8, N=8):
    """a case with its geometry and plan but few channels (the error of an element depends on K, not on M or N)"""
    return dict(c, M=min(M, c["M"]), N=min(N, c["N"]))


def _emulate(c, a, s, mutation=None):
    p = plan_of(c)
    return WB.emulate_wgrad(a, s, c["taps"], c["stride"], c["ps"], p["splits"], p["box_w"], mutation)


def _ratios(y, a, s, c):
    y64, E, R = WB.bounds(lambda u, v: WB.wgrad(u, v, c["taps"], c["stride"], c["ps"]), a, s)
    err = (y.double() - y64).abs()
    live = E > 0
    assert torch.equal(y[~live], torch.zeros_like(y[~live]))
    return (err[live] / (WB.C_E * E[live])).max().item(), (err[live] / (WB.C_R * R[live])).max().item()


@pytest.mark.parametrize("stride,pad,dil,per_sample", [(1, 1, 1, False), (2, 0, 1, False), (2, 1, 2, False), (1, 2, 1, True),
                                                       (2, 1, 1, True)])
def test_reference_matches_torch_weight_gradient(stride, pad, dil, per_sample):
    """wgrad() with taps (ky dil - pad, kx dil - pad) is torch's conv2d weight gradient (per sample: the groups = batch form)"""
    g = torch.Generator().manual_seed(0)
    B, Cin, Cout, H, W, kh, kw = 3, 5, 4, 13, 10, 3, 3
    x = torch.randn((B, Cin, H, W), generator=g, dtype=torch.float64)
    w = torch.randn((Cout, Cin, kh, kw), generator=g, dtype=torch.float64)
    taps = k(kh, kw, pad, dil)
    if per_sample:
        xw = x.reshape(1, B * Cin, H, W)
        go = torch.randn(F.conv2d(xw, w.repeat(B, 1, 1, 1), stride=stride, padding=pad, dilation=dil, groups=B).shape,
                         generator=g, dtype=torch.float64)
        ref = torch.nn.grad.conv2d_weight(xw, (B * Cout, Cin, kh, kw), go, stride=stride, padding=pad, dilation=dil, groups=B)
        a = go.reshape(B, Cout, *go.shape[2:])
    else:
        go = torch.randn(F.conv2d(x, w, stride=stride, padding=pad, dilation=dil).shape, generator=g, dtype=torch.float64)
        ref = torch.nn.grad.conv2d_weight(x, (Cout, Cin, kh, kw), go, stride=stride, padding=pad, dilation=dil)
        a = go
    y = WB.wgrad(a, x, taps, stride, per_sample).reshape(ref.shape)
    assert torch.allclose(y, ref, rtol=1e-12, atol=1e-12)


def test_emulation_matches_reference_without_rounding():
    """with operands exact in bf16 and small integer values every sum is exact: the emulation's index arithmetic (boxes, parity
    views, splits) is the reference's"""
    for c in (largest_k_case(), case("s2", 2, 8, 8, 9, 11, k(5, 5, 2), stride=2, sh=18, sw=22),
              case("ps", 3, 8, 8, 13, 18, k(3, 3, 1), ps=1), case("box8", 2, 8, 8, 17, 8, k(5, 5, 2))):
        c = _small(c, 4, 4)
        g = torch.Generator().manual_seed(1)
        a = torch.randint(-3, 4, (c["B"], c["M"], c["ah"], c["aw"]), generator=g).float()
        s = torch.randint(-3, 4, (c["B"], c["N"], c["sh"], c["sw"]), generator=g).float()
        y = _emulate(c, a, s)
        assert torch.equal(y.double(), WB.wgrad(a.double(), s.double(), c["taps"], c["stride"], c["ps"])), c["name"]


@pytest.mark.parametrize("data", ["randn", "positive", "scales", "loud", "both_positive"])
def test_emulation_headroom_at_largest_k(data):
    """the kernel's arithmetic stays within a quarter of both bars at the largest K of the GPU suite"""
    c = dict(_small(largest_k_case()), data="positive" if data == "both_positive" else data)
    a, s = case_data(c, 7)
    if data == "both_positive":
        a = 4.0 + 0.25 * a.clamp(-3, 3)
    hard, stat = _ratios(_emulate(c, a, s), a, s, c)
    print(f"{c['name']} K steps {plan_of(c)['ksteps']} splits {plan_of(c)['splits']} [{data}]: worst err/bound hard {hard:.3g} "
          f"statistical {stat:.3g}")
    assert hard * HEADROOM <= 1 and stat * HEADROOM <= 1


def test_emulation_headroom_over_the_case_list():
    worst = [0.0, 0.0]
    for c in CASES:
        c = _small(c, 4, 4)
        a, s = case_data(c, 8)
        r = _ratios(_emulate(c, a, s), a, s, c)
        worst = [max(w, v) for w, v in zip(worst, r)]
    print(f"every case, 4 x 4 channels: worst err/bound hard {worst[0]:.3g} statistical {worst[1]:.3g}")
    assert worst[0] * HEADROOM <= 1 and worst[1] * HEADROOM <= 1


MUTATION_CASES = [largest_k_case(), case("s2_shared", 2, 64, 64, 16, 16, k(3, 3, 1), stride=2, sh=32, sw=32)]


@pytest.mark.parametrize("mutation", WB.MUTATIONS)
@pytest.mark.parametrize("c", MUTATION_CASES, ids=lambda c: c["name"])
def test_statistical_bar_rejects_mutation(mutation, c):
    if mutation == "wrong_parity" and c["stride"] != 2:
        pytest.skip("parity views exist at stride 2 only")
    c = _small(c)
    a, s = case_data(c, 9)
    _, stat = _ratios(_emulate(c, a, s, mutation), a, s, c)
    print(f"{c['name']} mutation {mutation}: worst statistical err/bound {stat:.3g}")
    assert stat > 1, f"the statistical bar does not see mutation {mutation} ({stat:.3g})"


def test_case_list_reaches_every_plan():
    assert_plan_coverage(CASES, host_ws_floats)
