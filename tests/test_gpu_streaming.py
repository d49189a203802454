"""GPU: the streaming kernels of csrc/elementwise.cu that nothing else checks directly, against float64 (and bit for bit where
the kernel's arithmetic is one fp32 rounding):

* ``ops.gate_shortcut_add``: x * gate[b, c] + sc[b, s*y, s*x, c] (pSp's SE block and strided shortcut, BiSeNet's attention);
* ``ops.bilinear_add``: F.interpolate(x, (H, W), mode='bilinear', align_corners=True) + y (pSp's FPN _upsample_add);
* ``ops.axpby``: a * sa + b * sb (ToRGB skip, DualStyleGAN's style blend, encoder residuals, the frame loop's parsing copy).

In the tf32 precision mode each output is the fp32 output rounded by cvt.rna.tf32, bit for bit.  u = 2^-24.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_weight_prep_host import bits, rna_tf32

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

U = 2.0 ** -24


class precision:
    def __init__(self, p):
        self.p = p

    def __enter__(self):
        from vtoonify_b200 import ops
        self.old = ops.set_precision(self.p)

    def __exit__(self, *exc):
        from vtoonify_b200 import ops
        ops.set_precision(self.old)


def report(got, ref, bar, what):
    err = (got.double() - ref).abs()
    ratio = (err / bar.clamp_min(1e-300)).max().item()
    print(f"{what}: max err {err.max().item():.2e}, max err/bar {ratio:.3f}")
    assert (err <= bar).all(), f"{what}: {ratio:.2f} x the bar"


# ---- gate_shortcut_add -----------------------------------------------------------------------------------------------------------
# (B, H, W, C, sc_stride, Hs, Ws, gate): odd H and W with Hs = 2H - 1 and 2H; the last map has H*W*C/4 = 1M float4 per sample,
# above the grid cap of 16 blocks of 256 per SM (540672 threads on 132 SMs), so the stride loop runs
GATE_CASES = [(2, 7, 9, 4, 1, 7, 9, True), (2, 7, 9, 516, 2, 13, 17, True), (3, 5, 11, 4, 2, 10, 22, False),
              (2, 9, 5, 516, 2, 18, 9, False), (2, 128, 128, 256, 2, 256, 256, True)]


@pytest.mark.parametrize("case", GATE_CASES, ids=lambda c: "x".join(map(str, c[:7])) + ("-gate" if c[7] else "-nogate"))
def test_gate_shortcut_add_vs_float64(case):
    """with a gate: fl(fl(x g) + s) or fma(x, g, s), so |err| <= u |x g| + u |x g + s| <= 2u (|x g| + |s|); without: one fp32
    add, bit for bit against torch"""
    from vtoonify_b200 import ops
    B, H, W, C, st, Hs, Ws, has_gate = case
    g = torch.Generator().manual_seed(H * W + C)
    x = torch.randn((B, H, W, C), generator=g).cuda()
    sc = torch.randn((B, Hs, Ws, C), generator=g).cuda()
    gate = torch.rand((B, C), generator=g).cuda() if has_gate else None
    with precision("fp32"):
        got = ops.gate_shortcut_add(x, gate, sc, st)
    with precision("tf32"):
        got_r = ops.gate_shortcut_add(x, gate, sc, st)
    s = sc[:, ::st, ::st][:, :H, :W]
    if has_gate:
        xg = x.double() * gate.double()[:, None, None, :]
        report(got, xg + s.double(), 2 * U * (xg.abs() + s.double().abs()), f"gate_shortcut_add {case}")
    else:
        assert torch.equal(bits(got), bits(x + s))
    assert torch.equal(bits(got_r), bits(rna_tf32(got)))


# ---- bilinear_add ---------------------------------------------------------------------------------------------------------------
# (B, h, w, H, W, C)
BILINEAR_CASES = [(1, 16, 16, 32, 32, 512), (1, 32, 32, 64, 64, 512),      # pSp's FPN
                  (2, 9, 7, 9, 7, 8),                                       # identity
                  (2, 1, 1, 5, 6, 4), (2, 5, 6, 1, 1, 4),                   # 1 -> N and N -> 1
                  (2, 1, 7, 4, 13, 4),                                      # h = 1, w > 1
                  (2, 7, 7, 13, 13, 12), (2, 13, 13, 7, 7, 12), (2, 7, 13, 13, 7, 8),   # non-integer ratios
                  (1, 64, 64, 128, 128, 256)]                               # above the grid cap: the stride loop runs
EXACT = {(2, 9, 7, 9, 7, 8), (2, 1, 1, 5, 6, 4), (2, 5, 6, 1, 1, 4)}        # source coordinates are integers


@pytest.mark.parametrize("case", BILINEAR_CASES, ids=lambda c: "x".join(map(str, c)))
def test_bilinear_add_vs_float64(case):
    """Bar: the kernel computes the source coordinate as fl(o * fl((h - 1) / (H - 1))), within 2u (h - 1) of the exact one per axis;
    the interpolant's slope is at most 2 max|x|, so the coordinates cost <= 4u max|x| (h + w - 2).  The weights
    (1 - l)(1 - l') carry <= 3u, the 4 products and 4 adds (fused or not) and the add of y <= 5u of max|x| + |y|:
    |err| <= 8u (max|x| + |y|) + 4u max|x| (h + w - 2).  Where every source coordinate is an integer (identity, 1 -> N, N -> 1)
    the weights are exactly 1 and 0 and the output is one fp32 add, bit for bit."""
    from vtoonify_b200 import ops
    B, h, w, H, W, C = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn((B, h, w, C), generator=g).cuda()
    y = torch.randn((B, H, W, C), generator=g).cuda()
    with precision("fp32"):
        got = ops.bilinear_add(x, y)
    with precision("tf32"):
        got_r = ops.bilinear_add(x, y)
    up = F.interpolate(x.double().permute(0, 3, 1, 2), size=(H, W), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    ref = up + y.double()
    M = x.abs().max().item()
    bar = 8 * U * (M + y.double().abs()) + 4 * U * M * (h + w - 2)
    report(got, ref, bar, f"bilinear_add {case}")
    if case in EXACT:
        assert torch.equal(bits(got), bits(up.float() + y))
    assert torch.equal(bits(got_r), bits(rna_tf32(got)))


# ---- axpby ----------------------------------------------------------------------------------------------------------------------
SCALES = [(1 / 16, 0.0), (-1.0, 1 / 16), (0.0, -1.0), (1.0, 1.0), (2 ** -0.5, 2 ** -0.5), (0.7, -1.3)]


@pytest.mark.parametrize("n", [0, 1, 5, (1 << 22) + 3])
@pytest.mark.parametrize("with_b", [True, False])
@pytest.mark.parametrize("scales", SCALES, ids=lambda s: f"{s[0]:.3g},{s[1]:.3g}")
def test_axpby_vs_float64(n, with_b, scales):
    """a * sa + b * sb.  With sa, sb in {0, +-1, 1/16} both products are exact and the output is one rounding of their sum: bit
    for bit against torch.  Otherwise fl(fl(a sa) + fl(b sb)) or fma: |err| <= 2u (|a sa| + |b sb|).  n = (1 << 22) + 3 runs the
    capped grid's stride loop and a tail."""
    from vtoonify_b200 import ops
    sa, sb = scales
    g = torch.Generator().manual_seed(n + int(with_b))
    a = torch.randn(n, generator=g).cuda()
    b = torch.randn(n, generator=g).cuda() if with_b else None
    with precision("fp32"):
        got = ops.axpby(a, b, sa, sb)
    with precision("tf32"):
        got_r = ops.axpby(a, b, sa, sb)
    got_rr = ops.axpby(a, b, sa, sb, round_tf32=True)
    assert got.shape == a.shape
    exact = all(s in (0.0, 1.0, -1.0, 1 / 16) for s in scales)
    ta = a * sa
    ref32 = ta + b * sb if with_b else ta
    fa, fb = (float(torch.tensor(s, dtype=torch.float32)) for s in scales)     # the scales as the kernel receives them
    ref = a.double() * fa + (b.double() * fb if with_b else 0.0)
    bar = 2 * U * (a.double().abs() * abs(fa) + (b.double().abs() * abs(fb) if with_b else 0.0))
    if n:
        report(got, ref, bar, f"axpby n={n} b={with_b} sa={sa:.3g} sb={sb:.3g}")
    if exact or not with_b:
        assert torch.equal(bits(got), bits(ref32))
    assert torch.equal(bits(got_r), bits(rna_tf32(got)))
    assert torch.equal(bits(got_rr), bits(got_r))


def test_axpby_into_a_channel_slice():
    """frame_loop: the parsing logits / 16 written straight into channels 3: of the encoder's input x[b]; channels 0..2 and the
    other sample are untouched"""
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(5)
    p = torch.randn((2, 19, 13, 17), generator=g).cuda()
    x = torch.full((2, 22, 13, 17), float("nan"), device="cuda")
    with precision("fp32"):
        ops.axpby(p[1], None, 1.0 / 16.0, out=x[1, 3:])
    assert torch.equal(bits(x[1, 3:]), bits(p[1] / 16))
    assert torch.isnan(x[1, :3]).all() and torch.isnan(x[0]).all()
