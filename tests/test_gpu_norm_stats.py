"""GPU: instance-norm statistics against float64 statistics of the same fp32 tensor, on the planes where a (sum, sum of squares)
reduction cancels: means far from zero next to the spread (mean/std up to 1e4), near-constant and constant planes at values
that are not dyadic, all-zero planes, and planes whose only deviation is one spike at the first or the last pixel.

Producers: the standalone pass (vt_instnorm_stats_nhwc, both modes, every chunk plan) and the epilogue of the tensor-core
convolution (conv2d_nhwc(want_stats=True), every kernel form that can write statistics).  Consumers: the ModRes block on the
fused and the unfused AdaIN route, the Fusion mask conv with the AdaIN folded into its weights, and adain_apply.  Also
channel_sum, the other deterministic reduction, against float64.

Bars (eps = 1e-5, statistics of the fp32 tensor in float64):
  mean          |err| <= 1e-6 * (|mean| + std)
  rstd          |err| / rstd <= 1e-5
  normalised    |err| <= 1e-5 * max(1, max|ref|) + 2^-22 * |gamma| * |mean| * rstd per channel: the second term is the rounding of
                the stored fp32 mean, which no algorithm avoids; through a conv it is weighted by |w| and summed over the inputs.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

EPS = 1e-5
MEAN_TOL = 1e-6
RSTD_TOL = 1e-5
OUT_TOL = 1e-5
BF16X3_TOL = 3e-5     # max-abs error of a bf16x3 convolution relative to max(1, |ref|max), as in test_gpu_conv.py
U22 = 2.0 ** -22

# (name, mean, std, kind): kind "n" = mean + std * N(0, 1), "c" = constant, "s0" / "s1" = constant plus 1.0 at the first / last pixel
PLANES = [("m0", 0.0, 1.0, "n"), ("m1", 1.0, 1.0, "n"), ("m10", 10.0, 1.0, "n"), ("m100", 100.0, 1.0, "n"),
          ("m1e3", 1e3, 1.0, "n"), ("m1e4", 1e4, 1.0, "n"), ("-100/0.5", -100.0, 0.5, "n"), ("5.0/1e-2", 5.0, 1e-2, "n"),
          ("12.1/1e-3", 12.1, 1e-3, "n"), ("5.3/1e-4", 5.3, 1e-4, "n"), ("-2.9/1e-4", -2.9, 1e-4, "n"), ("c5.3", 5.3, 0.0, "c"),
          ("c-2.9", -2.9, 0.0, "c"), ("c12.1", 12.1, 0.0, "c"), ("zero", 0.0, 0.0, "c"), ("spike0", 5.3, 0.0, "s0"),
          ("spike-last", -2.9, 0.0, "s1")]


def planes(B, C, HW, seed, shift=0):
    """fp32 [B, C, HW]: plane (b, c) follows PLANES[(b * C + c + shift) % len(PLANES)]; returns (tensor, plane names)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, C, HW), generator=g, dtype=torch.float64)
    names = []
    for b in range(B):
        for c in range(C):
            name, m, s, kind = PLANES[(b * C + c + shift) % len(PLANES)]
            names.append(name)
            x[b, c] = m + s * x[b, c] if kind == "n" else m
            if kind == "s0":
                x[b, c, 0] += 1.0
            elif kind == "s1":
                x[b, c, -1] += 1.0
    return x.float(), names


def cat_names(names, names2, B, C):
    """plane names of cat(x, |x - x2|) [B, 2C] from the names of x and of x - x2, both [B, C]"""
    return [n for b in range(B) for n in names[b * C:(b + 1) * C] + ["|d|:" + m for m in names2[b * C:(b + 1) * C]]]


def ref_stats(x):
    """float64 (mean, std, rstd) per plane of an fp32 [B, C, ...] tensor"""
    xd = x.double().flatten(2)
    mean = xd.mean(dim=2)
    var = xd.var(dim=2, unbiased=False)
    return mean, var.sqrt(), 1.0 / torch.sqrt(var + EPS)


def check_stats(st, x, names, what):
    """st [B, C, 2] (mean, rstd) from a kernel against float64 statistics of the fp32 tensor x [B, C, H, W] (any device)"""
    mean, std, rstd = ref_stats(x.to(st.device))
    st = st.double()
    merr = (st[:, :, 0] - mean).abs() / (mean.abs() + std).clamp_min(1e-30)
    merr = torch.where((st[:, :, 0] - mean).abs() == 0, torch.zeros_like(merr), merr)
    rerr = ((st[:, :, 1] - rstd) / rstd).abs()
    worst = {}
    for i, n in enumerate(names):
        b, c = divmod(i, mean.shape[1])
        worst[n] = max(worst.get(n, 0.0), rerr[b, c].item())
    print(f"{what}: mean err/(|mean|+std) max {merr.max().item():.2e}, rstd rel err max {rerr.max().item():.2e}; per plane "
          + " ".join(f"{n}={e:.1e}" for n, e in worst.items()))
    assert merr.max().item() <= MEAN_TOL, f"{what}: mean error {merr.max().item():.3e} > {MEAN_TOL}"
    assert rerr.max().item() <= RSTD_TOL, f"{what}: rstd relative error {rerr.max().item():.3e} > {RSTD_TOL}"


@pytest.fixture(scope="module")
def lib():
    from vtoonify_b200 import _lib
    return _lib.load()


def under(lib, **opts):
    """context manager setting library options, restoring them afterwards"""
    class _Opts:
        def __enter__(self):
            self.old = {k: lib.vt_set_option(k.encode(), v) for k, v in opts.items()}

        def __exit__(self, *exc):
            for k, v in self.old.items():
                lib.vt_set_option(k.encode(), v)
    return _Opts()


# ---- the standalone pass ----------------------------------------------------------------------------------------------------
STATS_SHAPES = [(4, 72, 128, 512),      # the ModRes / Fusion maps of VToonify-D at 576 x 1024 (x / 8)
                (1, 288, 512, 128),     # a large map: ~2 chunks per SM under the default plan
                (2, 37, 61, 64),        # HW not a multiple of any chunk
                (1, 33, 50, 1024),      # one pixel lane per chunk
                (3, 4, 4, 12),          # smaller than one chunk, C / 4 not a power of two
                (6, 1, 7, 4),           # 1 x 7 map, C = 4
                (1, 9, 11, 64)]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("shape", STATS_SHAPES)
def test_instnorm_stats_vs_float64(lib, shape, mode):
    """ops.instnorm_stats (mode 0: x; mode 1: cat(x, |x - x2|) with x2 = x - d, d from the plane table, so |x - x2| is
    near-constant where d is) under every chunk plan; bit-identical across runs and a sample's statistics do not depend on
    its batch."""
    from vtoonify_b200 import ops
    B, H, W, C = shape
    x, names = planes(B, C, H * W, seed=H * W + C)
    xs = x.view(B, C, H, W)
    xn = ops.to_nhwc(xs.cuda(), round_tf32=False)
    x2n, ref, ref_names = None, xs, names
    if mode:
        d, dn = planes(B, C, H * W, seed=H * W + C + 1, shift=5)
        x2 = (x - d).view(B, C, H, W)
        x2n = ops.to_nhwc(x2.cuda(), round_tf32=False)
        ref = torch.cat([xs, (xs - x2).abs()], dim=1)   # |x - x2| in fp32, the tensor the kernel normalises
        ref_names = cat_names(names, dn, B, C)
    for plan in (0, 296, 7):
        with under(lib, instnorm_chunks=plan):
            st = ops.instnorm_stats(xn, x2n)
            check_stats(st, ref, ref_names, f"instnorm_stats mode {mode} {shape} plan {plan}")
            assert torch.equal(st, ops.instnorm_stats(xn, x2n)), "not bit-reproducible"
            if B > 1:
                one = ops.instnorm_stats(xn[1:2].contiguous(), None if x2n is None else x2n[1:2].contiguous())
                assert torch.equal(one, st[1:2]), "statistics of a sample depend on its batch"


@pytest.mark.parametrize("mode", [0, 1])
def test_instnorm_stats_channel_stride(lib, mode):
    """vt_instnorm_stats_nhwc with c_stride > C (a channel slice of a wider NHWC tensor): the other channels are never read."""
    from vtoonify_b200 import ops
    B, H, W, C, Cp = 2, 23, 41, 64, 96
    x, names = planes(B, C, H * W, seed=7)
    d, dn = planes(B, C, H * W, seed=8, shift=3)
    x2 = x - d
    xs, x2s = x.view(B, C, H, W), x2.view(B, C, H, W)
    wide = torch.full((B, H, W, Cp), float("nan"), device="cuda")
    wide2 = torch.full((B, H, W, Cp), float("nan"), device="cuda")
    wide[..., :C] = xs.permute(0, 2, 3, 1).cuda()
    wide2[..., :C] = x2s.permute(0, 2, 3, 1).cuda()
    Cs = 2 * C if mode else C
    st = torch.empty((B, Cs, 2), device="cuda")
    ws = torch.empty((lib.vt_instnorm_ws_bytes(B, H * W, C, mode) // 4,), device="cuda")
    rc = lib.vt_instnorm_stats_nhwc(wide.data_ptr(), wide2.data_ptr() if mode else None, mode, B, H * W, C, Cp, ctypes.c_float(EPS),
                                    st.data_ptr(), ws.data_ptr(), ops._stream())
    assert rc == 0, lib.vt_last_error()
    ref = torch.cat([xs, (xs - x2s).abs()], dim=1) if mode else xs
    check_stats(st, ref, cat_names(names, dn, B, C) if mode else names, f"instnorm_stats c_stride {Cp} mode {mode}")


# ---- statistics from the convolution epilogue -------------------------------------------------------------------------------
def offset_conv_inputs(B, Cin, Cout, H, W, k, seed):
    """Weights and bias that make offset and near-constant output channels on purpose: zero and 1e-4-scaled weight rows next to
    normal ones, biases from the plane table, and a residual with per-channel offsets."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, Cin, H, W), generator=g) * 1.5 + 0.25
    w = torch.randn((Cout, Cin, k, k), generator=g) / np.sqrt(Cin * k * k)
    rows = torch.arange(Cout) % 4
    w[rows == 1] = 0.0
    w[rows == 2] *= 1e-4
    means = torch.tensor([m for _, m, _, _ in PLANES])
    b = means[torch.arange(Cout) % len(means)].float()
    res = torch.randn((B, Cout, H, W), generator=g) * 1e-3 + means[(torch.arange(Cout) * 7) % len(means)].float()[None, :, None, None]
    return x, w, b, res


CONV_CASES = [(2, 64, 512, 19, 45, 3, 1, 1),     # partial tiles in x and y, 512 channels (2 N tiles, or one wide item)
              (2, 512, 512, 24, 40, 3, 2, 2),    # dilation 2, 512 -> 512 (the ModRes layer)
              (3, 32, 64, 9, 7, 3, 1, 1),        # smaller than one tile
              (8, 128, 256, 16, 24, 1, 0, 1),    # batch 8, 1x1
              (1, 64, 32, 13, 21, 3, 1, 1)]      # N = 32 (up to 4 M tiles per work item)
CONV_OPTS = [{}, {"tc_pingpong": 0}, {"tc_pingpong": 2}, {"tc_wide": 0}, {"tc_wide": 1}, {"tc_m_major": 1}, {"tc_transpose": 0},
             {"tc_transpose": 2}, {"tc_mt": 1}, {"tc_mt": 2}, {"tc_mt": 4}]


@pytest.mark.parametrize("opts", CONV_OPTS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()) or "default")
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_epilogue_stats_vs_float64(lib, case, opts):
    """conv2d_nhwc(want_stats=True) against float64 statistics of the output it stored; the output is the one written without
    statistics; bit-identical across runs; a sample's statistics do not depend on its batch; with fuse_stats off the output is
    unchanged and the separate pass meets the same bars."""
    from vtoonify_b200 import _lib, ops
    B, Cin, Cout, H, W, k, pad, dil = case
    x, w, b, res = offset_conv_inputs(B, Cin, Cout, H, W, k, seed=sum(case))
    xn = ops.to_nhwc(x.cuda(), round_tf32=False)
    wp = ops.prep_weights(w.cuda(), cin_pad=Cin)
    resn = ops.to_nhwc(res.cuda(), round_tf32=False)
    taps = ops.conv_taps(k, pad, dil)
    kw = dict(bias=b.cuda(), act=_lib.ACT_NONE, res=resn, alpha=0.7, beta=0.7)
    names = [PLANES[c % len(PLANES)][0] for c in range(Cout)] * B
    ops.set_precision("bf16x3")
    try:
        with under(lib, **opts):
            y0 = ops.conv2d_nhwc([xn], wp, taps, 1, H, W, **kw)
            y, st = ops.conv2d_nhwc([xn], wp, taps, 1, H, W, want_stats=True, **kw)
            assert torch.equal(y, y0)
            check_stats(st, ops.to_nchw(y), names, f"conv epilogue {case} {opts}")
            _, st_again = ops.conv2d_nhwc([xn], wp, taps, 1, H, W, want_stats=True, **kw)
            assert torch.equal(st, st_again), "not bit-reproducible"
            if B > 1:
                _, st1 = ops.conv2d_nhwc([xn[1:2].contiguous()], wp, taps, 1, H, W, want_stats=True,
                                         **{**kw, "res": resn[1:2].contiguous()})
                assert torch.equal(st1, st[1:2]), "statistics of a sample depend on its batch"
            ops.set_option("fuse_stats", False)
            y2, st2 = ops.conv2d_nhwc([xn], wp, taps, 1, H, W, want_stats=True, **kw)
            assert torch.equal(y2, y)
            check_stats(st2, ops.to_nchw(y), names, f"separate pass {case} {opts}")
    finally:
        ops.set_option("fuse_stats", True)
        ops.set_precision(ops.DEFAULT_PRECISION)


# ---- consumers --------------------------------------------------------------------------------------------------------------
def adain64(x, gb):
    """float64 AdaIN of an fp32 NCHW tensor: gamma * (x - mean) * rstd + beta, and the per-channel rounding term of the bar"""
    B, C = x.shape[:2]
    mean, _, rstd = ref_stats(x)
    gamma, beta = gb[:, :C].double(), gb[:, C:].double()
    y = gamma[:, :, None, None] * (x.double() - mean[:, :, None, None]) * rstd[:, :, None, None] + beta[:, :, None, None]
    return y, U22 * gamma.abs() * mean.abs() * rstd          # [B, C]


def style_rows(B, C, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.cat([1.0 + 0.5 * torch.randn((B, C), generator=g), torch.randn((B, C), generator=g)], dim=1).cuda()


@pytest.mark.parametrize("mode", [0, 1])
def test_adain_apply_vs_float64(mode):
    from vtoonify_b200 import ops
    B, C, H, W = 2, 64, 37, 29
    x, _ = planes(B, C, H * W, seed=11)
    d, _ = planes(B, C, H * W, seed=12, shift=4)
    xs, x2s = x.view(B, C, H, W), (x - d).view(B, C, H, W)
    xn, x2n = ops.to_nhwc(xs.cuda(), round_tf32=False), ops.to_nhwc(x2s.cuda(), round_tf32=False)
    ref_in = torch.cat([xs, (xs - x2s).abs()], dim=1) if mode else xs
    gb = style_rows(B, ref_in.shape[1], 13)
    with _fp32():
        y = ops.adain_apply(xn, ops.instnorm_stats(xn, x2n if mode else None), gb, x2n if mode else None)
    ref, term = adain64(ref_in.cuda(), gb)
    err = (ops.to_nchw(y).double() - ref).abs()
    bar = OUT_TOL * max(1.0, ref.abs().max().item()) + term[:, :, None, None]
    print(f"adain_apply mode {mode}: max err {err.max().item():.2e}, max err/bar {(err / bar).max().item():.2f}")
    assert (err <= bar).all()


class _fp32:
    """adain_apply rounds its output to tf32 in the tf32 precision mode only; the bar is for an fp32 output"""
    def __enter__(self):
        from vtoonify_b200 import ops
        self.old = ops._precision
        ops.set_precision("fp32")

    def __exit__(self, *exc):
        from vtoonify_b200 import ops
        ops.set_precision(self.old)


def conv64(h, w, b, dil, res=None, alpha=1.0):
    """float64 ConvLayer (EqualConv2d + FusedLeakyReLU(0.2, sqrt 2)) with v * alpha + res"""
    k = w.shape[-1]
    scale = 1.0 / np.sqrt(w.shape[1] * k * k)
    v = F.leaky_relu(F.conv2d(h, w.double() * scale, padding=dil, dilation=dil) + b.double()[None, :, None, None], 0.2) * np.sqrt(2)
    return v * alpha + (0.0 if res is None else res)


def conv_term(w, term, dil):
    """rounding term of the normalised input carried through the conv: sum over inputs and taps of |w| * term, per output"""
    k = w.shape[-1]
    scale = 1.0 / np.sqrt(w.shape[1] * k * k)
    return np.sqrt(2) * term.double() @ (w.double().abs().sum(dim=(2, 3)) * scale).t()     # [B, Cout]


@pytest.mark.parametrize("fuse", [True, False])
@pytest.mark.parametrize("case", [(2, 64, 19, 45, 1), (2, 512, 16, 24, 2)])
def test_modres_block_vs_float64(case, fuse):
    """AdaResBlock (x + w * conv2(AdaIN(conv(AdaIN(x, s)), s))) on the fused route (adain_affine + src_affine in conv_tc, the
    first conv's epilogue statistics feeding the second AdaIN) and the fuse_adain=False route (instnorm_stats + adain_apply).
    Each stage is checked against float64 of its own fp32 input; the block equals the composition of the stages.  conv's
    weights have zero and 1e-4-scaled rows next to biases far from zero, so its output has offset and near-constant channels."""
    from vtoonify_b200 import ops
    from vtoonify_b200.dualstylegan import AdaResBlock
    B, C, H, W, dil = case
    g = torch.Generator().manual_seed(C + H)
    blk = AdaResBlock(C, 512, dilation=dil)
    w1 = torch.randn((C, C, 3, 3), generator=g)
    rows = torch.arange(C) % 4
    w1[rows == 1] = 0.0
    w1[rows == 2] *= 1e-4
    means = torch.tensor([m for _, m, _, _ in PLANES])
    blk.conv[0].weight.data.copy_(w1)
    blk.conv[1].bias.data.copy_(means[torch.arange(C) % len(means)] / np.sqrt(2))
    blk.conv2[0].weight.data.copy_(torch.randn((C, C, 3, 3), generator=g))
    blk.conv2[1].bias.data.copy_(torch.randn(C, generator=g))
    blk = blk.cuda()
    x, _ = planes(B, C, H * W, seed=C + 1)
    xs = x.view(B, C, H, W).cuda()
    xn = ops.to_nhwc(xs, round_tf32=False)
    s = torch.randn((B, 512), generator=g).cuda()
    gb1, gb2 = blk.norm.gamma_beta(s, B), blk.norm2.gamma_beta(s, B)
    wgt = 0.75
    ops.set_precision("bf16x3")
    ops.set_option("fuse_adain", fuse)
    try:
        y_blk = blk.forward_nhwc(xn, s, wgt)
        if fuse:
            out, st = blk.conv.forward_nhwc(xn, src_affine=blk.norm.affine(xn, s), want_stats=True)
            y = blk.conv2.forward_nhwc(out, src_affine=blk.norm2.affine(out, s, st), res=xn, alpha=wgt, beta=1.0)
        else:
            out = blk.conv.forward_nhwc(blk.norm.forward_nhwc(xn, s))
            h2 = blk.norm2.forward_nhwc(out, s)
            ref_h2, term_h2 = adain64(ops.to_nchw(out), gb2)
            err = (ops.to_nchw(h2).double() - ref_h2).abs()
            bar = OUT_TOL * max(1.0, ref_h2.abs().max().item()) + term_h2[:, :, None, None]
            print(f"ModRes (unfused) AdaIN of conv out: max err/bar {(err / bar).max().item():.2f}")
            assert (err <= bar).all()
            y = blk.conv2.forward_nhwc(h2, res=xn, alpha=wgt, beta=1.0)
            st = ops.instnorm_stats(out)
        assert torch.equal(y, y_blk)
    finally:
        ops.set_option("fuse_adain", True)
        ops.set_precision(ops.DEFAULT_PRECISION)
    outc = ops.to_nchw(out)
    check_stats(st, outc, [PLANES[c % len(PLANES)][0] for c in range(C)] * B, f"ModRes conv output {case} fuse={fuse}")
    h1, term1 = adain64(xs, gb1)
    ref1 = conv64(h1, blk.conv[0].weight, blk.conv[1].bias, dil)
    h2, term2 = adain64(outc, gb2)
    ref2 = conv64(h2, blk.conv2[0].weight, blk.conv2[1].bias, dil, res=xs.double(), alpha=wgt)
    for name, got, ref, w, term in (("conv", outc, ref1, blk.conv[0].weight, term1),
                                    ("conv2", ops.to_nchw(y), ref2, blk.conv2[0].weight, term2)):
        err = (got.double() - ref).abs()
        bar = BF16X3_TOL * max(1.0, ref.abs().max().item()) + conv_term(w, term, dil)[:, :, None, None]
        print(f"ModRes {case} fuse={fuse} {name}: max err {err.max().item():.2e}, max err/bar {(err / bar).max().item():.2f}")
        assert (err <= bar).all(), f"{name}: {(err / bar).max().item():.2f} x the bar"


@pytest.mark.parametrize("shape", [(2, 256, 36, 64), (1, 64, 75, 133)])
def test_fusion_mask_conv_vs_float64(shape):
    """Fusion's mask conv: instnorm_stats(f_G, f_E) -> affine_fold_weights -> smalln_conv(tap_const, src2) against
    F.instance_norm(cat(f_G, |f_G - f_E|)) * gamma + beta then F.conv2d in float64 (model/vtoonify.py:125-127); f_E = f_G - d with d
    from the plane table, so |f_G - f_E| has offset and near-constant channels."""
    from vtoonify_b200 import _lib, ops
    B, C, H, W = shape
    fG, _ = planes(B, C, H * W, seed=C + 3)
    d, _ = planes(B, C, H * W, seed=C + 4, shift=6)
    fGs, fEs = fG.view(B, C, H, W).cuda(), (fG - d).view(B, C, H, W).cuda()
    fGn, fEn = ops.to_nhwc(fGs, round_tf32=False), ops.to_nhwc(fEs, round_tf32=False)
    g = torch.Generator().manual_seed(C)
    w = (torch.randn((1, 2 * C, 3, 3), generator=g) / np.sqrt(2 * C * 9)).cuda()
    b = torch.randn(1, generator=g).cuda()
    gb = style_rows(B, 2 * C, C + 5)
    stats = ops.instnorm_stats(fGn, fEn)
    w_fold, k_fold = ops.affine_fold_weights(ops.prep_weights(w, cin_pad=2 * C, round_tf32=False), stats, gb)
    m = ops.smalln_conv(fGn, w_fold, ops.conv_taps(3, 1), 1, B, H, W, bias=b, act=_lib.ACT_RELU_TANH, src2=fEn, tap_const=k_fold)
    cat = torch.cat([fGs, (fGs - fEs).abs()], dim=1)
    h, term = adain64(cat, gb)
    z = F.conv2d(h, w.double(), b.double(), padding=1)
    ref = torch.tanh(torch.relu(z))
    err = (m.double().view_as(ref) - ref).abs()
    bar = OUT_TOL * max(1.0, z.abs().max().item()) + (term @ w.double().abs().sum(dim=(2, 3)).t())[:, :, None, None]
    print(f"Fusion mask {shape}: max err {err.max().item():.2e}, max err/bar {(err / bar).max().item():.2f}")
    assert (err <= bar).all()


# ---- channel_sum ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(3, 5, 1000), (2, 64, 777), (4, 1, 300), (37, 70), (1, 513), (2, 3, 17, 19), (2, 64, 512, 512)])
@pytest.mark.parametrize("cancel", [False, True])
def test_channel_sum_vs_float64(shape, cancel):
    """ops.channel_sum (every bias gradient of conv2d_gradfix and fused_act: the sum over every dim but 1) against float64: inner
    extents not a multiple of 256, an outer extent > 1, 2-D inputs, C = 1, a 2x64x512x512 gradient, and data whose sum
    cancels (each channel's values followed by their negatives, shuffled, with a 1e-3 remainder).  Bar: 1e-6 * sum |x| per
    channel (fp32 accumulation)."""
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(len(shape) * 100 + shape[-1])
    x = torch.randn(shape, generator=g) * 3.0 + 1.0
    if cancel:
        flat = x.movedim(1, 0).reshape(shape[1], -1)
        n = flat.shape[1] // 2
        perm = torch.randperm(n, generator=g)
        flat[:, n:2 * n] = -flat[:, :n][:, perm] * (1.0 + 1e-3 * torch.randn((1, n), generator=g))
        x = flat.reshape([shape[1], shape[0]] + list(shape[2:])).movedim(0, 1).contiguous()
    xc = x.cuda()
    got = ops.channel_sum(xc)
    dims = [i for i in range(x.dim()) if i != 1]
    ref = x.double().sum(dim=dims)
    absum = x.double().abs().sum(dim=dims)
    err = (got.double().cpu() - ref).abs()
    print(f"channel_sum {shape} cancel={cancel}: max err/sum|x| {(err / absum).max().item():.2e}")
    assert (err <= 1e-6 * absum).all()
    assert torch.equal(got, ops.channel_sum(xc))
