"""GPU: the weight-preparation kernels of csrc/modulate.cu against float64 and bit patterns.

* ``ops.prep_weights`` (vt_modulate_weights_f32): modulation, demodulation and the [wB, k*k, Cout, cin_pad] layout, for
  realistic style rows, rows of ~1e-4 and ~1e-5 (where the 1e-8 epsilon matters and then dominates), all-zero rows and ~1e3 rows,
  at Cin*taps below, at and just above the 256-thread stride; pad channels exactly zero; the tf32 output bit for bit.
* ``ops.fold_upconv_weights`` (vt_fold_upconv_weights_f32): against the closed form (pinned on the CPU in
  test_weight_prep_host.py) for symmetric, asymmetric and full-rank blurs, up to a grid that needs the stride loop.
* ``ops.split_weights_bf16x3`` / ``split_weights_f16x3``: decoded bit for bit against torch's round-to-nearest-even conversions.

Bars (u = 2^-24; derivations next to each).  The worst error of every case is printed with ``-s``.
"""
import math

import pytest
import torch

from tests.test_weight_prep_host import bits, blur_kernels, fold64, prep64, rna_tf32

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

U = 2.0 ** -24


def style_rows(wB, Cin, families, seed):
    """[wB, Cin] style rows; row b follows families[b % len(families)]:
    real: 1 + 0.2 N(0,1) (modulation EqualLinear with bias_init = 1), e4 / e5: 1e-4 / 1e-5 N(0,1) (sum w^2 ~ 1e-8 / 1e-10 next to
    eps = 1e-8), zero, e3: 1e3 N(0,1)"""
    g = torch.Generator().manual_seed(seed)
    r = torch.randn((wB, Cin), generator=g)
    scale = {"real": None, "e4": 1e-4, "e5": 1e-5, "zero": 0.0, "e3": 1e3}
    for b in range(wB):
        f = families[b % len(families)]
        r[b] = 1.0 + 0.2 * r[b] if f == "real" else r[b] * scale[f]
    return r


FAMILIES = ["real", "e5", "zero", "e3", "e4"]

# (wB, Cout, Cin, k, cin_pad, demodulate)
PREP_CASES = [(5, 512, 512, 3, 512, True),      # Cin * taps = 4608 (18 terms per thread), every style family
              (2, 3, 512, 1, 512, False),       # ToRGB: no demodulation
              (5, 16, 3, 3, 32, True),          # the 3-channel input layer, pad 3 -> 32
              (5, 24, 19, 3, 64, True),         # 19 parsing channels, pad -> 64
              (5, 8, 16, 1, 32, True),          # Cin * taps = 16: fewer terms than threads
              (5, 8, 256, 1, 256, True),        # Cin * taps = 256: one term per thread
              (5, 8, 257, 1, 288, True),        # Cin * taps = 257: one thread sums two terms
              (1, 1, 1, 1, 32, True)]


def demod_bar(ref, ntaps):
    """Relative bound of one demodulated weight.  w = fl(fl(scale W) s) has relative error <= 2u.  Each of the 256 threads sums
    m = ceil(Cin*taps / 256) squares serially, then 5 shuffle levels and 3 levels across the 8 warps: the sum of non-negative
    terms is off by <= (m + 8)u relatively, plus 4u from squaring the 2u-accurate w.  + 1e-8, sqrtf, 1/x: 3 more roundings, the
    sqrt halves the sum's error, so demod is off by <= ((m + 12)/2 + 3)u, and the product w * demod adds 3u (w's 2u and the final
    rounding).  |err| <= ((m + 12)/2 + 6) u |ref|: an exact zero stays zero."""
    m = math.ceil(ntaps / 256)
    return ((m + 12) / 2 + 6) * U * ref.abs()


@pytest.mark.parametrize("case", PREP_CASES, ids=lambda c: "x".join(map(str, c[:5])) + ("-demod" if c[5] else ""))
def test_prep_weights_vs_float64(case):
    from vtoonify_b200 import ops
    wB, Cout, Cin, k, cin_pad, demod = case
    g = torch.Generator().manual_seed(Cout * 7 + Cin + k)
    W = torch.randn((Cout, Cin, k, k), generator=g).cuda()
    s = style_rows(wB, Cin, FAMILIES if wB > 2 else ["real"], seed=Cin + wB).cuda()
    scale = 1 / math.sqrt(Cin * k * k)
    out = ops.prep_weights(W, s, scale, demod, cin_pad, round_tf32=False)
    assert tuple(out.shape) == (wB, k * k, Cout, cin_pad)
    ref = prep64(W, s, scale, demod, cin_pad)
    assert torch.equal(out[..., Cin:], torch.zeros_like(out[..., Cin:])), "pad channels are not zero"
    err = (out.double() - ref).abs()
    if demod:
        bar = demod_bar(ref, Cin * k * k)
    else:
        # fl(fl(scale W) s): the same two roundings as fp32 torch, so bit for bit
        assert torch.equal(out[..., :Cin], (W * scale)[None].mul(s[:, None, :, None, None]).permute(0, 3, 4, 1, 2)
                           .reshape(wB, k * k, Cout, Cin))
        bar = 2 * U * ref.abs()
    for b in range(wB):
        fam = FAMILIES[b % len(FAMILIES)] if wB > 2 else "real"
        rel = (err[b] / bar[b].clamp_min(1e-300)).max().item()
        print(f"prep_weights {case} row {b} ({fam}): max rel err {(err[b] / ref[b].abs().clamp_min(1e-300)).max().item():.2e}, "
              f"max err/bar {rel:.3f}")
        if fam == "zero":
            assert torch.equal(out[b], torch.zeros_like(out[b])), "an all-zero style row must give exactly zero weights"
    assert (err <= bar).all(), f"{(err / bar.clamp_min(1e-300)).max().item():.2f} x the bar"
    # tf32 mode: the same weights rounded by cvt.rna.tf32, bit for bit; padding still +0
    out_r = ops.prep_weights(W, s, scale, demod, cin_pad, round_tf32=True)
    assert torch.equal(bits(out_r), bits(rna_tf32(out)))


def test_prep_weights_plain_relayout_and_tf32_ties():
    """style=None: the plain re-layout fl(scale * W) (bit for bit against torch, scale rounded to fp32 as the kernel gets it);
    with scale = 1 and round_tf32 the output is cvt.rna.tf32 of W itself, on crafted ties (low 13 bits 0x1000, both signs, hi
    mantissa even and odd) and their neighbours 0x0fff / 0x1001."""
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(9)
    Cout, Cin, k, cin_pad = 24, 19, 3, 32
    W = torch.randn((Cout, Cin, k, k), generator=g)
    out = ops.prep_weights(W.cuda(), None, 0.3, False, cin_pad, round_tf32=False)
    ref = (W * 0.3).permute(2, 3, 0, 1).reshape(1, 9, Cout, Cin)
    assert torch.equal(bits(out[..., :Cin].cpu()), bits(ref))
    assert torch.equal(out[..., Cin:], torch.zeros_like(out[..., Cin:]))
    u = bits(W) & ~0x1FFF
    low = torch.tensor([0x1000, 0x0FFF, 0x1001, 0x1000], dtype=torch.int32)[torch.arange(W.numel()) % 4].view(W.shape)
    u = u | low
    u[..., 0, 0] ^= 0x2000                                       # flip the last tf32 mantissa bit on some: even and odd hi
    Wt = u.view(torch.float32)
    assert (Wt < 0).any() and (Wt > 0).any()
    got = ops.prep_weights(Wt.cuda(), None, 1.0, False, cin_pad, round_tf32=True)
    ref = rna_tf32(Wt).permute(2, 3, 0, 1).reshape(1, 9, Cout, Cin)
    assert torch.equal(bits(got[..., :Cin].cpu()), bits(ref))
    assert torch.equal(bits(got[..., Cin:]), torch.zeros_like(bits(got[..., Cin:])))


def test_modulated_weights_end_to_end():
    """ModulatedConv2d.modulated_weights(style, cin_pad) from the 512-d style through the modulation EqualLinear, prep and (for the
    up-convolution) the fold, against float64 of the whole chain.  Bar: the modulation linear's error E_c (test_gpu_style_path's
    bound, here (16 + 8) u sum|x w scale| + 2u |bias|) moves v = scale W s by A = |scale W| E_c; the row's norm sqrt(|v|^2 + 1e-8)
    moves by at most |A|_2, a relative eta = |A|_2 * demod.  So |err| <= A * demod + eta |ref| + the demod bar (first order); the
    fold carries it through |K| and adds its own 9u."""
    from vtoonify_b200 import ops
    from vtoonify_b200.stylegan import ModulatedConv2d
    from vtoonify_b200.weights import det_state_dict
    for up in (False, True):
        m = ModulatedConv2d(64, 48, 3, 512, upsample=up)
        m.load_state_dict(det_state_dict(m, seed=3))
        m = m.cuda()
        g = torch.Generator().manual_seed(11)
        style = torch.randn((3, 512), generator=g).cuda()
        w = m.modulated_weights(style, 64, round_tf32=False, folded=up)
        Wm, bm = m.modulation.weight.double(), m.modulation.bias.double()
        ls = m.modulation.scale
        s64 = style.double() @ (Wm * ls).t() + bm
        E = 24 * U * (style.double().abs() @ (Wm.abs() * ls).t()) + 2 * U * bm.abs()
        ref = prep64(m.weight[0], s64, m.scale, True, 64)
        v = prep64(m.weight[0], s64, m.scale, False, 64)
        demod = 1.0 / torch.sqrt(v.pow(2).sum(dim=(1, 3), keepdim=True) + 1e-8)          # [B, 1, Cout, 1]
        A = prep64(m.weight[0].abs(), E, m.scale, False, 64)
        eta = A.pow(2).sum(dim=(1, 3), keepdim=True).sqrt() * demod
        bar = demod_bar(ref, 64 * 9) + A * demod + eta * ref.abs()
        srel = eta.max().item()
        if up:
            absref = fold64(ref.abs(), m.blur.kernel.abs())
            ref, bar = fold64(ref, m.blur.kernel), fold64(bar, m.blur.kernel.abs()) + 9 * U * absref
        err = (w.double() - ref).abs()
        print(f"modulated_weights up={up}: max eta {srel:.2e}, max err {err.max().item():.2e}, "
              f"max err/bar {(err / bar).max().item():.3f}")
        assert (err <= bar).all()


# ---- fold ---------------------------------------------------------------------------------------------------------------------
# (wB, Cout, Cin, cpad): cpad > Cin keeps zero pad channels; the last case has wB * Cout * cpad = 786432 > 132 SMs * 8 * 256
FOLD_CASES = [(1, 1, 3, 32), (3, 32, 19, 32), (1, 512, 64, 64), (3, 32, 32, 64), (3, 512, 512, 512)]


@pytest.mark.parametrize("blur", ["sym1331", "r1_1234", "rand"])
@pytest.mark.parametrize("case", FOLD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_fold_upconv_vs_float64(case, blur):
    """Each folded weight is a chain of at most 9 fmaf (up to 3 taps per axis reach one phase offset: 2d + k - r + 1 in [0, 3]),
    so |err| <= 9u sum |w k|, the closed form applied to |w| and |K|.  Pad channels (zero in the input) stay exactly zero; the tf32 mode's output is the
    fp32 output rounded by cvt.rna.tf32, bit for bit."""
    from vtoonify_b200 import ops
    wB, Cout, Cin, cpad = case
    if wB * Cout * cpad > 132 * 8 * 256:
        assert torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256 < wB * Cout * cpad
    g = torch.Generator().manual_seed(sum(case))
    W = torch.randn((Cout, Cin, 3, 3), generator=g).cuda()
    s = style_rows(wB, Cin, ["real"], seed=Cout).cuda()
    w = ops.prep_weights(W, s, 1 / math.sqrt(Cin * 9), True, cpad, round_tf32=False)
    K = blur_kernels()[blur].cuda()
    old = ops.set_precision("fp32")
    try:
        wf = ops.fold_upconv_weights(w, K)
        ops.set_precision("tf32")
        wf_r = ops.fold_upconv_weights(w, K)
    finally:
        ops.set_precision(old)
    assert tuple(wf.shape) == (wB, 9, 4 * Cout, cpad)
    ref = fold64(w, K)
    bar = 9 * U * fold64(w.abs(), K.abs())
    err = (wf.double() - ref).abs()
    print(f"fold {case} {blur}: max err {err.max().item():.2e}, max err/bar {(err / bar.clamp_min(1e-300)).max().item():.3f}")
    assert (err <= bar).all()
    assert torch.equal(bits(wf[..., Cin:]), torch.zeros_like(bits(wf[..., Cin:])))
    assert torch.equal(bits(wf_r), bits(rna_tf32(wf)))


def test_fold_transposed_weights_for_the_discriminator_input_gradient():
    """discriminator.py: conv2's input gradient folds prep_weights(W^T, cin_pad = the gradient's channel stride) with the
    ResBlock's downsampling blur; W^T is a non-contiguous view and its Cin (= the conv's Cout, 48) is padded to 64"""
    from vtoonify_b200 import ops
    from vtoonify_b200.stylegan import ResBlock
    blk = ResBlock(32, 48)
    c2, K = blk.conv2[1], blk.conv2[0].kernel
    Wt = c2.weight.detach().transpose(0, 1)
    w = ops.prep_weights(Wt.cuda(), None, c2.scale, False, 64, round_tf32=False)
    assert torch.equal(bits(w[..., :48].cpu()), bits((Wt * c2.scale).permute(2, 3, 0, 1).reshape(1, 9, 32, 48)))
    wf = ops.fold_upconv_weights(w, K.cuda())
    ref = fold64(w.cpu(), K)
    bar = 9 * U * fold64(w.cpu().abs(), K.abs())            # at most 9 fmaf per folded weight, as in test_fold_upconv_vs_float64
    err = (wf.cpu().double() - ref).abs()
    print(f"fold of transposed weights: max err {err.max().item():.2e}, max err/bar {(err / bar.clamp_min(1e-300)).max().item():.3f}")
    assert (err <= bar).all()
    assert torch.equal(bits(wf[..., 48:]), torch.zeros_like(bits(wf[..., 48:])))


# ---- operand splits ------------------------------------------------------------------------------------------------------------
def split_values(rows, C, family, seed):
    """fp32 [rows, C] weights of one value family (bit patterns built on the int32 view where the family needs exact values)"""
    g = torch.Generator().manual_seed(seed)
    n = rows * C
    if family == "normal":
        return torch.randn((rows, C), generator=g) / math.sqrt(4608)
    r = torch.randint(0, 1 << 30, (n,), generator=g, dtype=torch.int64)
    expo = 110 + (r >> 8) % 20                      # 2^-17 .. 2^2
    if family == "bf16_exact":                      # low 16 bits zero: lo must be +0
        u = ((expo << 7) | (r & 0x7F)) << 16
    elif family == "bf16_ties":                     # exactly halfway between two bf16 values, hi mantissa LSB even and odd
        u = (((expo << 7) | (r & 0x7F)) << 16) | 0x8000
    elif family == "tiny":                          # fp32 subnormals and the smallest normals
        u = torch.where(r % 3 == 0, (r >> 2) & 0x007FFFFF, (((r >> 2) % 3 + 1) << 23) | ((r >> 4) & 0x007FFFFF))
    else:
        raise ValueError(family)
    u = u | (((r >> 29) & 1) << 31)                 # both signs
    u = torch.where(u >= 1 << 31, u - (1 << 32), u).to(torch.int32)
    return u.view(torch.float32).view(rows, C)


def decode(buf, rows, C):
    """[rows, C] fp32 buffer of 32-channel chunks [hi x 32 | lo x 32] -> (hi, lo) int16 bit patterns [rows, C]"""
    h = buf.cpu().view(torch.int16).view(rows, C // 32, 2, 32)
    return h[:, :, 0].reshape(rows, C), h[:, :, 1].reshape(rows, C)


def ref_split(w, dtype, scale=1.0):
    """torch's RNE conversions on the CPU: hi = dtype(w * scale), lo = dtype(w * scale - hi) (the difference is exact in fp32)"""
    f = w * scale
    hi = f.to(dtype)
    lo = (f - hi.float()).to(dtype)
    return hi, lo


@pytest.mark.parametrize("family", ["normal", "bf16_exact", "bf16_ties", "tiny"])
@pytest.mark.parametrize("shape", [(64, 32), (9 * 32, 64), (18, 512), (9 * 4 * 48, 64)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_split_bf16x3_bitwise(shape, family):
    """[hi | lo] chunks bit for bit; |w - hi - lo| <= 2^-17 |w|: for |w| in [2^e, 2^(e+1)), |w - hi| <= 2^(e-8) (half of bf16's
    ulp 2^(e-7)), so lo's exponent is at most e - 9 and its rounding error at most 2^(e-17).  For fp32 subnormals (bf16 shares
    fp32's exponent range, 7 mantissa bits below 2^-126) it is half a bf16 subnormal step, 2^-134."""
    from vtoonify_b200 import ops
    rows, C = shape
    w = split_values(rows, C, family, seed=rows + C)
    buf = ops.split_weights_bf16x3(w.cuda())
    hi, lo = decode(buf, rows, C)
    rhi, rlo = ref_split(w, torch.bfloat16)
    mism = (hi != rhi.view(torch.int16)).sum().item() + (lo != rlo.view(torch.int16)).sum().item()
    rec = (w.double() - rhi.double() - rlo.double()).abs()
    recbar = torch.maximum(2.0 ** -17 * w.double().abs(), torch.full_like(rec, 2.0 ** -134))
    print(f"split bf16x3 {shape} {family}: {mism} mismatching halves, max |w - hi - lo| / bar {(rec / recbar).max().item():.3f}")
    assert torch.equal(hi, rhi.view(torch.int16)), "hi differs from torch's bf16 RNE"
    assert torch.equal(lo, rlo.view(torch.int16)), "lo differs from torch's bf16 RNE of w - hi"
    if family == "bf16_exact":
        assert (lo == 0).all()
    assert (rec <= recbar).all()


@pytest.mark.parametrize("R", [32, 48])
def test_split_bf16x3_nstack_layout(R):
    """nstack: input rows in groups of R (R = weight.shape[-2]); group g becomes R rows [hi|hi] then R rows [lo|lo]"""
    from vtoonify_b200 import ops
    taps, C = 9, 64
    w = split_values(taps * R, C, "normal", seed=R)
    buf = ops.split_weights_bf16x3(w.view(1, taps, R, C).cuda(), nstack=True)
    assert tuple(buf.shape) == (2 * taps * R, C)
    h = buf.cpu().view(torch.int16).view(taps, 2, R, C // 32, 2, 32)
    rhi, rlo = ref_split(w, torch.bfloat16)
    rhi, rlo = rhi.view(torch.int16).view(taps, R, C // 32, 32), rlo.view(torch.int16).view(taps, R, C // 32, 32)
    for half in range(2):
        assert torch.equal(h[:, 0, :, :, half], rhi), "hi rows"
        assert torch.equal(h[:, 1, :, :, half], rlo), "lo rows"


@pytest.mark.parametrize("family", ["normal", "range", "lo_subnormal", "tiny"])
@pytest.mark.parametrize("shape", [(64, 32), (18, 512), (9 * 4 * 32, 64)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_split_f16x3_bitwise(shape, family):
    """fp16 halves of w * 256 bit for bit; |w - (hi + lo) / 256| <= max(2^-22 |w|, 2^-33): 11 + 11 mantissa bits while lo is
    normal, half of fp16's subnormal step 2^-24 (/ 256) once lo is subnormal.  Families: demodulated-size weights, |w| up to
    255.875 (w * 256 up to fp16's max 65504, the documented range), weights ~4e-6 whose lo is an fp16 subnormal, and fp32
    values whose hi already underflows."""
    from vtoonify_b200 import ops
    rows, C = shape
    g = torch.Generator().manual_seed(rows * 3 + C)
    if family == "normal":
        w = torch.randn((rows, C), generator=g) / math.sqrt(4608)
    elif family == "range":
        w = (torch.rand((rows, C), generator=g) * 2 - 1) * 255.875
        w.view(-1)[:4] = torch.tensor([255.875, -255.875, 255.87, 0.0])
    elif family == "lo_subnormal":
        w = torch.randn((rows, C), generator=g) * 4e-6
    else:
        w = torch.randn((rows, C), generator=g) * 1e-10
    buf = ops.split_weights_f16x3(w.cuda())
    hi, lo = decode(buf, rows, C)
    rhi, rlo = ref_split(w, torch.float16, ops.F16_WEIGHT_SCALE)
    mism = (hi != rhi.view(torch.int16)).sum().item() + (lo != rlo.view(torch.int16)).sum().item()
    rec = (w.double() - (rhi.double() + rlo.double()) / ops.F16_WEIGHT_SCALE).abs()
    recbar = torch.maximum(2.0 ** -22 * w.double().abs(), torch.full_like(rec, 2.0 ** -33))
    nsub = (rlo.abs() < 2.0 ** -14).logical_and(rlo != 0).sum().item()
    print(f"split f16x3 {shape} {family}: {mism} mismatching halves, {nsub} subnormal lo, "
          f"max |w - (hi + lo)/256| / bar {(rec / recbar).max().item():.3f}")
    if family == "lo_subnormal":
        assert nsub > 0
    assert torch.equal(hi, rhi.view(torch.int16)), "hi differs from torch's fp16 RNE"
    assert torch.equal(lo, rlo.view(torch.int16)), "lo differs from torch's fp16 RNE of w * 256 - hi"
    assert (rec <= recbar).all()
