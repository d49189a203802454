"""CPU: the float64 references the weight-preparation GPU tests compare against, pinned here without a GPU, and the shape checks
of the ops wrappers.

* ``fold64``: the closed form of Blur o conv_transpose2d(stride 2) folded into 4 phase kernels (what vt_fold_upconv_weights_f32
  computes).  Convolving with the folded kernels must equal ``upfirdn2d(conv_transpose2d(x, w, stride=2), K, pad=(1, 1))`` for
  symmetric, asymmetric rank-1 and full-rank blurs: a missing or doubled kernel flip fails on the asymmetric ones.
* ``rna_tf32``: the bit emulation of ``cvt.rna.tf32.f32`` (round to 10 mantissa bits, ties away from zero) that the GPU tests
  apply to fp32 outputs to check the tf32-mode outputs bit for bit; checked here against a float64 restatement.
* ``prep64``: modulation, demodulation (eps 1e-8 inside the sqrt) and the [wB, k*k, Cout, cin_pad] layout.
* Every wrapper check added to ops (axpby, linear, prep_weights, gate_shortcut_add, bilinear_add) raises VtError on CPU
  tensors, before any device work, so no kernel is ever launched on mismatched shapes.
"""
import math

import pytest
import torch
import torch.nn.functional as F

torch.set_grad_enabled(False)

DEMOD_EPS = 1e-8


# ---- helpers shared with the GPU tests ------------------------------------------------------------------------------------------
def rna_tf32(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> fp32 rounded to tf32 (10 explicit mantissa bits) to nearest, ties away from zero: add half an ulp to the
    magnitude bits and clear the 13 low bits (sign-magnitude, so the same on negative values).  Finite inputs only."""
    u = t.contiguous().view(torch.int32)
    return ((u + 0x1000) & ~0x1FFF).view(torch.float32)


def bits(t: torch.Tensor) -> torch.Tensor:
    """int32 view of an fp32 tensor: torch.equal on it compares bit patterns (tells -0 from +0)"""
    return t.contiguous().view(torch.int32)


def fold64(w: torch.Tensor, blur: torch.Tensor) -> torch.Tensor:
    """[wB, 9, Cout, cpad] prep-layout 3x3 weights (slab ky*3+kx) and a 4x4 blur -> float64 [wB, 9, 4*Cout, cpad]: slab
    (dy+1)*3+(dx+1) of phase ry*2+rx holds G_r[d] = sum_k w[k] * kf[2d + k - r + 1] per axis, kf the flipped blur."""
    w = w.double()
    kf = torch.flip(blur.double(), [0, 1])
    wB, _, Cout, cpad = w.shape
    out = torch.zeros((wB, 9, 4 * Cout, cpad), dtype=torch.float64, device=w.device)
    for ry in range(2):
        for rx in range(2):
            ph = ry * 2 + rx
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    g = out[:, (dy + 1) * 3 + dx + 1, ph * Cout:(ph + 1) * Cout]
                    for ky in range(3):
                        iy = 2 * dy + ky - ry + 1
                        if not 0 <= iy <= 3:
                            continue
                        for kx in range(3):
                            ix = 2 * dx + kx - rx + 1
                            if 0 <= ix <= 3:
                                g += w[:, ky * 3 + kx] * kf[iy, ix].item()
    return out


def prep64(W: torch.Tensor, style, scale: float, demodulate: bool, cin_pad: int) -> torch.Tensor:
    """float64 ModulatedConv2d weights (model/stylegan/model.py:259-267): w = scale * W * s[b, c], demod = 1 / sqrt(sum w^2 + 1e-8)
    over (c, ky, kx), in the kernels' [wB, k*k, Cout, cin_pad] layout with zero pad channels.  ``scale`` is rounded to fp32 first,
    as the kernel receives it."""
    Cout, Cin, kh, kw = W.shape
    w = float(torch.tensor(scale, dtype=torch.float32)) * W.double()[None]
    if style is not None:
        w = w * style.double()[:, None, :, None, None]
    if demodulate:
        w = w / torch.sqrt(w.pow(2).sum(dim=(2, 3, 4), keepdim=True) + DEMOD_EPS)
    out = torch.zeros((w.shape[0], kh * kw, Cout, cin_pad), dtype=torch.float64, device=W.device)
    out[..., :Cin] = w.permute(0, 3, 4, 1, 2).reshape(w.shape[0], kh * kw, Cout, Cin)
    return out


def blur_kernels():
    """the blurs the fold is tested with: StyleGAN's symmetric [1,3,3,1] (x 4 for the 2x up-sampling), the asymmetric rank-1
    [1,2,3,4] and a full-rank random 4x4"""
    from vtoonify_b200.stylegan import make_kernel
    g = torch.Generator().manual_seed(44)
    return {"sym1331": make_kernel([1, 3, 3, 1]) * 4, "r1_1234": make_kernel([1, 2, 3, 4]) * 4,
            "rand": torch.randn((4, 4), generator=g)}


# ---- the fold's closed form --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("blur", ["sym1331", "r1_1234", "rand"])
@pytest.mark.parametrize("shape", [(1, 3, 2, 5, 6), (2, 4, 3, 7, 4)])
def test_fold_closed_form_equals_blur_of_conv_transpose(shape, blur):
    from oracle import vt_oracle as O
    B, Cin, Cout, H, W = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn((B, Cin, H, W), generator=g, dtype=torch.float64)
    w = torch.randn((Cout, Cin, 3, 3), generator=g, dtype=torch.float64)
    K = blur_kernels()[blur].double()
    ref = O.upfirdn2d(F.conv_transpose2d(x, w.transpose(0, 1), stride=2), K, pad=(1, 1))
    wp = w.permute(2, 3, 0, 1).reshape(1, 9, Cout, Cin)                  # prep layout, slab ky*3+kx
    G = fold64(wp, K)[0]                                                  # [9, 4*Cout, Cin]
    out = torch.zeros((B, Cout, 2 * H, 2 * W), dtype=torch.float64)
    for ry in range(2):
        for rx in range(2):
            ph = ry * 2 + rx
            kern = G[:, ph * Cout:(ph + 1) * Cout].permute(1, 2, 0).reshape(Cout, Cin, 3, 3)   # [n, c, dy+1, dx+1]
            out[:, :, ry::2, rx::2] = F.conv2d(x, kern, padding=1)
    assert ref.shape == out.shape
    err = (out - ref).abs().max().item()
    assert err <= 1e-12 * ref.abs().max().item(), err


def test_upsampling_modconv_with_any_4tap_blur_takes_the_folded_route():
    """an asymmetric 4-tap blur gives the same 4x4 kernel shape and (1, 1) padding as StyleGAN's, so the folded up-convolution
    (and the flip inside the fold) serves it"""
    from vtoonify_b200.stylegan import ModulatedConv2d
    m = ModulatedConv2d(8, 8, 3, 16, upsample=True, blur_kernel=[1, 2, 3, 4])
    assert tuple(m.blur.kernel.shape) == (4, 4) and tuple(m.blur.pad) == (1, 1)
    assert not torch.equal(m.blur.kernel, torch.flip(m.blur.kernel, [0, 1]))


# ---- the tf32 emulation ------------------------------------------------------------------------------------------------------
def rna_tf32_64(x: torch.Tensor) -> torch.Tensor:
    """float64 restatement: q = 2^(e - 10) for |x| in [2^e, 2^(e+1)), result sign(x) * floor(|x| / q + 1/2) * q"""
    xd = x.double()
    e = torch.floor(torch.log2(xd.abs()))
    q = torch.pow(2.0, e - 10)
    return torch.sign(xd) * torch.floor(xd.abs() / q + 0.5) * q


def test_rna_tf32_emulation():
    g = torch.Generator().manual_seed(3)
    mant = torch.randint(0, 1 << 10, (4096,), generator=g, dtype=torch.int32) << 13
    expo = torch.randint(80, 170, (4096,), generator=g, dtype=torch.int32) << 23
    low = torch.cat([torch.full((1024,), 0x1000), torch.full((1024,), 0x0FFF), torch.full((1024,), 0x1001),
                     torch.randint(0, 0x2000, (1024,), generator=g)]).to(torch.int32)
    sign = torch.where(torch.arange(4096) % 2 == 0, 0, -(1 << 31)).to(torch.int32)
    u = sign | expo | mant | low
    u = torch.cat([u, torch.tensor([0x3F801000, -0x407FF000, 0x3FFFF000, 0x00000000], dtype=torch.int32)])   # ties, carry into exponent
    x = u.view(torch.float32)
    got = rna_tf32(x)
    nz = x != 0
    assert torch.equal(got[nz].double(), rna_tf32_64(x[nz]))
    assert torch.equal(bits(got[~nz]), bits(x[~nz]))
    assert ((bits(got) & 0x1FFF) == 0).all()
    assert got[-4].item() == 1.0 + 2.0 ** -10 and got[-3].item() == -(1.0 + 2.0 ** -10) and got[-2].item() == 2.0   # ties away


# ---- prep64 against the reference's own formula ----------------------------------------------------------------------------
def test_prep64_matches_reference_modulation():
    """prep64 restates model.py:259-267 (weight = scale * W * style; demod = rsqrt(sum weight^2 + 1e-8)); the layout is the
    transpose [b, ky*kw+kx, n, c]"""
    g = torch.Generator().manual_seed(5)
    W = torch.randn((6, 5, 3, 3), generator=g, dtype=torch.float64)
    s = torch.randn((2, 5), generator=g, dtype=torch.float64)
    scale = 1 / math.sqrt(5 * 9)
    ref = scale * W[None] * s[:, None, :, None, None]
    ref = ref * torch.rsqrt(ref.pow(2).sum([2, 3, 4]) + 1e-8)[:, :, None, None, None]
    got = prep64(W, s, scale, True, 32)
    assert torch.equal(got[..., 5:], torch.zeros_like(got[..., 5:]))
    assert torch.allclose(got[1, 3 * 1 + 2, 4, 3], ref[1, 4, 3, 1, 2], rtol=1e-7, atol=0)   # scale rounded to fp32
    assert torch.allclose(got[..., :5], ref.permute(0, 3, 4, 1, 2).reshape(2, 9, 6, 5), rtol=1e-7, atol=0)


# ---- wrapper shape checks (CPU tensors: they must raise before anything reaches the device) -------------------------------------
def test_axpby_checks_b_length():
    from vtoonify_b200 import ops
    from vtoonify_b200._lib import VtError
    with pytest.raises(VtError, match=r"axpby: b has 5 elements, a has 6"):
        ops.axpby(torch.zeros(6), torch.zeros(5), 1.0, 1.0)


def test_linear_checks_weight_and_bias():
    from vtoonify_b200 import ops
    from vtoonify_b200._lib import VtError
    x = torch.zeros((3, 33))
    with pytest.raises(VtError, match=r"linear: weight \(8, 32\) does not match input \(3, 33\)"):
        ops.linear(x, torch.zeros((8, 32)), None)
    with pytest.raises(VtError, match=r"linear: weight \(33,\) does not match"):
        ops.linear(x, torch.zeros(33), None)
    with pytest.raises(VtError, match=r"linear: bias has 7 elements, out_dim is 8"):
        ops.linear(x, torch.zeros((8, 33)), torch.zeros(7))
    with pytest.raises(VtError, match=r"linear: weight \(8, 32\) does not match input \(2, 4, 33\)"):
        ops.linear(torch.zeros((2, 4, 33)), torch.zeros((8, 32)), torch.zeros(8))


def test_prep_weights_checks_style():
    from vtoonify_b200 import ops
    from vtoonify_b200._lib import VtError
    W = torch.zeros((4, 19, 3, 3))
    with pytest.raises(VtError, match=r"prep_weights: style \(2, 18\) must be \[wB, Cin\] with Cin = 19"):
        ops.prep_weights(W, torch.zeros((2, 18)))
    with pytest.raises(VtError, match=r"prep_weights: style \(19,\) must be \[wB, Cin\]"):
        ops.prep_weights(W, torch.zeros(19))
    with pytest.raises(VtError, match=r"prep_weights: W must be \[Cout, Cin, kh, kw\]"):
        ops.prep_weights(torch.zeros((1, 4, 19, 3, 3)))


def test_gate_shortcut_add_checks_shapes():
    from vtoonify_b200 import ops
    from vtoonify_b200._lib import VtError
    x = torch.zeros((2, 5, 7, 8))
    with pytest.raises(VtError, match=r"gate_shortcut_add: sc \(1, 5, 7, 8\) does not match the batch and channels"):
        ops.gate_shortcut_add(x, None, torch.zeros((1, 5, 7, 8)))
    with pytest.raises(VtError, match=r"gate_shortcut_add: sc \(2, 10, 14, 4\) does not match the batch and channels"):
        ops.gate_shortcut_add(x, None, torch.zeros((2, 10, 14, 4)), 2)
    with pytest.raises(VtError, match=r"gate_shortcut_add: gate \(2, 4\) must hold \[B, C\] = \[2, 8\] values"):
        ops.gate_shortcut_add(x, torch.zeros((2, 4)), x)
    with pytest.raises(VtError, match=r"gate_shortcut_add: gate \(1, 16\) must hold"):
        ops.gate_shortcut_add(x, torch.zeros((1, 16)), x)
    with pytest.raises(VtError, match=r"gate_shortcut_add: x \(2, 5, 7, 8\) and sc \(2, 5, 7, 8\) must be contiguous NHWC"):
        ops.gate_shortcut_add(torch.zeros((2, 8, 5, 7)).permute(0, 2, 3, 1), None, x)
    with pytest.raises(VtError, match=r"gate_shortcut_add: x \(5, 7, 8\)"):
        ops.gate_shortcut_add(x[0], None, x)


def test_bilinear_add_checks_batch_and_channels():
    from vtoonify_b200 import ops
    from vtoonify_b200._lib import VtError
    with pytest.raises(VtError, match=r"bilinear_add: x \(2, 4, 4, 8\) and y \(3, 8, 8, 8\) differ in batch or channels"):
        ops.bilinear_add(torch.zeros((2, 4, 4, 8)), torch.zeros((3, 8, 8, 8)))
    with pytest.raises(VtError, match=r"bilinear_add: x \(2, 4, 4, 8\) and y \(2, 8, 8, 12\) differ in batch or channels"):
        ops.bilinear_add(torch.zeros((2, 4, 4, 8)), torch.zeros((2, 8, 8, 12)))
    with pytest.raises(VtError, match=r"must be contiguous NHWC"):
        ops.bilinear_add(torch.zeros((2, 8, 4, 4)).permute(0, 2, 3, 1), torch.zeros((2, 8, 8, 8)))


def test_wrapper_checks_pass_matching_shapes_through_to_the_device_check():
    """matching shapes get past the new checks and stop at the CPU-tensor check, so the checks reject only mismatches"""
    from vtoonify_b200 import ops
    from vtoonify_b200._lib import VtError
    x = torch.zeros((2, 5, 7, 8))
    for call in (lambda: ops.axpby(torch.zeros(6), torch.zeros((2, 3)), 1.0, 1.0),
                 lambda: ops.linear(torch.zeros((2, 4, 33)), torch.zeros((8, 33)), torch.zeros(8)),
                 lambda: ops.prep_weights(torch.zeros((4, 19, 3, 3)), torch.zeros((2, 19))),
                 lambda: ops.gate_shortcut_add(x, torch.zeros((2, 8)), torch.zeros((2, 9, 13, 8)), 2),
                 lambda: ops.bilinear_add(torch.zeros((2, 4, 4, 8)), torch.zeros((2, 9, 3, 8)))):
        with pytest.raises(VtError, match="need CUDA tensors"):
            call()
