"""``random_apply_affine``: the geometric training augmentation of ``model/simple_augment.py`` (train_vtoonify_d.py:262,
train_vtoonify_t.py:206) on the library.

``random_apply_affine(img, p, G=None, antialiasing_kernel=SYM6) -> (img_out, G)`` keeps the reference's signature, return value and
random draws.  Per sample b and channel c the output is

    out[b, c] = down2(warp_b(up2(reflect_pad(img[b, c]))))

- ``reflect_pad``: one batch-wide reflect pad, wide enough for every sample's transformed corners plus the filter support;
- ``up2``: x2 upsampling with the 12-tap wavelet, a true convolution (``upfirdn2d`` with ``up=2``, pad (6, 5)), x then y, zeros
  beyond the padded extent;
- ``warp_b``: bilinear ``grid_sample`` (zeros outside the x2 image, ``align_corners=False``) on the grid of ``F.affine_grid`` with the
  sample's composed 2x3 matrix, over a ``2(H+6) x 2(W+6)`` grid;
- ``down2``: x2 downsampling with the flipped kernel (``upfirdn2d`` with ``down=2``, pad (-1, -1)), x then y.

The transform sampler, the pads and the composed matrix are formed on the CPU in float32 with the reference's operations, so ``G``
and the torch CPU generator's state afterwards are bit-identical to the reference's.  The image path is one launch of
``vt_augment_affine_f32`` whenever ``vt_augment_affine_plan`` finds a tile whose worst-sample footprint fits in shared memory;
otherwise (a caller-supplied ``G`` that zooms far out) the same statements run unfused on ``ops.upfirdn2d_planar`` and torch's
``affine_grid`` / ``grid_sample``.  Forward only: an ``img`` that requires grad in grad mode raises ``NotImplementedError``.
"""
import ctypes
import math

import torch
from torch.nn import functional as F

from . import _lib, ops

SYM6 = (
    0.015404109327027373,
    0.0034907120842174702,
    -0.11799011114819057,
    -0.048311742585633,
    0.4910559419267466,
    0.787641141030194,
    0.3379294217276218,
    -0.07263752278646252,
    -0.021060292512300564,
    0.04472490177066578,
    0.0017677118642428036,
    -0.007800708325034148,
)

TAPS = 12
PAD_K = TAPS // 4             # the warp grid is 2 * PAD_K samples wider than the x2 image of the input on each side


# ---------------------------------------------------------------------------------------------------------------------------------
# transform sampler (CPU, float32).  Every statement below is chosen for its float32 result and its generator draws: the same draws in
# the same order (a Bernoulli selection per stage, also at p = 0), and the same tensor operations, so that G is bit-identical.
# ---------------------------------------------------------------------------------------------------------------------------------
def _eye(n):
    return torch.eye(3).unsqueeze(0).repeat(n, 1, 1)


def _scale(sx, sy):
    m = _eye(sx.shape[0])
    m[:, 0, 0] = sx
    m[:, 1, 1] = sy
    return m


def _translate(tx, ty):
    m = _eye(tx.shape[0])
    m[:, :2, 2] = torch.stack((tx, ty), 1)
    return m


def _rotate(theta):
    n = theta.shape[0]
    m = _eye(n)
    s, c = torch.sin(theta), torch.cos(theta)
    m[:, :2, :2] = torch.stack((c, -s, s, c), 1).view(n, 2, 2)
    return m


def _maybe(p, transform, prev, eye):
    """prev, left-multiplied by transform on the samples a Bernoulli(p) draw selects"""
    n = transform.shape[0]
    sel = torch.empty(n).bernoulli_(p).view(n, 1, 1)
    return (sel * transform + (1 - sel) * eye) @ prev


def sample_affine(p: float, n: int, height: int, width: int) -> torch.Tensor:
    """[n, 3, 3] float32 forward transform: flip, integer translate, isotropic scale, pre-rotate, anisotropic scale, post-rotate,
    fractional translate, each applied with probability p (the rotations with 1 - sqrt(1 - p))."""
    eye = _eye(n)
    G = eye
    flip = torch.tensor((0, 1))[torch.randint(high=2, size=(n,))]
    G = _maybe(p, _scale(1 - 2.0 * flip, torch.ones(n)), G, eye)
    t = torch.empty(n).uniform_(-0.125, 0.125)
    G = _maybe(p, _translate(torch.round(t * width) / width, torch.round(t * height) / height), G, eye)
    s = torch.empty(n).log_normal_(mean=0, std=0.1 * math.log(2))
    G = _maybe(p, _scale(s, s), G, eye)
    p_rot = 1 - math.sqrt(1 - p)
    r = torch.empty(n).uniform_(-math.pi * 0.25, math.pi * 0.25)
    G = _maybe(p_rot, _rotate(-r), G, eye)
    s = torch.empty(n).log_normal_(mean=0, std=0.1 * math.log(2))
    G = _maybe(p, _scale(s, 1 / s), G, eye)
    r = torch.empty(n).uniform_(-math.pi * 0.25, math.pi * 0.25)
    G = _maybe(p_rot, _rotate(-r), G, eye)
    t = torch.empty(n).normal_(0, 0.125)
    G = _maybe(p, _translate(t, t), G, eye)
    return G


def padding(G: torch.Tensor, height: int, width: int):
    """batch-wide reflect pads (x1, x2, y1, y2): the extent of every sample's transformed image corners around the centre, plus
    2 * PAD_K for the filters, clamped to [0, size - 1] (the most a reflect pad can take) and rounded up"""
    cx, cy = (width - 1) / 2, (height - 1) / 2
    corners = torch.tensor([(-cx, -cy, 1), (cx, -cy, 1), (cx, cy, 1), (-cx, cy, 1)])
    xy = (G @ corners.T)[:, :2, :].permute(1, 0, 2).flatten(1)
    ext = torch.cat((-xy, xy)).max(1).values
    ext = ext + torch.tensor([PAD_K * 2 - cx, PAD_K * 2 - cy] * 2)
    ext = ext.max(torch.tensor([0, 0] * 2)).min(torch.tensor([width - 1, height - 1] * 2))
    x1, y1, x2, y2 = ext.ceil().to(torch.int32)
    return x1, x2, y1, y2


def _mat(sx, sy, tx, ty):
    return torch.tensor(((sx, 0, tx), (0, sy, ty), (0, 0, 1)), dtype=torch.float32)


def sampling_matrix(G: torch.Tensor, pads, height: int, width: int) -> torch.Tensor:
    """[B, 3, 3] float32 matrix whose top two rows are ``affine_grid``'s theta: G recentred on the padded image, conjugated to the x2
    image (scale 2, half-pixel shift), and normalised from the warp grid's size to the x2 image's."""
    x1, x2, y1, y2 = (int(v) for v in pads)
    M = _mat(1, 1, (x1 - x2) / 2, (y1 - y2) / 2) @ G
    M = _mat(2, 2, 0, 0) @ M @ _mat(1 / 2, 1 / 2, 0, 0)
    M = _mat(1, 1, -0.5, -0.5) @ M @ _mat(1, 1, 0.5, 0.5)
    up_w, up_h = (width + x1 + x2) * 2, (height + y1 + y2) * 2
    grid_w, grid_h = (width + PAD_K * 2) * 2, (height + PAD_K * 2) * 2
    return _mat(2 / up_w, 2 / up_h, 0, 0) @ M @ _mat(1 / (2 / grid_w), 1 / (2 / grid_h), 0, 0)


def warp_coefficients(theta: torch.Tensor, pads, height: int, width: int) -> torch.Tensor:
    """[B, 6] float64 (x0, x_col, x_row, y0, y_col, y_row): warp-grid (column j, row i) -> x2-image pixel coordinates
    x = x0 + x_col j + x_row i under align_corners=False, i.e. ((theta @ (u_j, v_i, 1)) + 1) * size / 2 - 1/2 with
    u_j = (2j + 1) / grid_w - 1, v_i = (2i + 1) / grid_h - 1, in exact arithmetic from the float32 theta."""
    x1, x2, y1, y2 = (int(v) for v in pads)
    up_w, up_h = (width + x1 + x2) * 2, (height + y1 + y2) * 2
    grid_w, grid_h = (width + PAD_K * 2) * 2, (height + PAD_K * 2) * 2
    t = theta[:, :2, :].double()
    out = torch.empty(t.shape[0], 6, dtype=torch.float64)
    for r, size in ((0, up_w), (1, up_h)):
        a, b, c = t[:, r, 0], t[:, r, 1], t[:, r, 2]
        out[:, 3 * r + 1] = a * (size / grid_w)
        out[:, 3 * r + 2] = b * (size / grid_h)
        out[:, 3 * r] = (a / grid_w + b / grid_h + c - a - b + 1) * (size / 2) - 0.5
    return out


def plan(coef: torch.Tensor, height: int, width: int):
    """-> (tile side, x2-image window width, height) of the fused kernel for these [B, 6] float64 CPU coefficients; the tile side is
    0 for the unfused route"""
    coef = coef.contiguous()
    win = (ctypes.c_int * 2)()
    lib = _lib.load()
    tile = lib.vt_augment_affine_plan(ctypes.c_void_p(coef.data_ptr()), coef.shape[0], height, width, win)
    if tile < 0:
        raise _lib.VtError(lib.vt_last_error().decode("utf-8", "replace"))
    return int(tile), int(win[0]), int(win[1])


def _check(img, antialiasing_kernel):
    if not isinstance(img, torch.Tensor) or img.dim() != 4:
        raise ValueError("random_apply_affine: img must be a [B, C, H, W] tensor")
    if torch.is_grad_enabled() and img.requires_grad:
        raise NotImplementedError("random_apply_affine: img requires grad, but the library has no backward for the augmentation; "
                                  "call it under torch.no_grad() or on a detached img")
    if len(antialiasing_kernel) != TAPS:
        raise NotImplementedError(f"random_apply_affine: antialiasing_kernel must have {TAPS} taps "
                                  f"(got {len(antialiasing_kernel)})")
    if not img.is_cuda:
        raise _lib.VtError("random_apply_affine: img must be a CUDA tensor (this library has no CPU path)")
    if img.dtype != torch.float32:
        raise _lib.VtError(f"random_apply_affine: img must be float32 (got {img.dtype})")


def _unfused(img, kernel, pads, theta):
    """the reference's statements on the library's upfirdn2d: for transforms whose footprint the fused kernel cannot stage"""
    B, C, H, W = img.shape
    x1, x2, y1, y2 = pads
    flip = torch.flip(kernel, (0,))
    x = F.pad(img, (x1, x2, y1, y2), mode="reflect")
    x = ops.upfirdn2d_planar(x, kernel.view(1, TAPS), (2, 1), (1, 1), (6, 5, 0, 0))
    x = ops.upfirdn2d_planar(x, kernel.view(TAPS, 1), (1, 2), (1, 1), (0, 0, 6, 5))
    grid = F.affine_grid(theta[:, :2, :].to(x), (B, C, (H + PAD_K * 2) * 2, (W + PAD_K * 2) * 2), align_corners=False)
    x = F.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
    x = ops.upfirdn2d_planar(x, flip.view(1, TAPS), (1, 1), (2, 1), (-1, -1, 0, 0))
    return ops.upfirdn2d_planar(x, flip.view(TAPS, 1), (1, 1), (1, 2), (0, 0, -1, -1))


def random_apply_affine(img: torch.Tensor, p: float, G: torch.Tensor = None, antialiasing_kernel=SYM6):
    """-> (augmented img, G).  ``G=None`` samples [B, 3, 3] float32 inverse transforms on the CPU generator; a given ``G`` (CPU
    float32) is used as is.  img: CUDA float32 [B, C, H, W]."""
    _check(img, antialiasing_kernel)
    B, C, H, W = img.shape
    if G is None:
        G = torch.inverse(sample_affine(p, B, H, W))
    pads = tuple(int(v) for v in padding(G, H, W))
    theta = sampling_matrix(G, pads, H, W)
    kernel = torch.as_tensor(antialiasing_kernel).to(img)
    img = img.contiguous()
    coef = warp_coefficients(theta, pads, H, W)
    tile, win_w, win_h = plan(coef, H, W)
    if tile == 0:
        return _unfused(img, kernel, pads, theta), G
    coef = coef.to(img.device)
    out = torch.empty_like(img)
    x1, x2, y1, y2 = pads
    _lib.check(_lib.load().vt_augment_affine_f32(img.data_ptr(), out.data_ptr(), kernel.data_ptr(), coef.data_ptr(), B, C, H, W,
                                                 x1, y1, H + y1 + y2, W + x1 + x2, tile, win_w, win_h, ops._stream()))
    return out, G
