"""NumPy oracle of the FFHQ face alignment (`align_face`, model/encoder/align_all_parallel.py:59-150), one function per stage.

Each stage restates the library the reference calls, with the roundings that library makes on x86-64:
- `lanczos_resize`: Pillow `Image.resize(size, LANCZOS)` on RGB uint8 (22-bit fixed point, horizontal pass first);
- `reflect_pad`: `np.pad(float32(img), ..., 'reflect')`;
- `gaussian_axis`: one axis of SciPy `gaussian_filter` in float32 (double accumulation, mode 'reflect');
- `pad_mask`, `blend`, `median`, `quantize`: the reference's NumPy statements on the padded image;
- `quad_warp`: Pillow `Image.transform(size, QUAD, corners, BILINEAR)`.
`align(img, params)` chains them as the reference does, from the geometry of `vtoonify_b200.align.align_params`.
"""
import math

import numpy as np

OUT = 256


def synth_image(seed, h, w):
    """a seeded uint8 RGB test image: two gradients, a few sharp-edged rectangles and discs, and noise"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w].astype(np.float64)
    img = np.empty((h, w, 3), np.float64)
    for c in range(3):
        a, b = rng.uniform(-1, 1, 2)
        img[..., c] = 128 + 90 * (a * xx / w + b * yy / h)
    for _ in range(8):
        y0, x0 = rng.integers(0, h), rng.integers(0, w)
        y1, x1 = y0 + rng.integers(2, max(3, h // 3)), x0 + rng.integers(2, max(3, w // 3))
        img[y0:y1, x0:x1] = rng.uniform(0, 255, 3)
    for _ in range(4):
        cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(2, max(3, min(h, w) / 5))
        img[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = rng.uniform(0, 255, 3)
    img += rng.normal(0, 12, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def synth_landmarks(seed, eye_left, eye_right, mouth_left, mouth_right):
    """[68, 2] float64 landmarks whose eyes average to the given centres and whose mouth corners are the given points; the other
    points (which the alignment never reads) are seeded noise around the face"""
    rng = np.random.default_rng(seed)
    lm = np.empty((68, 2))
    centre = (np.asarray(eye_left) + eye_right + mouth_left + mouth_right) / 4
    lm[:] = centre + rng.normal(0, 20, (68, 2))
    for lo, c in ((36, eye_left), (42, eye_right)):
        d = rng.normal(0, 3, (6, 2))
        d -= d.mean(0)
        lm[lo:lo + 6] = np.asarray(c, np.float64) + d
        lm[lo:lo + 6] += np.asarray(c, np.float64) - lm[lo:lo + 6].mean(0)   # np.mean of the six points is the centre to the ulp
    lm[48], lm[54] = mouth_left, mouth_right
    return lm


# -------------------------------------------------------------------------------------------------------------------------------
# Lanczos shrink (Pillow Resample.c: precompute_coeffs, normalize_coeffs_8bpc, ImagingResample{Horizontal,Vertical}_8bpc)
# -------------------------------------------------------------------------------------------------------------------------------
def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


def lanczos_coeffs(in_size, out_size):
    """-> (xmin [out], taps [out], kk [out, ksize] int64): the 22-bit fixed-point taps of Pillow's LANCZOS resize along one axis"""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 3.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    xmin = np.zeros(out_size, np.int64)
    taps = np.zeros(out_size, np.int64)
    kk = np.zeros((out_size, ksize), np.int64)
    ss = 1.0 / fs
    for i in range(out_size):
        c = (i + 0.5) * scale
        lo = max(int(c - support + 0.5), 0)
        n = min(int(c + support + 0.5), in_size) - lo
        w = [_lanczos((x + lo - c + 0.5) * ss) for x in range(n)]
        tot = 0.0
        for v in w:
            tot += v
        for x, v in enumerate(w):
            v = v / tot if tot != 0.0 else v
            kk[i, x] = int(-0.5 + v * (1 << 22)) if v < 0 else int(0.5 + v * (1 << 22))
        xmin[i], taps[i] = lo, n
    return xmin, taps, kk


def _resample_axis(img, out_size, axis):
    xmin, taps, kk = lanczos_coeffs(img.shape[axis], out_size)
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    out = np.empty((out_size,) + src.shape[1:], np.uint8)
    for i in range(out_size):
        acc = (1 << 21) + np.tensordot(kk[i, :taps[i]], src[xmin[i]:xmin[i] + taps[i]], axes=(0, 0))
        out[i] = np.clip(acc >> 22, 0, 255)
    return np.moveaxis(out, 0, axis)


def lanczos_resize(img, size):
    """Pillow ``Image.fromarray(img).resize(size, LANCZOS)`` of a uint8 [H, W, 3] image; size = (width, height)"""
    return _resample_axis(_resample_axis(img, size[0], 1), size[1], 0)


# -------------------------------------------------------------------------------------------------------------------------------
# padded blur (np.pad 'reflect', scipy.ndimage.gaussian_filter), the two blends, the median and the quantisation
# -------------------------------------------------------------------------------------------------------------------------------
def reflect101(i, n):
    """np.pad 'reflect' source index of padded index i (repeated reflection for pads wider than the image)"""
    if n == 1:
        return np.zeros_like(i)
    p = 2 * n - 2
    j = np.mod(i, p)
    return np.where(j >= n, p - j, j)


def reflect_pad(img, pad):
    """np.pad(np.float32(img), ((pad[1], pad[3]), (pad[0], pad[2]), (0, 0)), 'reflect') with pad = (left, top, right, bottom)"""
    h, w = img.shape[:2]
    rows = reflect101(np.arange(-pad[1], h + pad[3]), h)
    cols = reflect101(np.arange(-pad[0], w + pad[2]), w)
    return img.astype(np.float32)[rows][:, cols]


def gaussian_weights(sigma):
    """scipy.ndimage's 1-D Gaussian (truncate 4): [w_0, w_1, ..., w_r] float64"""
    r = int(4.0 * float(sigma) + 0.5)
    x = np.arange(-r, r + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    phi = phi / phi.sum()
    return phi[r:]


def gaussian_axis(img, sigma, axis):
    """one axis of scipy.ndimage.gaussian_filter on float32: per output, in double, w0 x0 + sum_{k=r..1} (x_-k + x_+k) w_k, with
    the half-sample symmetric ('reflect') boundary; stored as float32"""
    w = gaussian_weights(sigma)
    r = len(w) - 1
    x = np.moveaxis(img, axis, 0).astype(np.float64)
    n = x.shape[0]
    period = 2 * n
    idx = np.mod(np.arange(-r, n + r), period)
    idx = np.where(idx >= n, period - 1 - idx, idx)
    ext = x[idx]
    acc = ext[r:r + n] * w[0]
    for k in range(r, 0, -1):
        acc = acc + (ext[r - k:r - k + n] + ext[r + k:r + k + n]) * w[k]
    return np.moveaxis(acc.astype(np.float32), 0, axis)


def pad_mask(h, w, pad):
    """the reference's [h, w, 1] float64 mask of the padded image"""
    y, x, _ = np.ogrid[:h, :w, :1]
    p = np.asarray(pad, np.int64)
    return np.maximum(1.0 - np.minimum(np.float32(x) / p[0], np.float32(w - 1 - x) / p[2]),
                      1.0 - np.minimum(np.float32(y) / p[1], np.float32(h - 1 - y) / p[3]))


def blend(img, target, weight):
    """img + (target - img) * weight: float32 difference, float64 product and sum, rounded to float32"""
    out = img.copy()
    out += (target - img) * weight
    return out


def median(img):
    """np.median over the two image axes: float32 [3]"""
    return np.median(img, axis=(0, 1))


def quantize(img):
    return np.uint8(np.clip(np.rint(img), 0, 255))


def padded_blur(img, pad, sigma):
    """the reference's pad branch from the cropped uint8 image to the padded uint8 image"""
    x = reflect_pad(img, pad)
    h, w, _ = x.shape
    mask = pad_mask(h, w, pad)
    g = gaussian_axis(gaussian_axis(x, sigma, 0), sigma, 1)
    x = blend(x, g, np.clip(mask * 3.0 + 1.0, 0.0, 1.0))
    x = blend(x, median(x), np.clip(mask, 0.0, 1.0))
    return quantize(x)


# -------------------------------------------------------------------------------------------------------------------------------
# quad warp (Pillow Image.transform QUAD: quad_transform, bilinear_filter32RGB)
# -------------------------------------------------------------------------------------------------------------------------------
def quad_coeffs(corners, size=OUT):
    """the 8 float64 coefficients Pillow derives from the NW, SW, SE, NE corners (flattened x, y pairs)"""
    c = [float(v) for v in np.asarray(corners, np.float64).reshape(8)]
    x0, y0, swx, swy, sex, sey, nex, ney = c
    a = 1.0 / size
    return np.array([x0, (nex - x0) * a, (swx - x0) * a, (sex - swx - nex + x0) * a * a,
                     y0, (ney - y0) * a, (swy - y0) * a, (sey - swy - ney + y0) * a * a])


def quad_warp(img, corners, size=OUT):
    """Pillow ``Image.fromarray(img).transform((size, size), QUAD, corners, BILINEAR)`` of a uint8 [H, W, 3] image"""
    a = quad_coeffs(corners, size)
    H, W = img.shape[:2]
    v, u = np.mgrid[:size, :size].astype(np.float64) + 0.5
    xs = a[0] + a[1] * u + a[2] * v + a[3] * u * v
    ys = a[4] + a[5] * u + a[6] * v + a[7] * u * v
    inside = (xs >= 0) & (xs < W) & (ys >= 0) & (ys < H)
    xs, ys = xs - 0.5, ys - 0.5
    x = np.where(xs < 0, np.floor(xs), np.trunc(xs)).astype(np.int64)
    y = np.where(ys < 0, np.floor(ys), np.trunc(ys)).astype(np.int64)
    dx, dy = (xs - x)[..., None], (ys - y)[..., None]
    x0, x1 = np.clip(x, 0, W - 1), np.clip(x + 1, 0, W - 1)
    src = img.astype(np.int64)
    y0, y1 = np.clip(y, 0, H - 1), np.clip(y + 1, 0, H - 1)
    v1 = src[y0, x0] + (src[y0, x1] - src[y0, x0]) * dx
    v2 = src[y1, x0] + (src[y1, x1] - src[y1, x0]) * dx
    v2 = np.where(((y + 1 >= 0) & (y + 1 < H))[..., None], v2, v1)
    out = v1 + (v2 - v1) * dy
    out = np.where(inside[..., None], out, 0.0)
    return out.astype(np.uint8)


def align(img, p):
    """the reference's align_face image path for the geometry record p of vtoonify_b200.align.align_params"""
    if p.shrink > 1:
        img = lanczos_resize(img, p.rsize)
    if p.crop is not None:
        x0, y0, x1, y1 = p.crop
        img = img[y0:y1, x0:x1]
    if p.pad is not None:
        img = padded_blur(img, p.pad, p.blur)
    return quad_warp(img, p.corners)
