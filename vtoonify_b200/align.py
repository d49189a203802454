"""FFHQ face alignment on the device: the image path of the reference's ``align_face`` (model/encoder/align_all_parallel.py:59-150),
byte for byte, from the 68 dlib landmarks the caller supplies.

``align_faces(images, landmarks) -> CUDA uint8 [N, 256, 256, 3]``: per image, ``align_params`` restates the reference's geometry in
float64 NumPy on the host (landmarks and image size in, shrink / crop / pad / warp corners out), and the image stages run as CUDA
kernels (csrc/align.cu) enqueued on the current stream with no host synchronisation:

- shrink (only when ``shrink > 1``): Pillow ``resize(LANCZOS)``, one launch per axis, from 22-bit fixed-point tap tables built here;
- crop: a pointer offset into the (shrunk) image;
- pad (only when the padding test triggers): the reflect pad stays virtual; the Gaussian blur (rows, then columns with the first blend),
  the per-channel median (an exact radix select) and the second blend with ``np.rint`` quantisation;
- warp: Pillow ``transform(QUAD, BILINEAR)`` to 256 x 256.

dlib's detection and landmark regression (``get_landmark``) stay the caller's.  Forward only; output size 256 only (the reference fixes
``output_size = transform_size = 256``, so its final ANTIALIAS resize never runs).
"""
import ctypes
import math
from typing import NamedTuple, Optional, Tuple

import numpy as np
import torch

from . import _lib, ops

OUT = 256
INT32_LIMIT = 2 ** 31 - 1


class AlignParams(NamedTuple):
    """The reference's geometry for one image.  ``rsize`` (width, height) is set when ``shrink > 1``; ``crop`` (x0, y0, x1, y1) when
    the crop is smaller than the image; ``pad`` (left, top, right, bottom) and ``blur`` (the Gaussian's sigma) when padding triggers.
    ``size`` (height, width) is the image the warp reads, and ``corners`` the warp's NW, SW, SE, NE corners (x, y) in it."""
    shrink: int
    rsize: Optional[Tuple[int, int]]
    crop: Optional[Tuple[int, int, int, int]]
    pad: Optional[Tuple[int, int, int, int]]
    blur: Optional[float]
    qsize: float
    size: Tuple[int, int]
    corners: np.ndarray


def _landmarks(lm):
    if isinstance(lm, torch.Tensor):
        lm = lm.detach().cpu().numpy()
    lm = np.asarray(lm)
    if lm.shape != (68, 2) or not np.issubdtype(lm.dtype, np.number) or not np.all(np.isfinite(lm)):
        raise ValueError(f"align_params: landmarks must be a finite [68, 2] array (got shape {lm.shape}, dtype {lm.dtype})")
    return lm.astype(np.float64)


def _box(quad):
    return (int(np.floor(min(quad[:, 0]))), int(np.floor(min(quad[:, 1]))), int(np.ceil(max(quad[:, 0]))),
            int(np.ceil(max(quad[:, 1]))))


def align_params(landmarks, image_hw) -> AlignParams:
    """The reference's float64 arithmetic from 68 landmarks and the image's (height, width) to the warp parameters."""
    lm = _landmarks(landmarks)
    h, w = (int(v) for v in image_hw)
    if h < 1 or w < 1:
        raise ValueError(f"align_params: empty image {h} x {w}")
    # the oriented rectangle: only the eye centres and the mouth corners are read
    eye_l, eye_r = np.mean(lm[36:42], axis=0), np.mean(lm[42:48], axis=0)
    eye_avg = (eye_l + eye_r) * 0.5
    eye_to_eye = eye_r - eye_l
    mouth_avg = (lm[48] + lm[54]) * 0.5
    eye_to_mouth = mouth_avg - eye_avg
    x = eye_to_eye - np.flipud(eye_to_mouth) * [-1, 1]
    x /= np.hypot(*x)
    x *= max(np.hypot(*eye_to_eye) * 2.0, np.hypot(*eye_to_mouth) * 1.8)
    y = np.flipud(x) * [-1, 1]
    c = eye_avg + eye_to_mouth * 0.1
    quad = np.stack([c - x - y, c - x + y, c + x + y, c + x - y])
    qsize = np.hypot(*x) * 2

    shrink = int(np.floor(qsize / OUT * 0.5))
    rsize = None
    if shrink > 1:
        rsize = (int(np.rint(float(w) / shrink)), int(np.rint(float(h) / shrink)))
        w, h = rsize
        quad /= shrink
        qsize /= shrink

    border = max(int(np.rint(qsize * 0.1)), 3)
    b = _box(quad)
    crop = (max(b[0] - border, 0), max(b[1] - border, 0), min(b[2] + border, w), min(b[3] + border, h))
    if crop[2] - crop[0] < w or crop[3] - crop[1] < h:
        quad -= crop[0:2]
        w, h = crop[2] - crop[0], crop[3] - crop[1]
    else:
        crop = None

    b = _box(quad)
    pad = (max(-b[0] + border, 0), max(-b[1] + border, 0), max(b[2] - w + border, 0), max(b[3] - h + border, 0))
    blur = None
    if max(pad) > border - 4:
        least = int(np.rint(qsize * 0.3))
        if least == 0:
            raise ValueError(f"align_params: the face is too small to pad (qsize {qsize:.3g}; the reference divides by zero)")
        pad = tuple(int(v) for v in np.maximum(pad, least))
        blur = float(qsize * 0.02)
        quad += pad[:2]
        w, h = w + pad[0] + pad[2], h + pad[1] + pad[3]
    else:
        pad = None
    return AlignParams(shrink, rsize, crop, pad, blur, float(qsize), (h, w), (quad + 0.5).flatten())


# ---------------------------------------------------------------------------------------------------------------------------------
# host tables of the kernels
# ---------------------------------------------------------------------------------------------------------------------------------
def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def lanczos_table(in_size: int, out_size: int):
    """-> (int32 [2 * out_size + out_size * ksize] table, ksize): first tap, tap count and the 22-bit fixed-point taps of each output
    of Pillow's LANCZOS resize along one axis (Resample.c precompute_coeffs / normalize_coeffs_8bpc, in float64 with the C library's
    sin)."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 3.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / fs
    tab = np.zeros(2 * out_size + out_size * ksize, np.int32)
    kk = tab[2 * out_size:].reshape(out_size, ksize)
    for i in range(out_size):
        c = (i + 0.5) * scale
        lo = max(int(c - support + 0.5), 0)
        n = min(int(c + support + 0.5), in_size) - lo
        k = []
        for j in range(n):
            t = (j + lo - c + 0.5) * ss
            k.append(_sinc(t) * _sinc(t / 3) if -3.0 <= t < 3.0 else 0.0)
        tot = 0.0
        for v in k:
            tot += v
        for j, v in enumerate(k):
            if tot != 0.0:
                v /= tot
            kk[i, j] = int(-0.5 + v * (1 << 22)) if v < 0 else int(0.5 + v * (1 << 22))
        tab[i], tab[out_size + i] = lo, n
    return tab, ksize


def gaussian_taps(sigma: float) -> np.ndarray:
    """float64 [r + 1]: the centre tap, then taps 1..r, of scipy.ndimage.gaussian_filter1d's kernel (truncate 4)"""
    r = int(4.0 * float(sigma) + 0.5)
    if r > _lib.VT_ALIGN_MAX_RADIUS:
        raise ValueError(f"align: blur radius {r} exceeds {_lib.VT_ALIGN_MAX_RADIUS}")
    xs = np.arange(-r, r + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * xs ** 2)
    phi = phi / phi.sum()
    return np.ascontiguousarray(phi[r:])


# ---------------------------------------------------------------------------------------------------------------------------------
# stage launches (also called by the stage tests)
# ---------------------------------------------------------------------------------------------------------------------------------
def _ints(v):
    return (ctypes.c_int * 4)(*[int(x) for x in v])


def _doubles(a):
    a = np.ascontiguousarray(a, np.float64)
    return (ctypes.c_double * a.size)(*a.tolist())


def _to_device(arr: np.ndarray, device):
    return torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)


def lanczos(src: torch.Tensor, size, pitch=None) -> torch.Tensor:
    """Pillow resize(size=(width, height), LANCZOS) of a CUDA uint8 [H, W, 3] image (rows ``pitch`` bytes apart)"""
    H, W = src.shape[0], src.shape[1]
    pitch = W * 3 if pitch is None else pitch
    lib, st = _lib.load(), ops._stream()
    tx, kx = lanczos_table(W, size[0])
    ty, ky = lanczos_table(H, size[1])
    tab = _to_device(np.concatenate([tx, ty]), src.device)
    tmp = torch.empty((H, size[0], 3), dtype=torch.uint8, device=src.device)
    _lib.check(lib.vt_align_lanczos_u8(src.data_ptr(), pitch, H, W, tmp.data_ptr(), size[0], 1, tab.data_ptr(), kx, st))
    out = torch.empty((size[1], size[0], 3), dtype=torch.uint8, device=src.device)
    _lib.check(lib.vt_align_lanczos_u8(tmp.data_ptr(), size[0] * 3, H, size[0], out.data_ptr(), size[1], 0,
                                       tab.data_ptr() + 4 * tx.size, ky, st))
    return out


def blur_rows(src: torch.Tensor, pad, sigma, hw=None, pitch=None) -> torch.Tensor:
    """float32 [Hp, Wp, 3]: axis 0 of gaussian_filter over np.pad(float32(src), pad, 'reflect'); src CUDA uint8 [H, W, 3] (or the
    ``hw`` window at src's data pointer, rows ``pitch`` bytes apart)"""
    H, W = (src.shape[0], src.shape[1]) if hw is None else hw
    pitch = src.shape[1] * 3 if pitch is None else pitch
    w = gaussian_taps(sigma)
    out = torch.empty((H + pad[1] + pad[3], W + pad[0] + pad[2], 3), dtype=torch.float32, device=src.device)
    _lib.check(_lib.load().vt_align_blur_rows_f32(src.data_ptr(), pitch, H, W, _ints(pad), out.data_ptr(), _doubles(w), len(w) - 1,
                                                  ops._stream()))
    return out


def blur_cols(x: torch.Tensor, sigma, img=None, pad=None, hw=None, pitch=None) -> torch.Tensor:
    """float32 [Hp, Wp, 3]: axis 1 of gaussian_filter over x; with ``img`` (the uint8 image under the pad, see blur_rows) the first
    blend of the padded image towards the blurred one instead"""
    Hp, Wp = x.shape[0], x.shape[1]
    w = gaussian_taps(sigma)
    out = torch.empty_like(x)
    if img is None:
        args = (None, 0, 0, 0, None)
    else:
        H, W = (img.shape[0], img.shape[1]) if hw is None else hw
        args = (img.data_ptr(), img.shape[1] * 3 if pitch is None else pitch, H, W, _ints(pad))
    _lib.check(_lib.load().vt_align_blur_cols_f32(x.data_ptr(), out.data_ptr(), Hp, Wp, _doubles(w), len(w) - 1, *args,
                                                  ops._stream()))
    return out


def median(x: torch.Tensor) -> torch.Tensor:
    """CUDA float32 [3]: np.median(x, axis=(0, 1)) of a CUDA float32 [..., 3] tensor"""
    lib = _lib.load()
    ws = torch.empty(int(lib.vt_align_median_ws_bytes()), dtype=torch.uint8, device=x.device)
    med = torch.empty(3, dtype=torch.float32, device=x.device)
    _lib.check(lib.vt_align_median_f32(x.data_ptr(), x.numel() // 3, med.data_ptr(), ws.data_ptr(), ops._stream()))
    return med


def finish(x: torch.Tensor, med: torch.Tensor, pad) -> torch.Tensor:
    """uint8 [Hp, Wp, 3]: the second blend of x towards med, np.rint, clamp"""
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    _lib.check(_lib.load().vt_align_finish_u8(x.data_ptr(), med.data_ptr(), out.data_ptr(), x.shape[0], x.shape[1], _ints(pad),
                                              ops._stream()))
    return out


def quad_coeffs(corners, size=OUT) -> np.ndarray:
    """Pillow's QUAD coefficients (x0, x_u, x_v, x_uv, y0, y_u, y_v, y_uv) from the NW, SW, SE, NE corners"""
    x0, y0, swx, swy, sex, sey, nex, ney = (float(v) for v in np.asarray(corners, np.float64).reshape(8))
    a = 1.0 / size
    return np.array([x0, (nex - x0) * a, (swx - x0) * a, (sex - swx - nex + x0) * a * a,
                     y0, (ney - y0) * a, (swy - y0) * a, (sey - swy - ney + y0) * a * a])


def warp(src: torch.Tensor, corners, out: Optional[torch.Tensor] = None, hw=None, pitch=None) -> torch.Tensor:
    """uint8 [256, 256, 3]: Pillow transform(QUAD, corners, BILINEAR) of a CUDA uint8 [H, W, 3] image (or window, see blur_rows)"""
    H, W = (src.shape[0], src.shape[1]) if hw is None else hw
    pitch = src.shape[1] * 3 if pitch is None else pitch
    if out is None:
        out = torch.empty((OUT, OUT, 3), dtype=torch.uint8, device=src.device)
    _lib.check(_lib.load().vt_align_warp_u8(src.data_ptr(), pitch, H, W, _doubles(quad_coeffs(corners)), out.data_ptr(), OUT,
                                            ops._stream()))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# public entry
# ---------------------------------------------------------------------------------------------------------------------------------
def _image_list(images):
    if isinstance(images, (np.ndarray, torch.Tensor)) and images.ndim == 4:
        return [images[i] for i in range(images.shape[0])]
    if isinstance(images, (list, tuple)):
        return list(images)
    raise ValueError("align_faces: images must be a list of [H, W, 3] uint8 images or one [N, H, W, 3] uint8 array or tensor")


def _check_image(img, i):
    if isinstance(img, np.ndarray):
        dtype_ok = img.dtype == np.uint8
    elif isinstance(img, torch.Tensor):
        dtype_ok = img.dtype == torch.uint8
    else:
        raise ValueError(f"align_faces: image {i} is a {type(img).__name__}, not a NumPy array or a tensor")
    if not dtype_ok:
        raise _lib.VtError(f"align_faces: image {i} must be uint8 (got {img.dtype})")
    if img.ndim != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
        raise _lib.VtError(f"align_faces: image {i} must be [H, W, 3] RGB (got shape {tuple(img.shape)})")
    if img.shape[0] * img.shape[1] * 3 > INT32_LIMIT:
        raise ValueError(f"align_faces: image {i} ({img.shape[0]} x {img.shape[1]}) is too large for int32 indexing")


def align_faces(images, landmarks) -> torch.Tensor:
    """CUDA uint8 [N, 256, 256, 3]: the reference's ``align_face`` of each RGB uint8 image (NumPy arrays or host / CUDA tensors, a list
    of [H, W, 3] or one [N, H, W, 3]) with its [68, 2] landmarks (``landmarks`` [N, 68, 2], on the host).  Images of different sizes are
    aligned one launch sequence each, all on the current stream, with no host synchronisation."""
    imgs = _image_list(images)
    if isinstance(landmarks, torch.Tensor):
        landmarks = landmarks.detach().cpu().numpy()
    landmarks = np.asarray(landmarks)
    if landmarks.ndim != 3 or landmarks.shape[1:] != (68, 2):
        raise ValueError(f"align_faces: landmarks must be [N, 68, 2] (got shape {landmarks.shape})")
    if len(imgs) != landmarks.shape[0]:
        raise ValueError(f"align_faces: {len(imgs)} images but {landmarks.shape[0]} landmark sets")
    if not imgs:
        raise ValueError("align_faces: no images")
    for i, img in enumerate(imgs):
        _check_image(img, i)
    devs = {img.device for img in imgs if isinstance(img, torch.Tensor) and img.is_cuda}
    if len(devs) > 1:
        raise ValueError(f"align_faces: images on several devices {sorted(str(d) for d in devs)}")
    device = devs.pop() if devs else torch.device("cuda", torch.cuda.current_device())
    params = [align_params(landmarks[i], img.shape[:2]) for i, img in enumerate(imgs)]
    for p in params:
        if p.size[0] * p.size[1] * 3 > INT32_LIMIT:
            raise ValueError(f"align_faces: padded image {p.size[0]} x {p.size[1]} is too large for int32 indexing")

    out = torch.empty((len(imgs), OUT, OUT, 3), dtype=torch.uint8, device=device)
    for i, (img, p) in enumerate(zip(imgs, params)):
        if isinstance(img, np.ndarray):
            img = torch.from_numpy(img)
        if img.is_cuda:
            src = img.contiguous()
        else:
            src = img.contiguous().pin_memory().to(device, non_blocking=True)
        if p.shrink > 1:
            src = lanczos(src, p.rsize)
        H, W = src.shape[0], src.shape[1]
        pitch = W * 3
        if p.crop is not None:
            x0, y0, x1, y1 = p.crop
            src = src[y0:y1, x0:x1]
            H, W = y1 - y0, x1 - x0
        if p.pad is not None:
            x = blur_cols(blur_rows(src, p.pad, p.blur, (H, W), pitch), p.blur, src, p.pad, (H, W), pitch)
            src = finish(x, median(x), p.pad)
            H, W = src.shape[0], src.shape[1]
            pitch = W * 3
        warp(src, p.corners, out[i], (H, W), pitch)
    return out
