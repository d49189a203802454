"""Generates tests/golden/augment_sampler.npz and augment_{a,odd,id,zoom}.npz from the UNMODIFIED reference model/simple_augment.py
on the CPU, with model.stylegan.op pointed at the reference's op_cpu.  ``F`` inside the reference module is wrapped so that the pads
it passes to F.pad and the theta it passes to F.affine_grid are recorded; both calls still run as they are.

- augment_sampler.npz: per case (p, B, H, W) from a seeded generator: G, the pads, theta, and the next 8 draws of torch.rand after the
  call.  The upfirdn2d passes do not affect any of these, so here they are replaced by a stub of the right output shape and the call
  stops at F.affine_grid.
- augment_<case>.npz: a float32 input, G, the reference's output on the input cast to float64 (out64), and its output on the float32
  input (out32, the yardstick of a float32 implementation).

    python tests/golden/make_golden_augment.py
"""
import os
import sys
import types

import numpy as np
import torch
from torch.nn import functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference")

import model.stylegan.op_cpu as op_cpu  # noqa: E402

sys.modules["model.stylegan.op"] = op_cpu
import model.simple_augment as sa  # noqa: E402

SAMPLER = [(p, B, H, W) for p in (0.0, 0.2, 1.0) for B in (1, 8) for (H, W) in ((1024, 1024), (640, 896))]
# name: (shape, p, input seed, sampler seed (None: the first that transforms every sample), given G)
IMAGES = {
    "a": ((2, 6, 64, 48), 0.2, 11, None, None),
    "odd": ((1, 3, 50, 38), 1.0, 12, 3, None),
    "id": ((2, 3, 40, 56), 0.0, 13, 5, None),
    "zoom": ((1, 3, 40, 40), None, 14, None, "zoom"),
}


class _Stop(Exception):
    pass


def _record(rec, stop):
    def pad(x, p, mode):
        rec["pads"] = np.array([int(v) for v in p], dtype=np.int32)
        return F.pad(x, p, mode=mode)

    def affine_grid(theta, size, align_corners):
        rec["theta"] = theta.float().numpy().copy()
        if stop:
            raise _Stop
        return F.affine_grid(theta, size, align_corners=align_corners)

    return types.SimpleNamespace(pad=pad, affine_grid=affine_grid, grid_sample=F.grid_sample)


def _shape_only_upfirdn2d(x, kernel, up=1, down=1, pad=(0, 0)):
    up_x, up_y = (up, up) if isinstance(up, int) else up
    down_x, down_y = (down, down) if isinstance(down, int) else down
    _, _, H, W = x.shape
    kh, kw = kernel.shape
    return x.new_zeros(x.shape[0], x.shape[1], (H * up_y + pad[2] + pad[3] - kh + down_y) // down_y,
                       (W * up_x + pad[0] + pad[1] - kw + down_x) // down_x)


def sampler():
    out = {}
    real_up = sa.upfirdn2d
    sa.upfirdn2d = _shape_only_upfirdn2d
    try:
        for n, (p, B, H, W) in enumerate(SAMPLER):
            rec = {}
            sa.F = _record(rec, stop=True)
            torch.manual_seed(100 + n)
            try:
                sa.random_apply_affine(torch.zeros(B, 1, H, W), p, None)
            except _Stop:
                pass
            G = rec_G[0]
            key = f"c{n}_"
            out[key + "cfg"] = np.array([p, B, H, W, 100 + n], dtype=np.float64)
            out[key + "G"] = G
            out[key + "pads"] = rec["pads"]
            out[key + "theta"] = rec["theta"]
            out[key + "next"] = torch.rand(8).numpy()
    finally:
        sa.upfirdn2d = real_up
        sa.F = F
    np.savez(os.path.join(HERE, "augment_sampler.npz"), **out)


rec_G = [None]


def _capture_G():
    """wrap try_sample_affine_and_pad so the sampled G is kept even when the call stops early"""
    real = sa.try_sample_affine_and_pad

    def wrapped(img, p, kernel_size, G=None):
        r = real(img, p, kernel_size, G)
        rec_G[0] = r[1].numpy().copy()
        return r
    sa.try_sample_affine_and_pad = wrapped


def zoom_G():
    c, s = np.cos(0.1), np.sin(0.1)
    return torch.tensor([[[5.5 * c, -5.5 * s, 0.3], [5.5 * s, 5.5 * c, -0.2], [0, 0, 1]]], dtype=torch.float32)


def images():
    for name, (shape, p, img_seed, seed, given) in IMAGES.items():
        img = torch.randn(shape, generator=torch.Generator().manual_seed(img_seed))
        if given == "zoom":
            G = zoom_G()
        else:
            s = 0 if seed is None else seed
            while True:
                torch.manual_seed(s)
                G = torch.inverse(sa.sample_affine(p, shape[0], shape[2], shape[3]))
                if seed is not None or all(not torch.equal(g, torch.eye(3)) for g in G):
                    break
                s += 1
            torch.manual_seed(s)
            _, G2 = sa.random_apply_affine(img.double(), p, None)
            assert torch.equal(G, G2)
            seed = s
        out64, _ = sa.random_apply_affine(img.double(), p, G)
        out32, _ = sa.random_apply_affine(img, p, G)
        rel = ((out32.double() - out64).norm() / out64.norm()).item()
        print(f"{name}: {tuple(shape)} p={p} seed={seed} fp32 yardstick rel L2 {rel:.3e} max {(out32.double() - out64).abs().max():.3e}")
        np.savez(os.path.join(HERE, f"augment_{name}.npz"), img=img.numpy(), G=G.numpy(), out64=out64.numpy(), out32=out32.numpy(),
                 p=np.float64(-1 if p is None else p), seed=np.int64(-1 if seed is None else seed))


if __name__ == "__main__":
    _capture_G()
    sampler()
    images()
