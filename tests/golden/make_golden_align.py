"""Generates tests/golden/align_{frame,border,shrink,outside,small}.npz from the UNMODIFIED reference ``align_face``
(model/encoder/align_all_parallel.py:59-150) on the CPU, with three patches around it:
- a stub ``dlib`` module in sys.modules (the module imports dlib; the landmarks are given, so dlib is never called);
- ``get_landmark`` returns the case's landmarks;
- ``PIL.Image.ANTIALIAS = PIL.Image.LANCZOS`` (Pillow >= 10 removed the alias of the same filter).
The reference's intermediate geometry is recorded by wrapping, not replacing, the calls it makes: Image.resize (the shrunk size),
Image.crop (the box), np.pad (the pads), scipy.ndimage.gaussian_filter (the sigma) and Image.transform (the warp corners).

Each file holds the library versions, the seed and size of the synthetic input (tests/oracle_align.synth_image; the image itself is not
stored), the landmarks, the recorded geometry and the 256 x 256 uint8 output.

    python tests/golden/make_golden_align.py
"""
import os
import sys
import types

import numpy as np
import PIL
import PIL.Image
import scipy
import scipy.ndimage

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, "/root/reference")

from tests.oracle_align import synth_image, synth_landmarks  # noqa: E402

sys.modules["dlib"] = types.ModuleType("dlib")
PIL.Image.ANTIALIAS = PIL.Image.LANCZOS
import model.encoder.align_all_parallel as aap  # noqa: E402


def _rot(v, deg):
    t = np.deg2rad(deg)
    return np.array([np.cos(t) * v[0] - np.sin(t) * v[1], np.sin(t) * v[0] + np.cos(t) * v[1]])


def face(centre, eye_dist, angle, mouth_drop, seed):
    """landmarks of a face with the eye midpoint at centre, rotated by angle degrees"""
    c = np.asarray(centre, np.float64)
    el, er = c + _rot((-eye_dist / 2, 0), angle), c + _rot((eye_dist / 2, 0), angle)
    ml, mr = c + _rot((-eye_dist * 0.4, mouth_drop), angle), c + _rot((eye_dist * 0.4, mouth_drop), angle)
    return synth_landmarks(seed, el, er, ml, mr)


# name: (image seed, height, width, landmarks); what each covers is in DESIGN.md §15
CASES = {
    # a video frame (style_transfer.py:138-150): crop only
    "frame": (101, 400, 400, lambda: face((201.3, 170.6), 64.0, 3.0, 70.0, 1)),
    # face rotated by 25 degrees near the top-left corner: pad, blur, both blends, median
    "border": (102, 360, 480, lambda: face((70.2, 80.9), 56.0, 25.0, 60.0, 2)),
    # a large face: Lanczos shrink by 2, then the pad branch
    "shrink": (103, 856, 1280, lambda: face((610.4, 330.7), 262.0, -8.0, 280.0, 3)),
    # the quad 4 pixels inside the image's right edge after the crop, the widest reach that skips padding
    "outside": (104, 300, 420, lambda: face((315.75, 150.2), 50.0, 0.0, 55.0, 4)),
    # a face larger than a 97 x 80 image: pads wider than the image (repeated reflection), odd sizes, an even-count median
    "small": (105, 97, 80, lambda: face((41.3, 40.7), 60.0, -12.0, 64.0, 5)),
}


class Recorder:
    def __init__(self):
        self.rec = {}
        self._orig = {}

    def __enter__(self):
        rec = self.rec
        I = PIL.Image.Image
        self._orig = {"resize": I.resize, "crop": I.crop, "transform": I.transform, "pad": np.pad,
                      "gauss": scipy.ndimage.gaussian_filter}
        o = self._orig

        def resize(im, size, *a, **k):
            rec["rsize"] = np.array(size, np.int64)
            return o["resize"](im, size, *a, **k)

        def crop(im, box=None):
            rec["crop"] = np.array(box, np.int64)
            return o["crop"](im, box)

        def transform(im, size, method, data=None, *a, **k):
            rec["corners"] = np.array(data, np.float64)
            return o["transform"](im, size, method, data, *a, **k)

        def pad(arr, width, mode, **k):
            (t, b), (l, r), _ = width
            rec["pad"] = np.array([l, t, r, b], np.int64)
            return o["pad"](arr, width, mode, **k)

        def gauss(x, sigma, *a, **k):
            rec["blur"] = np.float64(sigma[0])
            return o["gauss"](x, sigma, *a, **k)

        I.resize, I.crop, I.transform = resize, crop, transform
        aap.np = types.SimpleNamespace(**{n: getattr(np, n) for n in dir(np) if not n.startswith("__")})
        aap.np.pad = pad
        aap.scipy = types.SimpleNamespace(ndimage=types.SimpleNamespace(gaussian_filter=gauss))
        return self

    def __exit__(self, *exc):
        I = PIL.Image.Image
        I.resize, I.crop, I.transform = self._orig["resize"], self._orig["crop"], self._orig["transform"]
        aap.np, aap.scipy = np, scipy
        return False


def run(img, lm):
    aap.get_landmark = lambda filepath, predictor: lm
    with Recorder() as r:
        out = aap.align_face(img, None)
    return np.asarray(out.convert("RGB")), r.rec


def main():
    for name, (seed, h, w, make_lm) in CASES.items():
        img = synth_image(seed, h, w)
        lm = make_lm()
        out, rec = run(img, lm)
        d = {"versions": np.array([np.__version__, scipy.__version__, PIL.__version__]),
             "image_seed": np.int64(seed), "image_hw": np.array([h, w], np.int64), "landmarks": lm, "out": out}
        for k in ("rsize", "crop", "pad", "blur", "corners"):
            if k in rec:
                d[k] = rec[k]
        np.savez_compressed(os.path.join(HERE, f"align_{name}.npz"), **d)
        print(name, {k: (v.tolist() if hasattr(v, "tolist") else v) for k, v in rec.items()})


if __name__ == "__main__":
    main()
