"""FFHQ face alignment (vtoonify_b200.align.align_faces) on the device against the same operations through Pillow, SciPy and NumPy on
the host CPU, and the style-code chain of style_transfer.py:138-144 (align, pSp, zplus2wplus).

Workloads: the frame (crop only), border (pad branch) and shrink (Lanczos shrink, then the pad branch) geometries of
tests/golden/make_golden_align.py on their seeded synthetic images, one image per call, and a batch of 16 images cycling through the
three.  Images are already on the device (uint8), so no host-to-device copy is timed.
- device: CUDA events around each call, median of --steps calls after --warmup calls; also the library launches per call;
- cpu:    the reference's statements (Pillow resize / crop / transform, np.pad, scipy.ndimage.gaussian_filter, np.median) on the
          geometry of align_params, wall clock, median of --cpu-steps calls, with the host's usable core count.
Then the chain at N = 1 and 16 on the frame geometry: align_faces, frames_u8_to_f32, pSp (GradualStyleEncoder, det_state_dict weights)
and VToonify.zplus2wplus, CUDA events, median of --steps.  One JSON line per measurement; the last line holds the card's name, power
limit and top SM clock from nvidia-smi, read in the same call.

    python tools/align_bench.py --steps 20 --warmup 3
"""
import argparse
import json
import os
import subprocess
import sys
import time
from argparse import Namespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import oracle_align as O  # noqa: E402
from vtoonify_b200 import _lib, align as A, ops  # noqa: E402

GEOMETRIES = ("frame", "border", "shrink")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def load_case(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", f"align_{name}.npz"))
    return O.synth_image(int(g["image_seed"]), *g["image_hw"]), g["landmarks"]


def cpu_align(img, lm):
    """the reference's image statements on Pillow, NumPy and SciPy, from the host geometry"""
    import PIL.Image
    import scipy.ndimage
    p = A.align_params(lm, img.shape[:2])
    im = PIL.Image.fromarray(img)
    if p.shrink > 1:
        im = im.resize(p.rsize, PIL.Image.LANCZOS)
    if p.crop is not None:
        im = im.crop(p.crop)
    if p.pad is not None:
        x = np.pad(np.float32(im), ((p.pad[1], p.pad[3]), (p.pad[0], p.pad[2]), (0, 0)), "reflect")
        h, w, _ = x.shape
        mask = O.pad_mask(h, w, p.pad)
        x += (scipy.ndimage.gaussian_filter(x, [p.blur, p.blur, 0]) - x) * np.clip(mask * 3.0 + 1.0, 0.0, 1.0)
        x += (np.median(x, axis=(0, 1)) - x) * np.clip(mask, 0.0, 1.0)
        im = PIL.Image.fromarray(np.uint8(np.clip(np.rint(x), 0, 255)), "RGB")
    return np.asarray(im.transform((256, 256), PIL.Image.QUAD, tuple(p.corners.tolist()), PIL.Image.BILINEAR))


def time_device(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), float(min(times)), float(max(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("align_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cores = len(os.sched_getaffinity(0))
    cases = {n: load_case(n) for n in GEOMETRIES}

    def run(name, imgs, lms):
        dimgs = [torch.from_numpy(i).to(dev) for i in imgs]
        lms = np.stack(lms)
        n0 = _lib.launch_count()
        want = A.align_faces(dimgs, lms)
        launches = _lib.launch_count() - n0
        for i, (img, lm) in enumerate(zip(imgs, lms)):
            assert np.array_equal(want[i].cpu().numpy(), cpu_align(img, lm)), f"{name}: device and CPU differ"
        med, lo, hi = time_device(lambda: A.align_faces(dimgs, lms), args.steps, args.warmup)
        cpu = []
        for _ in range(max(1, args.cpu_steps)):
            t = time.perf_counter()
            for img, lm in zip(imgs, lms):
                cpu_align(img, lm)
            cpu.append((time.perf_counter() - t) * 1e3)
        print(json.dumps({"workload": name, "images": len(imgs), "shapes": sorted({i.shape[:2] for i in imgs}),
                          "device_ms": round(med, 4), "device_ms_min": round(lo, 4), "device_ms_max": round(hi, 4),
                          "device_ms_per_image": round(med / len(imgs), 4), "launches_per_call": launches,
                          "cpu_ms": round(float(np.median(cpu)), 3), "cpu_ms_per_image": round(float(np.median(cpu)) / len(imgs), 3),
                          "cpu_cores": cores, "speedup": round(float(np.median(cpu)) / med, 1)}), flush=True)

    for n in GEOMETRIES:
        run(n, [cases[n][0]], [cases[n][1]])
    order = [GEOMETRIES[i % 3] for i in range(16)]
    run("batch16", [cases[n][0] for n in order], [cases[n][1] for n in order])

    # the style-code chain
    from vtoonify_b200.psp import GradualStyleEncoder
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict
    with torch.no_grad():
        psp = GradualStyleEncoder(50, "ir_se", Namespace(input_nc=3, n_styles=18)).eval()
        psp.load_state_dict(det_state_dict(psp, seed=11), strict=True)
        psp.to(dev)
        vt = VToonify(backbone="dualstylegan").eval()
        vt.load_state_dict(det_state_dict(vt, seed=0), strict=True)
        vt.to(dev)
        img, lm = cases["frame"]
        for N in (1, 16):
            dimgs = [torch.from_numpy(img).to(dev)] * N
            lms = np.stack([lm] * N)

            def chain():
                return vt.zplus2wplus(psp(ops.frames_u8_to_f32(A.align_faces(dimgs, lms))))
            s_w = chain()
            assert tuple(s_w.shape) == (N, 18, 512)
            med, lo, hi = time_device(chain, args.steps, args.warmup)
            al, _, _ = time_device(lambda: A.align_faces(dimgs, lms), args.steps, args.warmup)
            print(json.dumps({"workload": f"style_code_chain_N{N}", "chain_ms": round(med, 3), "chain_ms_min": round(lo, 3),
                              "chain_ms_max": round(hi, 3), "align_ms": round(al, 4), "align_share": round(al / med, 4),
                              "precision": ops.get_precision()}), flush=True)
    print(json.dumps({"card": card(), "note": "card name, power limit and max SM clock from nvidia-smi in the same call"}))


if __name__ == "__main__":
    main()
