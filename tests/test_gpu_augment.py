"""GPU: vtoonify_b200.simple_augment.random_apply_affine against the reference's float64 output (tests/golden/augment_*.npz) and the
float64 restatement (tests/oracle_augment.py) run on the device, on the fused route and the unfused one.

Bars: relative L2 and max |err| at most twice the reference's own float32 yardstick (its float32 output against its float64 output on
the same case).  Cases without a fixture (training size, shape grid) use twice the worst yardstick of the fixtures, whose inputs have
the same N(0, 1) scale.  Each test prints its measured errors."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from tests import oracle_augment as O
from vtoonify_b200 import _lib
from vtoonify_b200 import simple_augment as A

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = torch.device("cuda", 0)


def load(case):
    z = np.load(os.path.join(GOLDEN, f"augment_{case}.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def errors(out, ref):
    d = out.double() - ref.double()
    return (d.norm() / ref.double().norm()).item(), d.abs().max().item()


def yardstick(f):
    return errors(f["out32"], f["out64"])


def worst_yardstick():
    ys = [yardstick(load(c)) for c in ("a", "odd", "id", "zoom")]
    return max(r for r, _ in ys), max(m for _, m in ys)


def route(img, G):
    _, _, H, W = img.shape
    pads = tuple(int(v) for v in A.padding(G, H, W))
    return A.plan(A.warp_coefficients(A.sampling_matrix(G, pads, H, W), pads, H, W), H, W)[0]


def unfused(img, G):
    _, _, H, W = img.shape
    pads = tuple(int(v) for v in A.padding(G, H, W))
    k = torch.as_tensor(A.SYM6).to(img)
    return A._unfused(img, k, pads, A.sampling_matrix(G, pads, H, W))


@pytest.mark.parametrize("case", ["a", "odd", "id", "zoom"])
def test_matches_reference_fixture(case):
    f = load(case)
    img = f["img"].to(DEV)
    fused = case != "zoom"
    assert (route(img, f["G"]) > 0) == fused
    n0 = _lib.launch_count()
    with torch.no_grad():
        out, G = A.random_apply_affine(img, float(f["p"]), f["G"])
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    assert G is f["G"] and out.shape == img.shape and out.dtype == torch.float32
    y_rel, y_max = yardstick(f)
    rel, mx = errors(out.cpu(), f["out64"])
    print(f"{case} ({'fused' if fused else 'unfused'}): rel L2 {rel:.3e} max {mx:.3e}; yardstick {y_rel:.3e} / {y_max:.3e}")
    assert rel <= 2 * y_rel and mx <= 2 * y_max
    if fused:
        assert launches == 1
        # the unfused route on the same transform meets the same bars
        rel, mx = errors(unfused(img, f["G"]).cpu(), f["out64"])
        print(f"{case} (unfused): rel L2 {rel:.3e} max {mx:.3e}")
        assert rel <= 2 * y_rel and mx <= 2 * y_max


def test_matches_oracle_on_device_in_float64():
    """the fixture's float64 output is reproduced by the restatement run on the device (the yardstick of the larger tests)"""
    f = load("odd")
    ref = O.apply(f["img"].to(DEV).double(), f["G"])
    assert (ref.cpu() - f["out64"]).abs().max().item() <= 1e-12


def _training_G(seed, B, H, W, p=0.2):
    torch.manual_seed(seed)
    return torch.inverse(A.sample_affine(p, B, H, W))


def _median_pad_seed(B, H, W):
    """the first seed whose batch-wide pad is near the median of the training transforms (about 183 px per side at 1024^2)"""
    for seed in range(200):
        pads = A.padding(_training_G(seed, B, H, W), H, W)
        if 160 <= max(int(v) for v in pads) <= 210:
            return seed
    raise AssertionError("no seed near the median pad")


def test_training_size_against_float64_oracle():
    B, C, H, W = 8, 6, 1024, 1024
    bar_rel, bar_max = worst_yardstick()
    g = torch.Generator(device=DEV).manual_seed(0)
    img = torch.randn(B, C, H, W, device=DEV, generator=g)
    median = _median_pad_seed(B, H, W)
    seeds = [median] + [s for s in (1, 3) if s != median]
    for seed in seeds:
        G = _training_G(seed, B, H, W)
        pads = tuple(int(v) for v in A.padding(G, H, W))
        assert route(img, G) > 0
        with torch.no_grad():
            out, _ = A.random_apply_affine(img, 0.2, G)
            ref = O.apply(img.double(), G)
        rel, mx = errors(out, ref)
        print(f"seed {seed} pads {pads}: rel L2 {rel:.3e} max {mx:.3e} (bars {2 * bar_rel:.3e} / {2 * bar_max:.3e})")
        assert rel <= 2 * bar_rel and mx <= 2 * bar_max
        del ref


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("C", [1, 3, 6])
@pytest.mark.parametrize("HW", [(37, 61), (64, 48), (130, 96)])
def test_shapes_against_float64_oracle(B, C, HW):
    H, W = HW
    bar_rel, bar_max = worst_yardstick()
    img = torch.randn(B, C, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(B * 100 + C * 10 + H))
    torch.manual_seed(1000 + B + C + H)
    with torch.no_grad():
        out, G = A.random_apply_affine(img, 1.0)
    ref = O.apply(img.double(), G)
    rel, mx = errors(out, ref)
    print(f"B={B} C={C} {H}x{W}: tile {route(img, G)} rel L2 {rel:.3e} max {mx:.3e}")
    assert route(img, G) > 0
    assert rel <= 2 * bar_rel and mx <= 2 * bar_max


@pytest.mark.parametrize("scale,aniso,rot,tile", [(2.0, 1.0, 0.4, 16), (2.6, 1.1, 0.3, 8), (3.0, 1.0, 0.5, 8),
                                                    (3.5, 1.2, 0.2, 8)])
def test_large_given_scales_on_both_tiles(scale, aniso, rot, tile):
    """given G that zoom out 2x to 3.5x, rotated and anisotropic: the fused route with the largest windows the planner sizes, on
    T = 16 and on T = 8, against the float64 restatement"""
    B, C, H, W = 2, 3, 96, 80
    bar_rel, bar_max = worst_yardstick()
    c, r = math.cos(rot), math.sin(rot)
    G = torch.tensor([[[scale * aniso * c, -scale * r, 1.5], [scale * aniso * r, scale * c / aniso, -2.0], [0, 0, 1]]],
                     dtype=torch.float32).repeat(B, 1, 1)
    G[1, :2, :2] *= 0.9
    img = torch.randn(B, C, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(int(scale * 10)))
    assert route(img, G) == tile
    n0 = _lib.launch_count()
    out, _ = A.random_apply_affine(img, 0.2, G)
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == 1
    rel, mx = errors(out, O.apply(img.double(), G))
    print(f"scale {scale} aniso {aniso} rot {rot}: tile {tile} rel L2 {rel:.3e} max {mx:.3e}")
    assert rel <= 2 * bar_rel and mx <= 2 * bar_max


def test_one_launch_bit_identical_reruns_and_layouts():
    B, C, H, W = 8, 6, 256, 192
    img = torch.randn(B, C, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    G = _training_G(4, B, H, W, p=1.0)
    n0 = _lib.launch_count()
    a, _ = A.random_apply_affine(img, 1.0, G)
    b, _ = A.random_apply_affine(img, 1.0, G)
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == 2
    assert torch.equal(a, b)
    c, _ = A.random_apply_affine(img.to(memory_format=torch.channels_last), 1.0, G)
    assert torch.equal(a, c)
    req = img.clone().requires_grad_()
    with torch.no_grad():
        d, _ = A.random_apply_affine(req, 1.0, G)
    assert torch.equal(a, d)


def test_guard_regions_untouched():
    B, C, H, W = 2, 3, 45, 70
    img = torch.randn(B, C, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    G = _training_G(6, B, H, W, p=1.0)
    pads = tuple(int(v) for v in A.padding(G, H, W))
    coef = A.warp_coefficients(A.sampling_matrix(G, pads, H, W), pads, H, W)
    tile, win_w, win_h = A.plan(coef, H, W)
    assert tile > 0
    n, guard = B * C * H * W, 4096
    buf = torch.full((n + 2 * guard,), 1234.5, device=DEV)
    k = torch.as_tensor(A.SYM6, dtype=torch.float32, device=DEV)
    x1, x2, y1, y2 = pads
    _lib.check(_lib.load().vt_augment_affine_f32(img.data_ptr(), buf[guard:].data_ptr(), k.data_ptr(), coef.to(DEV).data_ptr(), B, C, H,
                                                 W, x1, y1, H + y1 + y2, W + x1 + x2, tile, win_w, win_h,
                                                 torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.all(buf[:guard] == 1234.5) and torch.all(buf[guard + n:] == 1234.5)
    ref, _ = A.random_apply_affine(img, 1.0, G)
    assert torch.equal(buf[guard:guard + n].view(B, C, H, W), ref)


def test_launch_argument_errors():
    lib = _lib.load()
    x = torch.zeros(1, 1, 8, 8, device=DEV)
    k = torch.zeros(12, device=DEV)
    coef = torch.zeros(1, 6, dtype=torch.float64, device=DEV)
    args = [x.data_ptr(), x.data_ptr(), k.data_ptr(), coef.data_ptr(), 1, 1, 8, 8, 6, 6, 20, 20]
    s = torch.cuda.current_stream().cuda_stream
    assert lib.vt_augment_affine_f32(*args, 12, 40, 40, s) != 0 and b"tile" in lib.vt_last_error()
    assert lib.vt_augment_affine_f32(*args, 16, 400, 400, s) != 0 and b"window" in lib.vt_last_error()
    bad = list(args)
    bad[8] = 8                                      # a reflect pad as wide as the image
    assert lib.vt_augment_affine_f32(*bad, 16, 40, 40, s) != 0 and b"reflect" in lib.vt_last_error()
    with pytest.raises(_lib.VtError, match="float32"):
        A.random_apply_affine(x.double(), 0.2)
