"""CPU: the host side of vtoonify_b200.simple_augment against the unmodified reference (tests/golden/augment_*.npz): the sampled G bit
for bit, the generator state after the call, the pads and the sampling matrix; the fused kernel's planner; the argument errors."""
import math
import os

import numpy as np
import pytest
import torch

from vtoonify_b200 import _lib
from vtoonify_b200 import simple_augment as A

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def sampler_cases():
    z = np.load(os.path.join(GOLDEN, "augment_sampler.npz"))
    names = sorted({k.split("_")[0] for k in z.files})
    return [{k.split("_", 1)[1]: z[k] for k in z.files if k.startswith(n + "_")} for n in names]


def image_case(name):
    z = np.load(os.path.join(GOLDEN, f"augment_{name}.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


SAMPLER = sampler_cases()


def test_sampler_fixtures_cover_the_issue_grid():
    cfg = {tuple(c["cfg"][:4]) for c in SAMPLER}
    assert {p for p, *_ in cfg} == {0.0, 0.2, 1.0} and {B for _, B, *_ in cfg} == {1, 8}
    assert (1024, 1024) in {(H, W) for *_, H, W in cfg} and any(H != W for *_, H, W in cfg)


@pytest.mark.parametrize("n", range(len(SAMPLER)))
def test_sampler_is_bit_identical(n):
    c = SAMPLER[n]
    p, B, H, W, seed = c["cfg"]
    B, H, W = int(B), int(H), int(W)
    torch.manual_seed(int(seed))
    G = torch.inverse(A.sample_affine(float(p), B, H, W))
    assert G.dtype == torch.float32 and G.shape == (B, 3, 3)
    assert np.array_equal(G.numpy().view(np.uint32), c["G"].view(np.uint32))
    # the generator is left where the reference leaves it: every later draw of the training loop is unchanged
    assert np.array_equal(torch.rand(8).numpy(), c["next"])
    pads = tuple(int(v) for v in A.padding(G, H, W))
    assert pads == tuple(int(v) for v in c["pads"])
    theta = A.sampling_matrix(G, pads, H, W)[:, :2, :]
    assert np.array_equal(theta.numpy().view(np.uint32), c["theta"].view(np.uint32))
    if p == 0:
        assert pads == (6, 6, 6, 6) and torch.equal(G, torch.eye(3).expand(B, 3, 3))


def test_coefficients_restate_affine_grid_and_grid_sample():
    """x2-image pixel coordinates of the warp grid from the coefficients == torch's unnormalised affine_grid, in float64"""
    for c in SAMPLER[:6]:
        p, B, H, W, _ = c["cfg"]
        B, H, W = int(B), int(H), int(W)
        G = torch.from_numpy(c["G"])
        pads = tuple(int(v) for v in c["pads"])
        theta = A.sampling_matrix(G, pads, H, W)
        gh, gw = (H + 6) * 2, (W + 6) * 2
        uh, uw = (H + pads[2] + pads[3]) * 2, (W + pads[0] + pads[1]) * 2
        grid = torch.nn.functional.affine_grid(theta[:, :2, :].double(), (B, 1, gh, gw), align_corners=False)
        ix, iy = ((grid[..., 0] + 1) * uw - 1) / 2, ((grid[..., 1] + 1) * uh - 1) / 2
        coef = A.warp_coefficients(theta, pads, H, W)
        j = torch.arange(gw, dtype=torch.float64).view(1, 1, gw)
        i = torch.arange(gh, dtype=torch.float64).view(1, gh, 1)
        cx = coef[:, None, None, :]
        assert torch.allclose(cx[..., 0] + cx[..., 1] * j + cx[..., 2] * i, ix, rtol=0, atol=1e-9)
        assert torch.allclose(cx[..., 3] + cx[..., 4] * j + cx[..., 5] * i, iy, rtol=0, atol=1e-9)


def _coef(G, H, W):
    pads = tuple(int(v) for v in A.padding(G, H, W))
    return A.warp_coefficients(A.sampling_matrix(G, pads, H, W), pads, H, W)


def test_planner_takes_the_fused_route_for_every_fixture_transform():
    for c in SAMPLER:
        _, _, H, W, _ = c["cfg"]
        tile, win_w, win_h = A.plan(_coef(torch.from_numpy(c["G"]), int(H), int(W)), int(H), int(W))
        assert tile in (8, 16) and win_w > 0 and win_h > 0
    for name in ("a", "odd", "id"):
        f = image_case(name)
        _, _, H, W = f["img"].shape
        assert A.plan(_coef(f["G"], H, W), H, W)[0] in (8, 16), name


def test_planner_sends_the_zoom_out_to_the_unfused_route():
    f = image_case("zoom")
    _, _, H, W = f["img"].shape
    assert A.plan(_coef(f["G"], H, W), H, W)[0] == 0


def test_planner_tile_is_non_increasing_in_scale():
    H = W = 256
    tiles = []
    for s in (0.5, 1.0, 1.26, 1.6, 2.0, 2.5, 3.0, 4.0, 5.0, 6.0, 8.0):
        c, r = math.cos(0.3), math.sin(0.3)
        G = torch.tensor([[[s * c, -s * r, 0.0], [s * r, s * c, 0.0], [0, 0, 1]]], dtype=torch.float32)
        tiles.append(A.plan(_coef(G, H, W), H, W)[0])
    assert tiles[0] == 16 and tiles[-1] == 0 and 8 in tiles
    assert all(a >= b for a, b in zip(tiles, tiles[1:])), tiles


def test_planner_rejects_non_finite_and_far_coordinates():
    coef = torch.tensor([[0.0, 1.0, 0.0, 0.0, 0.0, 1.0]], dtype=torch.float64)
    assert A.plan(coef, 64, 64)[0] == 16
    for bad in (float("nan"), float("inf"), 1e9):
        c = coef.clone()
        c[0, 0] = bad
        assert A.plan(c, 64, 64)[0] == 0
    lib = _lib.load()
    assert lib.vt_augment_affine_plan(None, 1, 64, 64, None) == -1 and b"bad arguments" in lib.vt_last_error()


def test_argument_errors():
    x = torch.zeros(1, 3, 8, 8)
    with pytest.raises(_lib.VtError, match="CUDA"):
        A.random_apply_affine(x, 0.2)
    with pytest.raises(_lib.VtError, match="CUDA"):
        A.random_apply_affine(x.double(), 0.2)
    with torch.enable_grad(), pytest.raises(NotImplementedError, match="img requires grad"):
        A.random_apply_affine(x.clone().requires_grad_(), 0.2)
    with pytest.raises(NotImplementedError, match="12 taps"):
        A.random_apply_affine(x, 0.2, None, A.SYM6[:8])
    with pytest.raises(ValueError):
        A.random_apply_affine(torch.zeros(3, 8, 8), 0.2)
