"""GPU: vtoonify_b200.align.align_faces byte for byte against the reference's align_face (tests/golden/align_*.npz), and each stage
kernel bit for bit against its NumPy oracle stage (tests/oracle_align.py)."""
import json
from argparse import Namespace

import numpy as np
import pytest
import torch

from tests import oracle_align as O
from vtoonify_b200 import align as A

pytestmark = pytest.mark.gpu

CASES = ("frame", "border", "shrink", "outside", "small")
DEV = torch.device("cuda", 0)


def _case(golden, name):
    g = golden(f"align_{name}")
    return g, O.synth_image(int(g["image_seed"]), *g["image_hw"])


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("name", CASES)
def test_fixture(golden, name):
    g, img = _case(golden, name)
    out = A.align_faces([img], g["landmarks"][None])
    assert out.is_cuda and out.dtype == torch.uint8 and tuple(out.shape) == (1, 256, 256, 3)
    got = out[0].cpu().numpy()
    assert np.array_equal(got, g["out"]), f"{int((got != g['out']).any(-1).sum())} pixels differ"


# ---- stage kernels against the oracle stages -------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw,size", [((856, 1280), (640, 428)), ((375, 500), (167, 125)), ((101, 77), (33, 25)),
                                     ((64, 64), (21, 64)), ((40, 3), (1, 2))])
def test_lanczos(hw, size):
    img = O.synth_image(hw[0] * 7 + hw[1], *hw)
    got = A.lanczos(_dev(img), size).cpu().numpy()
    assert np.array_equal(got, O.lanczos_resize(img, size))


@pytest.mark.parametrize("hw,pad,sigma,window", [((60, 50), (20, 21, 22, 23), 3.7, None), ((20, 17), (30, 31, 29, 40), 4.8, None),
                                                 ((7, 5), (1, 1, 1, 1), 0.3, None), ((90, 70), (40, 33, 35, 38), 10.48, (5, 9, 61, 50))])
def test_blur_axes(hw, pad, sigma, window):
    img = O.synth_image(sum(hw), *hw)
    src = _dev(img)
    if window is not None:                 # a crop window: pointer offset and the full image's row pitch
        x0, y0, x1, y1 = window
        view, win, kw = src[y0:y1, x0:x1], img[y0:y1, x0:x1], dict(hw=(y1 - y0, x1 - x0), pitch=hw[1] * 3)
    else:
        view, win, kw = src, img, {}
    rows = A.blur_rows(view, pad, sigma, **kw)
    want_rows = O.gaussian_axis(O.reflect_pad(win, pad), sigma, 0)
    assert np.array_equal(rows.cpu().numpy(), want_rows)
    cols = A.blur_cols(rows, sigma)
    want_cols = O.gaussian_axis(want_rows, sigma, 1)
    assert np.array_equal(cols.cpu().numpy(), want_cols)
    # the column pass with the first blend
    x = O.reflect_pad(win, pad)
    mask = O.pad_mask(x.shape[0], x.shape[1], pad)
    want = O.blend(x, want_cols, np.clip(mask * 3.0 + 1.0, 0.0, 1.0))
    assert np.array_equal(A.blur_cols(rows, sigma, view, pad, **kw).cpu().numpy(), want)


def _median_cases():
    rng = np.random.default_rng(3)
    yield "odd", rng.uniform(0, 255, (101, 3)).astype(np.float32)
    yield "even", rng.uniform(0, 255, (1000, 3)).astype(np.float32)
    yield "one", np.array([[3.5, -2.0, 0.0]], np.float32)
    yield "two", np.array([[1.0, 2.0, 3.0], [2.0, 2.0, 1.0]], np.float32)
    ties = np.repeat(np.array([[7.25, 1.0, 0.0]], np.float32), 64, 0)
    ties[:31] = [1.0, 1.0, 0.0]
    ties[40:] = [250.0, 3.0, 0.0]
    yield "ties", ties
    # the two middle values in different digits of the key, with duplicates around them
    d = np.concatenate([np.full((50, 3), 1.0), np.full((50, 3), 1.0000001), rng.uniform(-9, 9, (200, 3))]).astype(np.float32)
    yield "duplicates_signed", rng.permutation(d)
    yield "large_even", rng.normal(100, 40, (410 * 412, 3)).astype(np.float32)
    yield "large_odd", np.round(rng.normal(100, 40, (333 * 335, 3))).astype(np.float32)


@pytest.mark.parametrize("name,x", list(_median_cases()), ids=[c[0] for c in _median_cases()])
def test_median(name, x):
    got = A.median(_dev(x)).cpu().numpy()
    want = np.median(x, axis=0)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32)), (got, want)


def test_finish_rounds_half_to_even():
    rng = np.random.default_rng(4)
    Hp, Wp, pad = 40, 36, (9, 7, 10, 8)
    x = (rng.integers(-3, 259, (Hp, Wp, 3)) + 0.5).astype(np.float32)       # interior pixels (mask <= 0) keep their .5
    x[::3] = rng.uniform(-5, 260, x[::3].shape).astype(np.float32)
    med = np.array([126.5, 3.5, 0.5], np.float32)
    mask = O.pad_mask(Hp, Wp, pad)
    want = O.quantize(O.blend(x, med, np.clip(mask, 0.0, 1.0)))
    got = A.finish(_dev(x), _dev(med), pad).cpu().numpy()
    assert np.array_equal(got, want)
    assert (x[mask[..., 0] <= 0] % 1 == 0.5).any()


@pytest.mark.parametrize("hw,corners", [
    ((90, 110), [-20.0, 10.0, 5.0, 110.0, 120.0, 95.0, 90.0, -15.0]),      # zero fill on every side
    ((41, 37), [0.0, 0.0, 0.0, 41.0, 37.0, 41.0, 37.0, 0.0]),              # the image exactly: last row and column edges
    ((41, 37), [0.5, 0.5, 0.5, 40.999, 36.999, 40.999, 36.999, 0.5]),
    ((300, 200), [20.3, 280.7, 19.8, 40.1, 180.2, 39.6, 181.1, 279.9]),    # a flipped, rotated quad
    ((5, 6), [-1.0, -1.0, -1.0, 6.0, 7.0, 6.0, 7.0, -1.0]),
])
def test_warp(hw, corners):
    img = O.synth_image(hw[0] + 3 * hw[1], *hw)
    got = A.warp(_dev(img), np.array(corners)).cpu().numpy()
    want = O.quad_warp(img, np.array(corners))
    assert np.array_equal(got, want)
    if corners[0] < 0:
        assert (want == 0).all(-1).any()


# ---- the public call ------------------------------------------------------------------------------------------------------------
def test_mixed_batch_equals_single_calls(golden):
    imgs, lms = [], []
    for n in CASES:
        g, img = _case(golden, n)
        imgs.append(img)
        lms.append(g["landmarks"])
    batch = A.align_faces(imgs, np.stack(lms))
    for i, (img, lm) in enumerate(zip(imgs, lms)):
        assert torch.equal(batch[i], A.align_faces([img], lm[None])[0])
    assert torch.equal(A.align_faces(imgs, np.stack(lms)), batch)


def test_inputs_and_sync_free(golden):
    """NumPy, host-tensor and CUDA-tensor images give the same bytes; with CUDA images the call never synchronises"""
    imgs, lms, want = [], [], []
    for n in ("frame", "border", "shrink"):
        g, img = _case(golden, n)
        imgs.append(img)
        lms.append(g["landmarks"])
        want.append(torch.from_numpy(g["out"]))
    lms = np.stack(lms)
    dev_imgs = [_dev(i) for i in imgs]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = A.align_faces(dev_imgs, lms)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(out.cpu(), torch.stack(want))
    assert torch.equal(A.align_faces([torch.from_numpy(i) for i in imgs], torch.from_numpy(lms)).cpu(), torch.stack(want))
    same = np.stack([imgs[0], imgs[0]])
    assert torch.equal(A.align_faces(torch.from_numpy(same).to(DEV), lms[[0, 0]]).cpu(), torch.stack([want[0], want[0]]))


def test_rejects_mixed_devices_and_dtypes(golden):
    from vtoonify_b200._lib import VtError
    g, img = _case(golden, "frame")
    with pytest.raises(VtError, match="uint8"):
        A.align_faces([_dev(img).float()], g["landmarks"][None])
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="several devices"):
            A.align_faces([_dev(img), _dev(img).to("cuda:1")], np.stack([g["landmarks"]] * 2))


def test_psp_on_aligned_frame(golden):
    """style_transfer.py:141-144 on the device: pSp on the aligned frame equals pSp on the reference's aligned image"""
    from vtoonify_b200 import ops
    from vtoonify_b200.psp import GradualStyleEncoder
    from vtoonify_b200.weights import det_state_dict
    g, img = _case(golden, "frame")
    m = GradualStyleEncoder(50, "ir_se", Namespace(input_nc=3, n_styles=18)).eval()
    keys = json.load(open("tests/golden/state_dict_keys_psp.json"))
    assert list(m.state_dict().keys()) == list(keys.keys())
    m.load_state_dict(det_state_dict(m, seed=11), strict=True)
    m.cuda()
    with torch.no_grad():
        y = m(ops.frames_u8_to_f32(A.align_faces([_dev(img)], g["landmarks"][None])))
        ref = m(ops.frames_u8_to_f32(torch.from_numpy(g["out"][None]).to(DEV)))
    assert tuple(y.shape) == (1, 18, 512) and torch.isfinite(y).all()
    assert torch.equal(y, ref)
