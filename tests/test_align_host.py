"""CPU: the face alignment's host geometry (vtoonify_b200.align.align_params) and its NumPy oracle (tests/oracle_align.py) against the
fixtures of tests/golden/make_golden_align.py, each oracle stage against the library it restates, and the argument checks."""
import numpy as np
import pytest

from tests import oracle_align as O
from vtoonify_b200 import align as A

CASES = ("frame", "border", "shrink", "outside", "small")


def _case(golden, name):
    g = golden(f"align_{name}")
    return g, O.synth_image(int(g["image_seed"]), *g["image_hw"])


@pytest.mark.parametrize("name", CASES)
def test_params_equal_the_reference_geometry(golden, name):
    g, _ = _case(golden, name)
    p = A.align_params(g["landmarks"], tuple(g["image_hw"]))
    for key, got in (("rsize", p.rsize), ("crop", p.crop), ("pad", p.pad)):
        if key in g:
            assert got is not None and list(got) == g[key].tolist(), key
        else:
            assert got is None, key
    assert (p.blur is None) == ("blur" not in g)
    if p.blur is not None:
        assert p.blur == float(g["blur"])
    assert p.shrink > 1 if "rsize" in g else p.shrink <= 1
    assert p.corners.dtype == np.float64 and np.array_equal(p.corners, g["corners"])


def test_cases_cover_their_stages(golden):
    """each fixture exercises the branch it is named for"""
    ps = {n: A.align_params(golden(f"align_{n}")["landmarks"], tuple(golden(f"align_{n}")["image_hw"])) for n in CASES}
    assert ps["frame"].crop is not None and ps["frame"].pad is None and ps["frame"].shrink <= 1
    assert ps["border"].pad is not None and ps["border"].crop is not None
    assert ps["shrink"].shrink == 2 and ps["shrink"].pad is not None
    assert ps["outside"].pad is None and ps["outside"].crop is not None
    # the quad reaches 4 pixels from the cropped image's right edge (ceil(max x) = W - 4): any further and padding triggers
    h, w = ps["outside"].size
    assert int(np.ceil(ps["outside"].corners[0::2].max() - 0.5)) == w - 4
    s = ps["small"]
    hw = golden("align_small")["image_hw"]
    assert s.crop is None and min(s.pad[0], s.pad[2]) > hw[1] and min(s.pad[1], s.pad[3]) > hw[0]
    assert (s.size[0] * s.size[1]) % 2 == 0 and (s.size[0] % 2 == 1 or s.size[1] % 2 == 1)


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_fixture(golden, name):
    g, img = _case(golden, name)
    out = O.align(img, A.align_params(g["landmarks"], tuple(g["image_hw"])))
    assert out.dtype == np.uint8 and out.shape == (256, 256, 3)
    assert np.array_equal(out, g["out"])


def test_host_tables_equal_the_oracle():
    for n_in, n_out in ((1280, 640), (856, 428), (500, 167), (97, 31), (90, 89)):
        tab, ksize = A.lanczos_table(n_in, n_out)
        xmin, taps, kk = O.lanczos_coeffs(n_in, n_out)
        assert np.array_equal(tab[:n_out], xmin) and np.array_equal(tab[n_out:2 * n_out], taps)
        assert np.array_equal(tab[2 * n_out:].reshape(n_out, ksize), kk)
    for s in (0.3, 2.0, 4.48, 10.48, 20.47):
        w = A.gaussian_taps(s)
        assert np.array_equal(w, O.gaussian_weights(s))
    corners = np.array([3.5, 2.25, 1.0, 70.5, 80.75, 81.0, 90.0, -4.5])
    assert np.array_equal(A.quad_coeffs(corners), O.quad_coeffs(corners))


def test_reflect_pad_repeats_for_wide_pads():
    img = O.synth_image(7, 5, 4)
    for pad in ((1, 2, 3, 4), (9, 11, 13, 17), (4, 3, 4, 3)):
        want = np.pad(np.float32(img), ((pad[1], pad[3]), (pad[0], pad[2]), (0, 0)), "reflect")
        assert np.array_equal(O.reflect_pad(img, pad), want)


# ---- each oracle stage against the library it restates ----------------------------------------------------------------------
def _libraries(golden):
    PIL = pytest.importorskip("PIL")
    pytest.importorskip("PIL.Image")
    scipy = pytest.importorskip("scipy")
    pytest.importorskip("scipy.ndimage")
    have = [np.__version__, scipy.__version__, PIL.__version__]
    pinned = golden("align_frame")["versions"].tolist()
    if have != pinned:
        pytest.skip(f"NumPy / SciPy / Pillow {have} differ from the fixtures' {pinned}")


@pytest.mark.parametrize("hw,size", [((853, 1280), (640, 427)), ((375, 500), (167, 125)), ((333, 500), (167, 111)),
                                     ((101, 77), (33, 25)), ((64, 64), (21, 64))])
def test_lanczos_equals_pillow(golden, hw, size):
    _libraries(golden)
    from PIL import Image
    img = O.synth_image(hw[0] + hw[1], *hw)
    want = np.asarray(Image.fromarray(img).resize(size, Image.LANCZOS))
    assert np.array_equal(O.lanczos_resize(img, size), want)


@pytest.mark.parametrize("hw,pad,sigma", [((60, 50), (20, 21, 22, 23), 3.7), ((31, 45), (9, 9, 9, 9), 0.9),
                                          ((20, 17), (30, 31, 29, 40), 4.8)])
def test_blur_blends_median_equal_scipy_numpy(golden, hw, pad, sigma):
    _libraries(golden)
    import scipy.ndimage
    img = O.synth_image(sum(hw), *hw)
    x = O.reflect_pad(img, pad)
    g = O.gaussian_axis(O.gaussian_axis(x, sigma, 0), sigma, 1)
    want = scipy.ndimage.gaussian_filter(x, [sigma, sigma, 0])
    assert g.dtype == np.float32 and np.array_equal(g, want)
    # the reference's statements on the same padded image
    h, w, _ = x.shape
    ref = x.copy()
    mask = O.pad_mask(h, w, pad)
    ref += (want - ref) * np.clip(mask * 3.0 + 1.0, 0.0, 1.0)
    ref += (np.median(ref, axis=(0, 1)) - ref) * np.clip(mask, 0.0, 1.0)
    ref = np.uint8(np.clip(np.rint(ref), 0, 255))
    assert np.array_equal(O.padded_blur(img, pad, sigma), ref)


@pytest.mark.parametrize("hw,seed", [((90, 110), 0), ((41, 37), 1), ((300, 200), 2)])
def test_quad_warp_equals_pillow(golden, hw, seed):
    _libraries(golden)
    from PIL import Image
    img = O.synth_image(seed, *hw)
    rng = np.random.default_rng(seed)
    h, w = hw
    # corners inside, across and beyond the image
    corners = np.array([-0.2 * w, 0.1 * h, 0.05 * w, 1.2 * h, 1.1 * w, 0.9 * h, 0.8 * w, -0.15 * h]) + rng.uniform(-3, 3, 8)
    want = np.asarray(Image.fromarray(img).transform((256, 256), Image.QUAD, tuple(corners.tolist()), Image.BILINEAR))
    assert np.array_equal(O.quad_warp(img, corners), want)


# ---- argument checks -----------------------------------------------------------------------------------------------------------
def test_params_reject_bad_landmarks():
    lm = O.synth_landmarks(0, (40, 40), (80, 40), (45, 90), (75, 90))
    for bad in (lm[:67], lm.reshape(2, 68), lm[None], np.full((68, 2), np.nan), np.where(np.arange(68)[:, None] == 3, np.inf, lm)):
        with pytest.raises(ValueError, match="landmarks"):
            A.align_params(bad, (200, 200))
    A.align_params(lm.astype(np.int64), (200, 200))


def test_params_reject_a_pad_the_reference_divides_by_zero_on():
    # a face of qsize < 5/3 at the image corner: padding triggers with rint(0.3 qsize) == 0
    lm = O.synth_landmarks(1, (0.1, 0.1), (0.4, 0.1), (0.15, 0.5), (0.35, 0.5))
    with pytest.raises(ValueError, match="divides by zero"):
        A.align_params(lm, (50, 50))


def test_align_faces_rejects_bad_inputs():
    from vtoonify_b200._lib import VtError
    lm = O.synth_landmarks(0, (40, 40), (80, 40), (45, 90), (75, 90))
    img = O.synth_image(0, 120, 120)
    with pytest.raises(VtError, match="uint8"):
        A.align_faces([img.astype(np.float32)], lm[None])
    with pytest.raises(VtError, match=r"\[H, W, 3\]"):
        A.align_faces([img[..., :2]], lm[None])
    with pytest.raises(VtError, match=r"\[H, W, 3\]"):
        A.align_faces([img[..., 0]], lm[None])
    with pytest.raises(ValueError, match="images"):
        A.align_faces(img, lm[None])
    with pytest.raises(ValueError, match="2 images but 1"):
        A.align_faces([img, img], lm[None])
    with pytest.raises(ValueError, match=r"\[N, 68, 2\]"):
        A.align_faces([img], lm)
    big = np.lib.stride_tricks.as_strided(np.zeros(3, np.uint8), (40000, 20000, 3), (0, 0, 1))
    with pytest.raises(ValueError, match="int32"):
        A.align_faces([big], lm[None])
