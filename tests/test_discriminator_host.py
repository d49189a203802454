"""CPU, float64: the identities the discriminator's NHWC route rests on, its state_dict, and the deterministic weights."""
import glob
import json
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import vt_oracle as O
from tests.oracle_discriminator import mbstd

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _rand(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def test_skip_reads_the_pad2_blur_at_tap_1_1():
    """the reference skip (Blur pad (1, 1), 1x1 stride 2) is the 1x1 stride-2 conv at offset (1, 1) of the pad (2, 2) blur"""
    K = O.make_kernel([1, 3, 3, 1]).double()
    x, w = _rand((2, 5, 16, 16), 1), _rand((7, 5, 1, 1), 2)
    ref = F.conv2d(O.upfirdn2d(x, K, pad=(1, 1)), w, stride=2)
    xb = O.upfirdn2d(x, K, pad=(2, 2))
    assert xb.shape[-1] == 17
    got = F.conv2d(xb[:, :, 1:, 1:], w, stride=2)
    assert torch.equal(got, ref)


def test_blurred_path_adjoint_is_the_upconvolution_with_K():
    """adjoint of Blur(pad (2, 2)) o conv(3x3, stride 2) = upfirdn2d(conv_transpose2d(g, W, stride 2), K, pad (1, 1))"""
    K = O.make_kernel([1, 3, 3, 1]).double()
    x, w = _rand((2, 5, 16, 16), 3).requires_grad_(), _rand((7, 5, 3, 3), 4)
    with torch.enable_grad():
        y = F.conv2d(O.upfirdn2d(x, K, pad=(2, 2)), w, stride=2)
        g = _rand(y.shape, 5)
        (y * g).sum().backward()
    got = O.upfirdn2d(F.conv_transpose2d(g, w, stride=2), K, pad=(1, 1))
    assert got.shape == x.shape
    assert (got - x.grad).abs().max().item() <= 1e-12 * x.grad.abs().max().item()


def test_skip_adjoint_is_the_odd_pixel_scatter_then_the_pad1_blur():
    """the skip's input gradient: the transposed 1x1 onto the odd pixels of the (H+1)^2 grid, then upfirdn2d(K, pad (1, 1))"""
    K = O.make_kernel([1, 3, 3, 1]).double()
    x, w = _rand((2, 5, 16, 16), 6).requires_grad_(), _rand((7, 5, 1, 1), 7)
    with torch.enable_grad():
        y = F.conv2d(O.upfirdn2d(x, K, pad=(1, 1)), w, stride=2)
        g = _rand(y.shape, 8)
        (y * g).sum().backward()
    grid = torch.zeros((2, 5, 17, 17), dtype=torch.float64)
    grid[:, :, 1::2, 1::2] = F.conv_transpose2d(g, w)
    got = O.upfirdn2d(grid, K, pad=(1, 1))
    assert (got - x.grad).abs().max().item() <= 1e-12 * x.grad.abs().max().item()


@pytest.mark.parametrize("B", [1, 2, 4, 8, 12])
def test_stddev_column_mapping(B):
    """sample b is in column b % (B / group) and every sample of a column gets its statistic"""
    x = _rand((B, 6, 2, 3), 9)
    out = mbstd(x)
    group = min(B, 4)
    M = B // group
    for m in range(M):
        col = x[[g * M + m for g in range(group)]]
        s = torch.sqrt(col.var(0, unbiased=False) + 1e-8).mean()
        for g in range(group):
            assert torch.allclose(out[g * M + m, 6], s.expand(2, 3), rtol=1e-14, atol=0)


def test_stddev_rejects_uneven_batch():
    with pytest.raises(RuntimeError):
        mbstd(_rand((6, 4, 2, 2), 10))
    from vtoonify_b200.discriminator import stddev_group
    from vtoonify_b200.vtoonify import ConditionalDiscriminator
    D = ConditionalDiscriminator(32, channel_multiplier=1)
    with pytest.raises(ValueError):
        stddev_group(D, 6)
    assert stddev_group(D, 8) == 4 and stddev_group(D, 2) == 2


def test_det_state_dict_new_rules_touch_no_existing_key():
    from vtoonify_b200.weights import DISCRIMINATOR_EQUAL_WEIGHT
    files = [f for f in glob.glob(os.path.join(GOLDEN, "state_dict_keys_*.json")) if "discriminator" not in f]
    assert len(files) >= 5
    for f in files:
        with open(f) as fh:
            keys = json.load(fh)
        hits = [k for k in keys if DISCRIMINATOR_EQUAL_WEIGHT.search(k) or k.endswith(".0.kernel")]
        assert not hits, (os.path.basename(f), hits[:3])


def test_det_state_dict_keeps_the_blur_taps():
    from vtoonify_b200.vtoonify import ConditionalDiscriminator
    from vtoonify_b200.weights import det_state_dict
    D = ConditionalDiscriminator(64, channel_multiplier=1, use_condition=True, style_num=2)
    sd = det_state_dict(D, seed=0)
    K = O.make_kernel([1, 3, 3, 1])
    blur = [k for k in sd if k.endswith(".0.kernel")]
    assert len(blur) == 2 * 4
    for k in blur:
        assert torch.equal(sd[k], K), k
    # EqualConv2d / EqualLinear weights are randn (the layer scales them): O(1) entries
    assert 0.8 < sd["convs.1.conv2.1.weight"].std().item() < 1.2
    assert 0.8 < sd["final_linear.0.weight"].std().item() < 1.2


@pytest.mark.parametrize("name,kw", [("discriminator", {}), ("discriminator_cond", dict(use_condition=True, style_num=3))])
def test_state_dict_keys_and_shapes_match_the_reference(name, kw):
    from vtoonify_b200.vtoonify import ConditionalDiscriminator
    with open(os.path.join(GOLDEN, f"state_dict_keys_{name}.json")) as f:
        ref = json.load(f)
    sd = ConditionalDiscriminator(256, **kw).state_dict()
    assert {k: list(v.shape) for k, v in sd.items()} == ref
    assert list(sd) == list(ref)
