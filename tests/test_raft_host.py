"""RAFT drop-in: state_dict layout, loading, argument errors and the host-side weight algebra (CPU, float64 against torch)."""
import argparse
import json
import os

import pytest
import torch
import torch.nn.functional as F

from tests.conftest import GOLDEN
from tests.golden.make_golden_raft import raft_args
from vtoonify_b200 import raft as R
from vtoonify_b200.bisenet import S2D_TAPS, s2d_stem_weight
from vtoonify_b200.weights import det_state_dict


def _model():
    return R.RAFT(raft_args()).eval()


def test_state_dict_keys():
    with open(os.path.join(GOLDEN, "state_dict_keys_raft.json")) as f:
        ref = json.load(f)
    sd = _model().state_dict()
    assert len(ref) == 179 and list(sd.keys()) == ref


def test_dataparallel_strict_load():
    """the smoothing script's sequence: DataParallel(RAFT(args)).load_state_dict(module.-prefixed keys), then .module"""
    m = _model()
    sd = {"module." + k: v for k, v in det_state_dict(m).items()}
    dp = torch.nn.DataParallel(m)
    dp.load_state_dict(sd, strict=True)
    mod = dp.module
    # (DataParallel moves the module to cuda:0 where a GPU exists)
    assert torch.equal(mod.cnet.layer2[0].norm3.running_var.cpu(), sd["module.cnet.layer2.0.downsample.1.running_var"])
    assert mod.hidden_dim == 128 and mod.context_dim == 128


def test_constructor_args():
    a = raft_args()
    R.RAFT(a)
    assert (a.corr_levels, a.corr_radius, a.dropout, a.alternate_corr) == (4, 4, 0, False)
    for argv, flag in ((["--small"], "small"), (["--mixed_precision"], "mixed_precision"), (["--alternate_corr"], "alternate_corr")):
        with pytest.raises(NotImplementedError, match=flag):
            R.RAFT(raft_args(argv))
    a = raft_args()
    a.dropout = 0.1
    with pytest.raises(NotImplementedError, match="dropout"):
        R.RAFT(a)


def _imgs(B=1, H=128, W=128, **kw):
    return torch.rand(B, 3, H, W, **kw) * 255, torch.rand(B, 3, H, W, **kw) * 255


def test_forward_errors():
    m = _model()
    i1, i2 = _imgs()
    with torch.enable_grad():
        with pytest.raises(NotImplementedError, match="parameter"):      # grad mode with trainable parameters
            m(i1, i2)
        m.requires_grad_(False)
        with pytest.raises(NotImplementedError, match="image1"):
            m(i1.clone().requires_grad_(True), i2)
        with pytest.raises(NotImplementedError, match="image2"):
            m(i1, i2.clone().requires_grad_(True))
    with torch.no_grad():
        for H, W in ((120, 128), (128, 132), (64, 96), (128, 120)):
            with pytest.raises(ValueError, match="multiples of 8"):
                m(*_imgs(1, H, W))
        with pytest.raises(ValueError, match="flow_init"):
            m(i1, i2, flow_init=torch.zeros(1, 2, 8, 8))
        with pytest.raises(ValueError, match="image1"):
            m(i1, i2[:, :2])
        m.train()
        with pytest.raises(NotImplementedError, match="train"):
            m(i1, i2)


def test_fold_bn_with_bias():
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(8, 16, 3, padding=1).double()
    bn = torch.nn.BatchNorm2d(16).double().eval()
    bn.running_mean.normal_()
    bn.running_var.uniform_(0.5, 1.5)
    bn.weight.data.normal_()
    bn.bias.data.normal_()
    x = torch.randn(2, 8, 9, 7, dtype=torch.float64)
    w, b = R.fold_bn(conv, bn)
    with torch.no_grad():
        ref = bn(conv(x))
    assert torch.allclose(F.conv2d(x, w, b, padding=1), ref, rtol=1e-12, atol=1e-12)


def test_stem_space_to_depth():
    """the 7x7 / 2 stem with bias over 2 * (x / 255) - 1, as a 4x4 convolution over the space-to-depth tensor (S2D_TAPS)"""
    torch.manual_seed(1)
    w7, b = torch.randn(4, 3, 7, 7, dtype=torch.float64), torch.randn(4, dtype=torch.float64)
    img = torch.rand(1, 3, 16, 12, dtype=torch.float64) * 255
    x = 2 * (img / 255.0) - 1.0
    ref = F.conv2d(x, w7, b, stride=2, padding=3)
    z = x.reshape(1, 3, 8, 2, 6, 2).permute(0, 3, 5, 1, 2, 4).reshape(1, 12, 8, 6)       # (py, px, c) channel order
    w4 = s2d_stem_weight(w7)
    out = F.conv2d(F.pad(z, (2, 1, 2, 1)), w4, b)
    assert [t[2] for t in S2D_TAPS] == list(range(16))
    assert torch.allclose(out, ref, rtol=1e-12, atol=1e-10)


def test_stacked_zr_and_gates():
    torch.manual_seed(2)
    gru = R.SepConvGRU(128, 256).double()
    h, x = torch.randn(1, 128, 5, 6, dtype=torch.float64), torch.randn(1, 256, 5, 6, dtype=torch.float64)
    hx = torch.cat([h, x], 1)
    w, b = R.stacked_zr(gru.convz1, gru.convr1)
    with torch.no_grad():
        zr = F.conv2d(hx, w, b, padding=(0, 2))
        assert torch.allclose(zr[:, :128], gru.convz1(hx), rtol=0, atol=1e-12)
        assert torch.allclose(zr[:, 128:], gru.convr1(hx), rtol=0, atol=1e-12)


def test_motion_mask_and_convf1_weights():
    torch.manual_seed(3)
    m = _model().double()
    enc, mk = m.update_block.encoder, m.update_block.mask
    x = torch.randn(1, 256, 6, 5, dtype=torch.float64)
    w, b = R.motion_conv_weights(enc.conv)
    with torch.no_grad():
        out = F.relu(F.conv2d(x, w, b, padding=1))
        assert torch.allclose(out[:, :126], F.relu(enc.conv(x)), rtol=0, atol=1e-12) and not out[:, 126:].any()
        n = torch.randn(1, 256, 4, 3, dtype=torch.float64)
        w, b = R.mask_weights(mk[2])
        assert torch.equal(F.conv2d(n, w, b), 0.25 * mk[2](n))
        wf = R.convf1_weights(enc.convf1)
        assert wf.shape == (49, 2, 128)
        assert torch.equal(wf[3 * 7 + 5, 1], enc.convf1.weight[:, 1, 3, 5])
    assert R.rect_taps(1, 5) == [(0, dx, dx + 2) for dx in range(-2, 3)]
    assert R.rect_taps(5, 1) == [(dy, 0, dy + 2) for dy in range(-2, 3)]


def test_initialize_flow():
    m = _model()
    c0, c1 = m.initialize_flow(torch.zeros(2, 3, 128, 160))
    assert c0.shape == (2, 2, 16, 20) and torch.equal(c0, c1) and c0 is not c1
    assert c0[1, 0, 3, 7] == 7 and c0[1, 1, 3, 7] == 3
