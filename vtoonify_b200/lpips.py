"""The LPIPS perceptual loss of both training scripts (model/stylegan/lpips: ``PerceptualLoss(model='net-lin', net='vgg')``) on the
library's sm_90a kernels, with the reference's constructor, call, return value and ``percept.model.net`` state-dict keys.

``forward(pred, target)`` runs the VGG16 trunk once on ``cat(target, pred)`` as one NHWC batch of 2B:
  * ScalingLayer ``(x - shift) / scale`` (with ``normalize``'s ``2x - 1`` folded in) is a per-channel affine of the staged pixels, applied
    before the convolution's zero padding: conv1_1's ``src_affine`` in bf16x3, ``adain_apply`` otherwise;
  * each 3x3 convolution has bias + ReLU in its epilogue (``ACT_LRELU`` with slope 0), on whatever route the planner picks;
  * ``vt_maxpool2x2_nhwc_f32`` between the slices; the five slice outputs (relu1_2 .. relu5_3) are the taps;
  * one head launch for all taps (``vt_lpips_head_nhwc``: channel-normalise, squared difference, ``lin`` projection, spatial mean,
    summed over the taps; a fixed double reduction, so reruns are bit-identical).
In grad mode, when ``pred`` or ``target`` requires grad, an autograd ``Function`` keeps the ReLU outputs and the taps and goes back
top-down: the head's gradient per tap (``vt_lpips_head_grad_nhwc``), the max-pool adjoint with that tap gradient added
(``vt_maxpool2x2_grad_nhwc_f32``), the ReLU gate (``act_grad``) and the transposed convolution of every layer, conv1_1's carrying the
ScalingLayer's ``1 / scale``.  The trunk and ``lin`` weights are frozen: no weight gradient is computed, and a parameter that requires
grad raises.  Weights come from local files only; nothing is downloaded.
"""
import importlib.util
import os

import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ops
from ._lib import ACT_LRELU
from .encoder_grad import _input_grad
from .op.conv2d_gradfix import _pad_rows, conv_transpose_nhwc
from .stylegan import _conv_plain_nhwc
from .vtoonify import Conv2d
from .weights import det_state_dict

VGG16_CHECKPOINT = "vgg16-397923af.pth"     # the file tv.vgg16(pretrained=True) caches under <torch.hub.get_dir()>/checkpoints
# torchvision `features` index -> (slice, Cin, Cout) of the 13 convolutions (pretrained_networks.py:97-116); every other index of a
# slice is a ReLU, and indices 4, 9, 16 and 23 are the 2x2 max-pools that open slices 2 to 5
VGG_CONVS = {0: (1, 3, 64), 2: (1, 64, 64), 5: (2, 64, 128), 7: (2, 128, 128), 10: (3, 128, 256), 12: (3, 256, 256), 14: (3, 256, 256),
             17: (4, 256, 512), 19: (4, 512, 512), 21: (4, 512, 512), 24: (5, 512, 512), 26: (5, 512, 512), 28: (5, 512, 512)}
SLICE_RANGES = {1: range(0, 4), 2: range(4, 9), 3: range(9, 16), 4: range(16, 23), 5: range(23, 30)}
CHANNELS = [64, 128, 256, 512, 512]
MIN_SIZE = 16                               # four 2x2 poolings: relu5_3 needs at least one pixel


def default_vgg_path() -> str:
    return os.path.join(torch.hub.get_dir(), "checkpoints", VGG16_CHECKPOINT)


def default_model_path(net: str, version: str = "0.1") -> str:
    """``weights/v<version>/<net>.pth`` next to ``model.stylegan.lpips`` (dist_model.py:67-69), located without running its
    ``__init__`` (the parent packages' ``__init__.py`` files are empty)."""
    try:
        spec = importlib.util.find_spec("model.stylegan.lpips")
    except ModuleNotFoundError:
        spec = None
    if spec is None or not spec.submodule_search_locations:
        raise FileNotFoundError(f"lin weights: `model.stylegan.lpips` is not importable, so weights/v{version}/{net}.pth next to it "
                                "cannot be located; pass model_path")
    return os.path.join(list(spec.submodule_search_locations)[0], "weights", f"v{version}", f"{net}.pth")


def _load(path: str, what: str):
    if not os.path.isfile(path):
        raise FileNotFoundError(f"{what}: {path} does not exist (vtoonify_b200.lpips reads local files only and downloads nothing)")
    return torch.load(path, map_location="cpu", weights_only=True)


def vgg_state_dict(features_sd) -> dict:
    """torchvision ``vgg16`` state dict (``features.{i}.weight|bias``) -> the trunk's ``net.slice{k}.{i}.weight|bias`` entries."""
    out = {}
    for i, (s, _, _) in VGG_CONVS.items():
        for p in ("weight", "bias"):
            key = f"features.{i}.{p}"
            if key not in features_sd:
                raise KeyError(f"VGG16 checkpoint has no `{key}`")
            out[f"net.slice{s}.{i}.{p}"] = features_sd[key]
    return out


class ScalingLayer(nn.Module):
    """networks_basic.py:94-101 (buffers ``shift``, ``scale``; applied inside conv1_1's staging on the fast path)."""

    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.Tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer("scale", torch.Tensor([.458, .448, .450])[None, :, None, None])


class VGG16(nn.Module):
    """pretrained_networks.py:97-135: ``slice1..5`` hold torchvision's ``features`` modules at their original indices."""

    def __init__(self):
        super().__init__()
        for s, idx in SLICE_RANGES.items():
            seq = nn.Sequential()
            for i in idx:
                if i in VGG_CONVS:
                    m = Conv2d(VGG_CONVS[i][1], VGG_CONVS[i][2], 3, padding=1)
                elif i in (4, 9, 16, 23):
                    m = nn.MaxPool2d(2, 2)
                else:
                    m = nn.ReLU(inplace=True)
                seq.add_module(str(i), m)
            setattr(self, f"slice{s}", seq)

    def convs(self):
        return [getattr(getattr(self, f"slice{s}"), str(i)) for i, (s, _, _) in VGG_CONVS.items()]


class NetLinLayer(nn.Module):
    """networks_basic.py:104-111 with dropout: ``model.1`` is the 1x1 projection (the module is always in eval mode)."""

    def __init__(self, chn_in, chn_out=1):
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(), nn.Conv2d(chn_in, chn_out, 1, stride=1, padding=0, bias=False))


class PNetLin(nn.Module):
    """networks_basic.py:27-92 for ``pnet_type='vgg'``, version 0.1, ``lpips=True``, ``spatial=False``: 33 state-dict keys.
    ``pnet_rand=True``: deterministic synthetic trunk weights (``weights.det_state_dict``) instead of ``vgg_path``'s."""

    def __init__(self, pnet_rand=False, vgg_path=None):
        super().__init__()
        self.scaling_layer = ScalingLayer()
        self.chns = CHANNELS
        self.L = len(CHANNELS)
        self.net = VGG16()
        for k, c in enumerate(CHANNELS):
            setattr(self, f"lin{k}", NetLinLayer(c))
        self.lins = [getattr(self, f"lin{k}") for k in range(self.L)]
        if pnet_rand:
            trunk = {k: v for k, v in det_state_dict(self).items() if k.startswith("net.")}
        else:
            trunk = vgg_state_dict(_load(default_vgg_path() if vgg_path is None else vgg_path, "VGG16 weights"))
        self.load_state_dict(trunk, strict=False)
        for p in self.net.parameters():         # pnet_tune=False (networks_basic.py:50, pretrained_networks.py:117-119)
            p.requires_grad = False
        self.eval()

    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        """-> ``[B, 1, 1, 1]`` distances between ``in0`` and ``in1`` (``[B, 3, H, W]`` in [-1, 1], or [0, 1] with ``normalize``)."""
        if retPerLayer:
            raise NotImplementedError("vtoonify_b200 PNetLin: retPerLayer is not supported")
        if in0.dim() != 4 or in0.shape != in1.shape or in0.shape[1] != 3 or min(in0.shape[2:]) < MIN_SIZE:
            raise ValueError(f"PNetLin: in0 {tuple(in0.shape)} and in1 {tuple(in1.shape)} must both be [B, 3, H, W] with H, W >= {MIN_SIZE}")
        if torch.is_grad_enabled():
            for name, p in self.named_parameters():
                if p.requires_grad:
                    raise NotImplementedError(
                        f"vtoonify_b200 LPIPS computes no weight gradients, but `{name}` requires grad: freeze the network first "
                        f"(the training scripts call requires_grad(percept.model.net, False))")
            if in0.requires_grad or in1.requires_grad:
                return _LPIPS.apply(self, bool(normalize), in0, in1)
        with torch.no_grad():
            return _forward(self, in0, in1, bool(normalize), keep=False)[0]


# ------------------------------------------------------------------------------------------------ forward
def _input_affine(net, normalize):
    """per-channel (a, b) with ScalingLayer(x') = a x + b, x' = 2x - 1 under ``normalize``"""
    shift, scale = net.scaling_layer.shift.reshape(3), net.scaling_layer.scale.reshape(3)
    if normalize:
        return 2.0 / scale, (-1.0 - shift) / scale, (1.0 + shift) / 2.0
    return 1.0 / scale, -shift / scale, shift


def _forward(net, in0, in1, normalize, keep):
    """-> (loss [B, 1, 1, 1], ReLU outputs of the 13 convolutions, the 5 taps); the lists are empty unless ``keep``."""
    B = in0.shape[0]
    x = ops.to_nhwc(torch.cat([in0, in1]), 32)
    a, b, mean = _input_affine(net, normalize)
    convs = net.net.convs()
    c0 = convs[0]
    if ops.affine_fusable():
        table = torch.zeros((2 * B, 32, 2), device=x.device, dtype=torch.float32)
        table[:, :3, 0], table[:, :3, 1] = a, b
        h = _conv_plain_nhwc(x, c0.weight, c0._w, 1.0, c0.bias, 1, 1, 1, act=ACT_LRELU, slope=0.0, gain=1.0, src_affine=table)
    else:
        stats = torch.zeros((2 * B, 32, 2), device=x.device, dtype=torch.float32)
        stats[:, :, 1] = 1.0
        stats[:, :3, 0], stats[:, :3, 1] = mean, a
        gb = torch.cat([torch.ones((2 * B, 32), device=x.device), torch.zeros((2 * B, 32), device=x.device)], 1)
        h = c0.forward_nhwc(ops.adain_apply(x, stats, gb), act=ACT_LRELU, slope=0.0, gain=1.0)
    ys, taps = [h], []
    slices = [s for s, _, _ in VGG_CONVS.values()]
    for j in range(1, len(convs)):
        if slices[j] != slices[j - 1]:
            taps.append(h)
            h = ops.maxpool2x2(h)
        h = convs[j].forward_nhwc(h, act=ACT_LRELU, slope=0.0, gain=1.0)
        ys.append(h)
    taps.append(h)
    val = ops.lpips_head(taps, [lin.model[1].weight.detach().reshape(-1) for lin in net.lins])
    return val.reshape(B, 1, 1, 1), (ys if keep else []), (taps if keep else [])


# ------------------------------------------------------------------------------------------------ backward
def _backward(net, normalize, ys, taps, g_b, want0, want1):
    """-> (gradient of in0 or None, gradient of in1 or None); the trunk goes back on the rows of whichever inputs want one."""
    B = g_b.shape[0]
    rows = slice(0 if want0 else B, 2 * B if want1 else B)
    convs = net.net.convs()
    slices = [s for s, _, _ in VGG_CONVS.values()]
    lins = [lin.model[1].weight.detach().reshape(-1) for lin in net.lins]
    k = len(taps) - 1
    g = None
    for j in range(len(convs) - 1, -1, -1):
        y = ys[j][rows]
        if j == len(convs) - 1 or slices[j + 1] != slices[j]:     # a tap: the head's gradient joins (before the pool above it)
            gt = ops.lpips_head_grad(taps[k], lins[k], g_b, want0, want1)
            g = gt if g is None else ops.maxpool2x2_grad(g, y, add=gt)
            k -= 1
        gp = ops.act_grad(g, ref=y, slope=0.0, gain=1.0)
        _, H, W, _ = y.shape
        if j > 0:
            g = _input_grad(convs[j], 1.0, gp, H, W, 1, 1, 1)
    # conv1_1: 3 output rows padded to 32, each carrying the ScalingLayer's d(a x + b)/dx = a
    c0 = convs[0]
    a = _input_affine(net, normalize)[0]
    wt = ops.prep_weights(_pad_rows(c0.weight.detach().transpose(0, 1) * a.reshape(3, 1, 1, 1), 32), cin_pad=gp.shape[3])
    gx = ops.to_nchw(conv_transpose_nhwc(gp, wt, 3, 3, 1, (1, 1), (1, 1), H, W), 3)
    g0 = gx[:B] if want0 else None
    g1 = (gx[B:] if want0 else gx) if want1 else None
    return g0, g1


class _LPIPS(Function):
    @staticmethod
    def forward(ctx, net, normalize, in0, in1):
        val, ys, taps = _forward(net, in0, in1, normalize, keep=True)
        ctx.net, ctx.normalize, ctx.rec = net, normalize, (ys, taps)
        return val

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        ys, taps = ctx.rec
        ctx.rec = None
        want0, want1 = ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        if not (want0 or want1):
            return None, None, None, None
        g0, g1 = _backward(ctx.net, ctx.normalize, ys, taps, g.reshape(-1).contiguous(), want0, want1)
        return None, None, g0, g1


# ------------------------------------------------------------------------------------------------ public interface
class DistModel:
    """dist_model.py:24-117 for ``model='net-lin'``: holds ``net`` (a PNetLin, not wrapped in DataParallel) in eval mode."""

    def name(self):
        return self.model_name

    def initialize(self, model="net-lin", net="alex", colorspace="Lab", pnet_rand=False, model_path=None, use_gpu=True, spatial=False,
                   gpu_ids=[0], vgg_path=None):
        self.model, self.spatial, self.gpu_ids = model, spatial, gpu_ids
        self.model_name = f"{model} [{net}]"
        self.net = PNetLin(pnet_rand=pnet_rand, vgg_path=vgg_path)
        path = default_model_path(net) if model_path is None else model_path
        self.net.load_state_dict(_load(path, "LPIPS lin weights"), strict=False)
        self.parameters = list(self.net.parameters())
        if use_gpu:
            self.net.to(torch.device("cuda", gpu_ids[0]))

    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        return self.net.forward(in0, in1, retPerLayer=retPerLayer, normalize=normalize)


class PerceptualLoss(nn.Module):
    """lpips/__init__.py:14-41: ``PerceptualLoss(model='net-lin', net='vgg', use_gpu=True, gpu_ids=[rank])`` of both training scripts.
    Weights are read from ``vgg_path`` (default: torchvision's cached ``vgg16-397923af.pth``) and ``model_path`` (default: the reference
    checkout's ``weights/v0.1/<net>.pth``); a missing file raises ``FileNotFoundError``.  ``pnet_rand=True``: synthetic trunk weights."""

    def __init__(self, model="net-lin", net="alex", colorspace="rgb", spatial=False, use_gpu=True, gpu_ids=[0], *, model_path=None,
                 vgg_path=None, pnet_rand=False):
        super().__init__()
        if model != "net-lin":
            raise NotImplementedError(f"vtoonify_b200 PerceptualLoss: model={model!r} is not supported (only 'net-lin')")
        if net not in ("vgg", "vgg16"):
            raise NotImplementedError(f"vtoonify_b200 PerceptualLoss: net={net!r} is not supported (only 'vgg' / 'vgg16')")
        if spatial:
            raise NotImplementedError("vtoonify_b200 PerceptualLoss: spatial=True is not supported")
        self.use_gpu, self.spatial, self.gpu_ids = use_gpu, spatial, gpu_ids
        self.model = DistModel()
        self.model.initialize(model=model, net=net, use_gpu=use_gpu, colorspace=colorspace, spatial=spatial, gpu_ids=gpu_ids,
                              model_path=model_path, vgg_path=vgg_path, pnet_rand=pnet_rand)

    def forward(self, pred, target, normalize=False):
        """-> ``[B, 1, 1, 1]``; ``normalize=True`` maps [0, 1] inputs to [-1, 1] first."""
        return self.model.forward(target, pred, normalize=normalize)
