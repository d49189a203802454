"""Plain-torch restatement of the LPIPS VGG16 loss (model/stylegan/lpips: PerceptualLoss(model='net-lin', net='vgg'),
networks_basic.py:64-111, pretrained_networks.py:97-135, lpips/__init__.py:43-45) on a PNetLin state dict.  It runs in whatever
dtype and on whatever device its inputs have: float64 on the CPU is the oracle the tests compare against; fp32 on the device (cuDNN)
is the training-size check and tools/lpips_bench.py's baseline.  Pinned to the reference by tests/test_oracle_lpips.py."""
import torch
import torch.nn.functional as F

# (slice, torchvision `features` index) of the 13 convolutions; a 2x2 max-pool opens slices 2 to 5, and each slice's last ReLU
# output is a tap
VGG_CONVS = [(1, 0), (1, 2), (2, 5), (2, 7), (3, 10), (3, 12), (3, 14), (4, 17), (4, 19), (4, 21), (5, 24), (5, 26), (5, 28)]
CHANNELS = [64, 128, 256, 512, 512]
EPS = 1e-10


def vgg_taps(sd, x):
    """relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3 of the scaled input ``x``."""
    taps, h, cur = [], x, 1
    for s, i in VGG_CONVS:
        if s != cur:
            taps.append(h)
            h = F.max_pool2d(h, 2, 2)
            cur = s
        h = F.relu(F.conv2d(h, sd[f"net.slice{s}.{i}.weight"], sd[f"net.slice{s}.{i}.bias"], padding=1))
    taps.append(h)
    return taps


def normalize_tensor(f):
    return f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + EPS)


def pnetlin(sd, in0, in1):
    """PNetLin.forward(in0, in1) (version 0.1, spatial=False) -> [B, 1, 1, 1]; the trunk runs once on cat(in0, in1)."""
    shift, scale = sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    B = in0.shape[0]
    taps = vgg_taps(sd, (torch.cat([in0, in1]) - shift) / scale)
    val = 0
    for k, t in enumerate(taps):
        d = (normalize_tensor(t[:B]) - normalize_tensor(t[B:])) ** 2
        val = val + F.conv2d(d, sd[f"lin{k}.model.1.weight"]).mean([2, 3], keepdim=True)
    return val


def perceptual_loss(sd, pred, target, normalize=False):
    """PerceptualLoss.forward(pred, target, normalize) = DistModel.forward(target, pred)."""
    if normalize:
        pred, target = 2 * pred - 1, 2 * target - 1
    return pnetlin(sd, target, pred)


def inputs(shape, seed):
    """seeded pred and target images in [-1, 1] (float64)"""
    g = torch.Generator().manual_seed(seed)
    pred = torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1
    target = (pred + 0.5 * torch.randn(shape, generator=g, dtype=torch.float64)).clamp(-1, 1)
    return pred, target


def loss_weights(B, seed):
    """per-sample weights of the scalar that is back-propagated (so every sample's gradient is pinned, not only their sum)"""
    g = torch.Generator().manual_seed(seed + 7)
    return 0.5 + torch.rand(B, generator=g, dtype=torch.float64)


# golden cases: name -> (shape, seed, grad to pred, grad to target)
CASES = {
    "sq": ((2, 3, 64, 64), 1, True, False),
    "odd": ((1, 3, 50, 38), 2, True, False),
    "both": ((2, 3, 48, 40), 3, True, True),
}
