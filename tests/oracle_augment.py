"""Plain-torch restatement of ``random_apply_affine``'s image path (model/simple_augment.py:391-441) for a given G: the batch-wide
reflect pad, two upfirdn2d passes up, ``affine_grid`` + ``grid_sample``, two upfirdn2d passes down.  The pads and the float32 sampling
matrix come from ``vtoonify_b200.simple_augment`` (pinned bit for bit to the reference by tests/test_augment_host.py); everything
after them runs in the dtype of ``img``, float64 for the fixtures' restatement.

``upfirdn`` takes the reference wrapper's signature ``upfirdn2d(x, kernel, up, down, pad)``; the default is the planar torch
restatement below, and tools/augment_bench.py passes the reference's CUDA op or ``vtoonify_b200.op.upfirdn2d`` to time the statements.
"""
import torch
from torch.nn import functional as F

from vtoonify_b200.simple_augment import PAD_K, SYM6, padding, sampling_matrix


def upfirdn2d(x, kernel, up=1, down=1, pad=(0, 0)):
    """zero insertion by ``up``, zero pad (negative: crop) by ``pad`` = (x0, x1, y0, y1), true convolution with ``kernel`` [kh, kw],
    keep every ``down``-th sample"""
    up_x, up_y = (up, up) if isinstance(up, int) else up
    down_x, down_y = (down, down) if isinstance(down, int) else down
    if len(pad) == 2:
        pad = (pad[0], pad[1], pad[0], pad[1])
    B, C, H, W = x.shape
    x = x.reshape(B * C, 1, H, W)
    if up_x > 1 or up_y > 1:
        z = x.new_zeros(B * C, 1, H * up_y, W * up_x)
        z[:, :, ::up_y, ::up_x] = x
        x = z
    x = F.pad(x, [max(p, 0) for p in pad])
    x = x[:, :, max(-pad[2], 0):x.shape[2] - max(-pad[3], 0), max(-pad[0], 0):x.shape[3] - max(-pad[1], 0)]
    kh, kw = kernel.shape
    x = F.conv2d(x, torch.flip(kernel, (0, 1)).view(1, 1, kh, kw))
    x = x[:, :, ::down_y, ::down_x]
    return x.reshape(B, C, x.shape[2], x.shape[3])


def apply(img, G, kernel=SYM6, upfirdn=upfirdn2d):
    """random_apply_affine(img, p, G)[0] for a given [B, 3, 3] float32 CPU G"""
    B, C, H, W = img.shape
    pads = tuple(int(v) for v in padding(G, H, W))
    theta = sampling_matrix(G, pads, H, W).to(img.device)
    k = torch.as_tensor(kernel).to(img)
    n = k.shape[0]
    kf = torch.flip(k, (0,))
    x = F.pad(img, pads, mode="reflect")
    up0, up1 = (n + 1) // 2, (n - 2) // 2
    x = upfirdn(x, k.unsqueeze(0), up=(2, 1), pad=(up0, up1, 0, 0))
    x = upfirdn(x, k.unsqueeze(1), up=(1, 2), pad=(0, 0, up0, up1))
    grid = F.affine_grid(theta[:, :2, :].to(x), (B, C, (H + PAD_K * 2) * 2, (W + PAD_K * 2) * 2), align_corners=False)
    x = F.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
    d0, d1 = -PAD_K * 2 + (n - 1) // 2, -PAD_K * 2 + (n - 2) // 2
    x = upfirdn(x, kf.unsqueeze(0), down=(2, 1), pad=(d0, d1, 0, 0))
    return upfirdn(x, kf.unsqueeze(1), down=(1, 2), pad=(0, 0, d0, d1))
