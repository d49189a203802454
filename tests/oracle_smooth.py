"""Plain-torch restatement of smooth_parsing_map.py's warp (lines 38-74), window fusion (155-165), ``Downsample([1, 3, 3, 1], 2)`` and
whole smoothing loop (143-167), in the dtype and on the device of its inputs; the flows come from tests/oracle_raft.py.  Pinned to the
reference's float32 fixtures on the CPU (tests/test_smooth_host.py), it is the float64 yardstick of the library.

One deliberate difference from the script's text: ``v / max(W - 1, 1)`` divides by a tensor on the inputs' device.  On CUDA, torch
turns a division by a CPU scalar into a multiplication by its reciprocal, which is not the reference's (CPU) or the library's rounding;
dividing by a device tensor is the true division everywhere."""
import torch
import torch.nn.functional as F


def sample_grid(flo):
    """the normalised grid_sample grid [B, H, W, 2] of the script's warp for flow [B, 2, H, W]"""
    B, _, H, W = flo.shape
    xx = torch.arange(W, device=flo.device, dtype=flo.dtype).view(1, 1, 1, W).expand(B, 1, H, W)
    yy = torch.arange(H, device=flo.device, dtype=flo.dtype).view(1, 1, H, 1).expand(B, 1, H, W)
    v = torch.cat((xx, yy), 1) + flo
    dx = torch.tensor(float(max(W - 1, 1)), device=flo.device, dtype=flo.dtype)
    dy = torch.tensor(float(max(H - 1, 1)), device=flo.device, dtype=flo.dtype)
    gx = 2.0 * v[:, 0] / dx - 1.0
    gy = 2.0 * v[:, 1] / dy - 1.0
    return torch.stack((gx, gy), -1)


def warp(x, flo):
    """(grid_sample(x) * mask, mask), mask = the thresholded grid_sample of ones, [B, C, H, W]"""
    g = sample_grid(flo)
    out = F.grid_sample(x, g, align_corners=True)
    mask = F.grid_sample(torch.ones_like(x), g, align_corners=True)
    mask = torch.where(mask < 0.9999, torch.zeros_like(mask), mask)
    mask = torch.where(mask > 0, torch.ones_like(mask), mask)
    return out * mask, mask


def temporal_weights(window, dtype=torch.float32, device="cpu"):
    return torch.exp(-(torch.arange(2 * window + 1).float() - window) ** 2 / (2 * ((window + 0.5) ** 2))).to(device, dtype)


def fuse(imgs, pars, flows, wt):
    """imgs [S, 3, H, W], pars [S, C, H, W], flows [S, 2, H, W] (slot S // 2's is not used), wt [S] -> fused [C, H, W]"""
    window = imgs.shape[0] // 2
    out, mask = warp(torch.cat((imgs, pars), 1), flows)
    a_i, a_p = out[:, :3], out[:, 3:].clone()
    ws = torch.exp(-((a_i - imgs[window:window + 1]) ** 2).mean(dim=1, keepdim=True) / (2 * (0.2 ** 2))) * mask[:, 0:1]
    a_p[window] = pars[window]
    ws[window] = 1.0
    weights = ws * wt.view(-1, 1, 1, 1).to(ws)
    weights = weights / weights.sum(dim=0, keepdim=True)
    return (a_p * weights).sum(dim=0)


def down(x):
    """Downsample([1, 3, 3, 1], 2) = upfirdn2d(x, k, down=2, pad=(1, 1)) on [N, C, H, W]"""
    f = torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=x.dtype, device=x.device)
    k = (f[None, :] * f[:, None]) / 64.0
    C = x.shape[1]
    return F.conv2d(F.pad(x, (1, 1, 1, 1)), k.flip(0, 1).expand(C, 1, 4, 4), stride=2, groups=C)


def smooth(sd, Is, Ps, window=5, iters=20):
    """the script's loop on Is [N, 3, H, W] (in [-1, 1]) and Ps [N, C, H, W] -> parse [N, C, H/2, W/2]; RAFT runs on the 2 * window
    non-centre pairs (the centre pair's results are overwritten by the script)"""
    from tests import oracle_raft as R
    N = Is.shape[0]
    w = window
    Is_ = torch.cat((Is[0:w], Is, Is[-w:]), 0)
    Ps_ = torch.cat((Ps[0:w], Ps, Ps[-w:]), 0)
    wt = temporal_weights(w, Is.dtype, Is.device)
    out = []
    for ii in range(N):
        i = ii + w
        image2 = Is_[i - w:i + w + 1]
        flows = torch.zeros((2 * w + 1, 2) + tuple(Is.shape[2:]), dtype=Is.dtype, device=Is.device)
        if w:
            nb = torch.cat((image2[:w], image2[w + 1:]), 0)
            image1 = Is_[i].repeat(2 * w, 1, 1, 1)
            _, up = R.raft_forward(sd, (image1 + 1) * 255.0 / 2, (nb + 1) * 255.0 / 2, iters, None, True, every_mask=False)
            flows[:w], flows[w + 1:] = up[:w], up[w:]
        out.append(down(fuse(image2, Ps_[i - w:i + w + 1], flows, wt)[None]))
    return torch.cat(out, 0)
