"""Plain-torch restatement of RAFT's on-demand correlation (model/raft/core/corr.py AlternateCorrBlock with alt_cuda_corr's forward)
in the dtype and on the device of its inputs: the pooled fmap2 pyramid, then per pixel and level the dot products of fmap1 with it at
the 10 x 10 integer positions around floor(coords / 2^l) - 4, combined into the 81 bilinear taps and scaled by 1 / sqrt(C).  In exact
arithmetic this is ``oracle_raft.lookup(oracle_raft.pyramid(fmap1, fmap2), coords)`` (pooling is linear), which
tests/test_raft_ondemand_host.py checks in float64."""
import torch
import torch.nn.functional as F


def fmap_pyramid(fmap2, levels=4):
    """fmap2 [B, C, h, w] and its 2x2 mean pools (floor sizes)"""
    pyr = [fmap2]
    for _ in range(levels - 1):
        pyr.append(F.avg_pool2d(pyr[-1], 2, stride=2))
    return pyr


def window_dots(fmap1, f2, coords_l, radius=4):
    """fmap1 [B, C, h, w], one level f2 [B, C, H, W], coords_l [B, h*w, 2] (x, y) at that level -> (dots [B, h*w, 10 (y), 10 (x)] of
    fmap1 . f2 / sqrt(C) at the positions (by + i, bx + j), zeros outside the map; (bx, by) [B, h*w, 2] = floor(coords_l) - radius)"""
    B, C, h, w = fmap1.shape
    H, W = f2.shape[2:]
    S = 2 * radius + 2
    base = torch.floor(coords_l) - radius
    j = torch.arange(S, dtype=coords_l.dtype, device=coords_l.device)
    X = (base[..., 0:1] + j)[:, :, None, :].expand(B, h * w, S, S)
    Y = (base[..., 1:2] + j)[:, :, :, None].expand(B, h * w, S, S)
    ok = (X >= 0) & (X < W) & (Y >= 0) & (Y < H)
    idx = (Y.clamp(0, H - 1) * W + X.clamp(0, W - 1)).long().reshape(B, -1)
    g = torch.gather(f2.reshape(B, C, H * W), 2, idx[:, None, :].expand(B, C, idx.shape[1]))      # [B, C, hw * S * S]
    f1 = fmap1.reshape(B, C, h * w, 1).expand(B, C, h * w, S * S).reshape(B, C, -1)
    dots = (f1 * g).sum(1).reshape(B, h * w, S, S) / torch.sqrt(torch.tensor(float(C), dtype=f1.dtype))
    return torch.where(ok, dots, torch.zeros_like(dots)), base


def ondemand(fmap1, pyr, coords, radius=4):
    """fmap1 [B, C, h, w], pyr (fmap_pyramid of fmap2), coords [B, 2, h, w] -> [B, levels * 81, h, w]; channel l*81 + 9i + j is the tap
    at x-offset i - radius, y-offset j - radius (the CorrBlock order)"""
    B, C, h, w = fmap1.shape
    c = coords.permute(0, 2, 3, 1).reshape(B, h * w, 2)
    r = radius
    out = []
    for lvl, f2 in enumerate(pyr):
        cl = c / 2 ** lvl
        dots, base = window_dots(fmap1, f2, cl, r)
        flat = dots.reshape(B, h * w, -1)
        taps = []
        for i in range(2 * r + 1):
            for jj in range(2 * r + 1):
                ix, iy = cl[..., 0] + (i - r), cl[..., 1] + (jj - r)
                x0, y0 = torch.floor(ix), torch.floor(iy)
                tx, ty = ix - x0, iy - y0
                jx, jy = (x0 - base[..., 0]).long(), (y0 - base[..., 1]).long()      # i and jj here: float64 adds no rounding
                v = torch.zeros_like(tx)
                for dx, dy, wgt in ((0, 0, (1 - tx) * (1 - ty)), (1, 0, tx * (1 - ty)), (0, 1, (1 - tx) * ty), (1, 1, tx * ty)):
                    ax, ay = jx + dx, jy + dy
                    inw = (ax < 2 * r + 2) & (ay < 2 * r + 2)
                    k = (ay.clamp(max=2 * r + 1) * (2 * r + 2) + ax.clamp(max=2 * r + 1))
                    v = v + torch.where(inw, flat.gather(2, k[..., None])[..., 0] * wgt, torch.zeros_like(wgt))
                taps.append(v)
        out.append(torch.stack(taps, -1))
    return torch.cat(out, -1).reshape(B, h, w, -1).permute(0, 3, 1, 2)
