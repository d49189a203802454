"""Plain-torch restatement of RAFT's forward (model/raft/core/raft.py, extractor.py, update.py, corr.py; full model, eval) on a
state_dict, in the dtype and on the device of its inputs.  The reference itself cannot run in float64 (its CorrBlock returns
``.float()``), so the float64 yardstick of the library is this restatement, pinned to the reference's float32 fixtures on the CPU
(tests/test_oracle_raft.py)."""
import torch
import torch.nn.functional as F


def _conv(sd, k, x, stride=1, padding=0):
    return F.conv2d(x, sd[k + ".weight"].to(x), sd[k + ".bias"].to(x), stride, padding)


def _norm(sd, k, x, kind):
    if kind == "instance":
        return F.instance_norm(x, eps=1e-5)
    return F.batch_norm(x, sd[k + ".running_mean"].to(x), sd[k + ".running_var"].to(x), sd[k + ".weight"].to(x), sd[k + ".bias"].to(x),
                        False, 0.0, 1e-5)


def encoder(sd, p, x, kind):
    """BasicEncoder: 7x7/2 stem, three stages of two residual blocks (strides 1, 2, 2), 1x1 output conv."""
    x = F.relu(_norm(sd, p + ".norm1", _conv(sd, p + ".conv1", x, 2, 3), kind))
    for li, s0 in ((1, 1), (2, 2), (3, 2)):
        for bi, s in enumerate((s0, 1)):
            q = f"{p}.layer{li}.{bi}"
            y = F.relu(_norm(sd, q + ".norm1", _conv(sd, q + ".conv1", x, s, 1), kind))
            y = F.relu(_norm(sd, q + ".norm2", _conv(sd, q + ".conv2", y, 1, 1), kind))
            if s != 1:
                # norm3 is downsample.1 (one module under two names); a state_dict's downsample.1 entries load last
                x = _norm(sd, q + ".downsample.1", _conv(sd, q + ".downsample.0", x, s, 0), kind)
            x = F.relu(x + y)
    return _conv(sd, p + ".conv2", x)


def sample(img, x, y):
    """bilinear samples of img [N, H, W] at pixel coordinates x, y [N, K]; corners outside the map count as 0"""
    N, H, W = img.shape
    x0, y0 = torch.floor(x), torch.floor(y)
    tx, ty = x - x0, y - y0
    flat = img.reshape(N, H * W)
    out = torch.zeros_like(x)
    for dx, dy, wgt in ((0, 0, (1 - tx) * (1 - ty)), (1, 0, tx * (1 - ty)), (0, 1, (1 - tx) * ty), (1, 1, tx * ty)):
        xi, yi = x0 + dx, y0 + dy
        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long()
        out = out + torch.where(ok, flat.gather(1, idx) * wgt, torch.zeros_like(wgt))
    return out


def pyramid(fmap1, fmap2, levels=4):
    B, C, h, w = fmap1.shape
    corr = torch.matmul(fmap1.reshape(B, C, h * w).transpose(1, 2), fmap2.reshape(B, C, h * w)) / torch.sqrt(torch.tensor(float(C)))
    pyr = [corr.reshape(B * h * w, 1, h, w)]
    for _ in range(levels - 1):
        pyr.append(F.avg_pool2d(pyr[-1], 2, stride=2))
    return [p[:, 0] for p in pyr]


def lookup(pyr, coords, radius=4):
    """coords [B, 2, h, w] (x, y) -> [B, levels * (2r+1)^2, h, w]; channel l*81 + 9i + j samples x-offset i - r, y-offset j - r"""
    B, _, h, w = coords.shape
    c = coords.permute(0, 2, 3, 1).reshape(B * h * w, 2)
    d = torch.arange(-radius, radius + 1, dtype=coords.dtype, device=coords.device)
    di = d.view(-1, 1).expand(2 * radius + 1, 2 * radius + 1).reshape(1, -1)    # x offset (slow index)
    dj = d.view(1, -1).expand(2 * radius + 1, 2 * radius + 1).reshape(1, -1)    # y offset (fast index)
    out = [sample(lvl, c[:, :1] / 2 ** i + di, c[:, 1:] / 2 ** i + dj) for i, lvl in enumerate(pyr)]
    return torch.cat(out, 1).reshape(B, h, w, -1).permute(0, 3, 1, 2)


def update(sd, net, inp, corr, flow):
    p = "update_block."
    cor = F.relu(_conv(sd, p + "encoder.convc1", corr))
    cor = F.relu(_conv(sd, p + "encoder.convc2", cor, 1, 1))
    flo = F.relu(_conv(sd, p + "encoder.convf1", flow, 1, 3))
    flo = F.relu(_conv(sd, p + "encoder.convf2", flo, 1, 1))
    mot = torch.cat([F.relu(_conv(sd, p + "encoder.conv", torch.cat([cor, flo], 1), 1, 1)), flow], 1)
    x = torch.cat([inp, mot], 1)
    h = net
    for i, pad in ((1, (0, 2)), (2, (2, 0))):
        hx = torch.cat([h, x], 1)
        z = torch.sigmoid(_conv(sd, f"{p}gru.convz{i}", hx, 1, pad))
        r = torch.sigmoid(_conv(sd, f"{p}gru.convr{i}", hx, 1, pad))
        q = torch.tanh(_conv(sd, f"{p}gru.convq{i}", torch.cat([r * h, x], 1), 1, pad))
        h = (1 - z) * h + z * q
    delta = _conv(sd, p + "flow_head.conv2", F.relu(_conv(sd, p + "flow_head.conv1", h, 1, 1)), 1, 1)
    return h, delta


def mask(sd, net):
    p = "update_block.mask."
    return 0.25 * _conv(sd, p + "2", F.relu(_conv(sd, p + "0", net, 1, 1)))


def upsample(flow, m):
    N, _, h, w = flow.shape
    m = torch.softmax(m.view(N, 1, 9, 8, 8, h, w), dim=2)
    up = F.unfold(8 * flow, [3, 3], padding=1).view(N, 2, 9, 1, 1, h, w)
    up = torch.sum(m * up, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(N, 2, 8 * h, 8 * w)


def raft_forward(sd, image1, image2, iters=12, flow_init=None, test_mode=False, every_mask=True):
    """RAFT.forward.  ``every_mask=False`` runs the mask head only where its result is returned (test mode: the last iteration)."""
    image1 = 2 * (image1 / 255.0) - 1.0
    image2 = 2 * (image2 / 255.0) - 1.0
    B, _, H, W = image1.shape
    fmap = encoder(sd, "fnet", torch.cat([image1, image2], 0), "instance")
    pyr = pyramid(fmap[:B], fmap[B:])
    cnet = encoder(sd, "cnet", image1, "batch")
    net, inp = torch.tanh(cnet[:, :128]), torch.relu(cnet[:, 128:])
    ys, xs = torch.meshgrid(torch.arange(H // 8, device=image1.device), torch.arange(W // 8, device=image1.device), indexing="ij")
    coords0 = torch.stack([xs, ys], 0).to(image1.dtype)[None].repeat(B, 1, 1, 1)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init.to(image1)
    preds = []
    for itr in range(iters):
        corr = lookup(pyr, coords1)
        net, delta = update(sd, net, inp, corr, coords1 - coords0)
        coords1 = coords1 + delta
        if every_mask or not test_mode or itr == iters - 1:
            preds.append(upsample(coords1 - coords0, mask(sd, net)))
    if test_mode:
        return coords1 - coords0, preds[-1]
    return preds
