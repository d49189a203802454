"""Float64 oracle of the G step's gradients: ``oracle.vt_oracle.vtoonify_forward`` (model/vtoonify.py:210-286) differentiated with torch
autograd into ``x`` and every ``encoder.*``, ``fusion_out.*`` and ``fusion_skip.*`` tensor of a state_dict.  Pinned against the
unmodified reference by tests/test_oracle_gstep.py (fixtures tests/golden/gstep_*.npz from tests/golden/make_golden_gstep.py).  Also
holds the case table, the seeded inputs and targets, the loss, float64 restatements of the mask-head backward that the GPU kernel
tests compare against, and :func:`restated_forward`, the reference module's own statements parametrised by their StyleGAN ops (the
level (b) arm of tools/gstep_bench.py)."""
import math

import torch
import torch.nn.functional as F

from oracle import vt_oracle as O
from tests.oracle_vtoonify_feat import case_inputs

# case -> (backbone, d_s)
CASES = {"d05": ("dualstylegan", 0.5), "d0": ("dualstylegan", 0.0), "t": ("toonify", 0.5)}
GEOMS = {"sq": (2, 32, 32), "ns": (1, 48, 40)}       # (B, H, W) of x
MASK_W = (0.3, 0.55, 0.8, 1.05)                       # distinct weights of mean(m_E) per fusion level
WSTEP = 997


def trained(key):
    return key.startswith(("encoder.", "fusion_out.", "fusion_skip."))


def inputs(geom, seed=0):
    B, H, W = GEOMS[geom]
    return case_inputs(B, H, W, seed=seed)


def image_target(shape, seed=0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(2468 + seed))


def loss_of(img, masks, target):
    """mse to a seeded target plus a distinct weight on every mean(m_E), so every output carries gradient."""
    loss = F.mse_loss(img, target.to(img.device, img.dtype))
    for w, m in zip(MASK_W, masks):
        loss = loss + w * m.mean()
    return loss


def loss_and_grads(sd, x, style, d_s, backbone, dtype=torch.float64, x_grad=True, target=None):
    """-> dict(loss, img, masks, x_grad, grads={trained key: gradient}), all in ``dtype``."""
    sd = {k: v.detach().to(dtype).requires_grad_(trained(k)) for k, v in sd.items()}
    x = x.detach().to(dtype).requires_grad_(x_grad)
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)          # the restatement builds Fusion's d_s label with torch.zeros, as the reference does
    try:
        with torch.enable_grad():
            r = O.vtoonify_forward(sd, x, style.to(x.device, dtype), d_s, backbone, return_mask=True)
    finally:
        torch.set_default_dtype(old)
    with torch.enable_grad():
        img, masks = r if backbone == "dualstylegan" else (r, [])
        if target is None:
            target = image_target(img.shape)
        loss = loss_of(img, masks, target)
        loss.backward()
    return {"loss": loss.detach(), "img": img.detach(), "masks": [m.detach() for m in masks],
            "x_grad": x.grad if x_grad else None, "grads": {k: v.grad for k, v in sd.items() if trained(k)}}


# ---- the mask head's backward, restated in float64 (the formulas of ops.fusion_mask_grad / fusion_adain_grad_stats /
# fusion_input_grad), with ``u`` = conv2's input gradient materialised
def mask_head_backward(g_p, f_g, f_e, m, g_m, w2, stats, gb):
    """NCHW float64 tensors; ``w2`` conv2's weight [1, 2C, 3, 3]; ``stats`` [B, 2C, 2]; ``gb`` [B, 4C] ->
    (g_z, db2, sums [B, 2C, 2], g_fg (without the conv's direct term), g_fe (with the g_p * m term))."""
    C = f_g.shape[1]
    s = (g_p * f_e).sum(1, keepdim=True) + (0 if g_m is None else g_m)
    g_z = s * (1 - m * m) * (m > 0)
    u = F.conv_transpose2d(g_z, w2, padding=1)                       # [B, 2C, H, W]
    a = torch.cat([f_g, (f_g - f_e).abs()], 1)
    mean, rstd = stats[..., 0, None, None], stats[..., 1, None, None]
    ahat = (a - mean) * rstd
    sums = torch.stack([u.sum((2, 3)), (u * ahat).sum((2, 3))], -1)
    hw = a.shape[2] * a.shape[3]
    gamma = gb[:, :2 * C, None, None]
    t = gamma * rstd * ((u - sums[..., 0, None, None] / hw) - ahat * sums[..., 1, None, None] / hw)
    sg = torch.sign(f_g - f_e)
    return g_z, g_z.sum().reshape(1), sums, t[:, :C] + sg * t[:, C:], g_p * m - sg * t[:, C:]


# ---- the reference module's statements (model/vtoonify.py:210-286, model/stylegan/model.py:93-392, model/dualstylegan.py:6-45) with
# the StyleGAN ops as parameters, as tests/oracle_discriminator.py does for the discriminator: with the defaults it is a CPU/cuDNN
# restatement (checked against oracle.vt_oracle.vtoonify_forward by tests/test_oracle_gstep.py); with vtoonify_b200.op's
# conv2d_gradfix / upfirdn2d / fused_leaky_relu it is the reference module run on the library's ops ("level (b)").  nn.Conv2d,
# nn.Linear and the instance norm stay torch, as in the reference.
def _torch_ops():
    return {"conv2d": F.conv2d, "conv_transpose2d": F.conv_transpose2d, "upfirdn2d": O.upfirdn2d, "flrelu": O.fused_leaky_relu}


def library_ops():
    from vtoonify_b200.op import conv2d_gradfix, fused_leaky_relu, upfirdn2d
    return {"conv2d": conv2d_gradfix.conv2d, "conv_transpose2d": conv2d_gradfix.conv_transpose2d, "upfirdn2d": upfirdn2d,
            "flrelu": fused_leaky_relu}


def _equal_linear(op, x, sd, p, lr_mul=1.0, act=False):
    w = sd[p + "weight"]
    scale = (1 / math.sqrt(w.shape[1])) * lr_mul
    if act:
        return op["flrelu"](F.linear(x, w * scale), sd[p + "bias"] * lr_mul)
    return F.linear(x, w * scale, bias=sd[p + "bias"] * lr_mul)


def _modconv(op, x, style, sd, p, demodulate=True, upsample=False):
    """ModulatedConv2d.forward, fused form (model/stylegan/model.py:259-306): one grouped convolution per call."""
    B, Cin, H, W = x.shape
    w0 = sd[p + "weight"]
    _, Cout, _, k, _ = w0.shape
    s = _equal_linear(op, style, sd, p + "modulation.").view(B, 1, Cin, 1, 1)
    w = (1 / math.sqrt(Cin * k * k)) * w0 * s
    if demodulate:
        w = w * torch.rsqrt(w.pow(2).sum([2, 3, 4]) + 1e-8).view(B, Cout, 1, 1, 1)
    xg = x.reshape(1, B * Cin, H, W)
    if upsample:
        wt = w.transpose(1, 2).reshape(B * Cin, Cout, k, k)
        out = op["conv_transpose2d"](xg, wt, padding=0, stride=2, groups=B)
        out = out.reshape(B, Cout, out.shape[2], out.shape[3])
        kern = sd[p + "blur.kernel"]
        q = (kern.shape[0] - 2) - (k - 1)
        return op["upfirdn2d"](out, kern, pad=((q + 1) // 2 + 1, q // 2 + 1))
    out = op["conv2d"](xg, w.reshape(B * Cout, Cin, k, k), padding=k // 2, groups=B)
    return out.reshape(B, Cout, H, W)


def restated_forward(sd, x, style, d_s, backbone="dualstylegan", in_size=256, ops=None):
    """-> (image, [m_E]) of the reference VToonify.forward(x, style, d_s, return_mask=True) (masks [] on toonify), noise all zero."""
    op = ops or _torch_ops()
    D = backbone == "dualstylegan"
    gp = "generator.generator." if D else "generator."
    if style.ndim < 3:
        style = style.unsqueeze(1).repeat(1, 18, 1)
    nB, nL, nD = style.shape
    adastyles = style
    if D:
        t = O.pixel_norm(style.reshape(nB * nL, nD))
        for i in (1, 2):
            t = _equal_linear(op, t, sd, f"generator.style.{i}.", 0.01, True)
        resstyles = t.reshape(nB, nL, nD)
        adastyles = adastyles.clone()
        for i in range(7, 18):
            adastyles[:, i] = _equal_linear(op, adastyles[:, i], sd, f"generator.res.{i}.")

    def conv(t, key, stride=1, padding=1):                 # nn.Conv2d
        return F.conv2d(t, sd[key + ".weight"], sd[key + ".bias"], stride=stride, padding=padding)

    def adain(t, s, p):
        gamma, beta = F.linear(s, sd[p + "style.weight"], sd[p + "style.bias"])[:, :, None, None].chunk(2, 1)
        return gamma * F.instance_norm(t, eps=1e-5) + beta

    def conv_layer(t, p, dil):                             # ConvLayer: EqualConv2d (conv2d_gradfix) + FusedLeakyReLU
        w = sd[p + "0.weight"]
        out = op["conv2d"](t, w * (1 / math.sqrt(w.shape[1] * w.shape[2] ** 2)), padding=w.shape[2] // 2 + dil - 1, dilation=dil)
        return op["flrelu"](out, sd[p + "1.bias"])

    n_blocks = int(math.log2(in_size)) - 4
    feat, feats = x, []
    for bi in range(n_blocks):
        feat = F.leaky_relu(conv(feat, f"encoder.{bi}.0", stride=1 if bi == 0 else 2), 0.2)
        feat = F.leaky_relu(conv(feat, f"encoder.{bi}.2"), 0.2)
        feats.append(feat)
    feats = feats[::-1]
    dil = {1: 4, 2: 4, 3: 2, 4: 2, 5: 1, 6: 1}
    for ii in range(6):
        p = f"encoder.{n_blocks}.{ii}."
        out = F.leaky_relu(conv(F.leaky_relu(conv(feat, p + "conv"), 0.2), p + "conv2"), 0.2)
        feat = (out + feat) / math.sqrt(2)
        if D and d_s != 0:
            r, s = f"res.{ii + 1}.", resstyles[:, ii + 1]
            h = conv_layer(adain(feat, s, r + "norm."), r + "conv.", dil[ii + 1])
            feat = conv_layer(adain(h, s, r + "norm2."), r + "conv2.", dil[ii + 1]) * d_s + feat
    out, skip = feat, conv(feat, f"encoder.{n_blocks + 1}", padding=0)
    m_Es = []
    for lv in range(5):
        idx = 2 * lv + 1
        if 2 ** (5 + lv) <= in_size:
            f_E = feats[lv]
            if D:
                fp = f"fusion_out.{lv}."
                label = torch.full((out.shape[0], 1), float(d_s), dtype=out.dtype, device=out.device)
                label = F.leaky_relu(F.linear(label, sd[fp + "linear.0.weight"], sd[fp + "linear.0.bias"]), 0.2)
                label = F.leaky_relu(F.linear(label, sd[fp + "linear.2.weight"], sd[fp + "linear.2.bias"]), 0.2)
                m_E = torch.tanh(F.relu(conv(adain(torch.cat([out, (out - f_E).abs()], 1), label, fp + "norm."), fp + "conv2")))
                out = conv(torch.cat([out, f_E * m_E], 1), fp + "conv")
                skip = conv(torch.cat([skip, f_E * m_E], 1), f"fusion_skip.{lv}")
                m_Es.append(m_E)
            else:
                out = conv(torch.cat([out, f_E], 1), f"fusion_out.{lv}")
                skip = conv(torch.cat([skip, f_E], 1), f"fusion_skip.{lv}")
        c1, c2, rgb = f"{gp}convs.{6 + 2 * lv}.", f"{gp}convs.{7 + 2 * lv}.", f"{gp}to_rgbs.{3 + lv}."
        out = op["flrelu"](_modconv(op, out, adastyles[:, idx + 6], sd, c1 + "conv.", upsample=True), sd[c1 + "activate.bias"])
        out = op["flrelu"](_modconv(op, out, adastyles[:, idx + 7], sd, c2 + "conv."), sd[c2 + "activate.bias"])
        img = _modconv(op, out, adastyles[:, idx + 8], sd, rgb + "conv.", demodulate=False) + sd[rgb + "bias"]
        skip = img + op["upfirdn2d"](skip, sd[rgb + "upsample.kernel"], up=2, pad=(2, 1))
    return skip, m_Es
