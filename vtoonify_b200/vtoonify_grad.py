"""Gradients of ``VToonify.forward(x, style, d_s, return_mask)``: the G step of both training scripts (train_vtoonify_d.py:299-338,
train_vtoonify_t.py:242-270), where the image and mask losses are back-propagated into the encoder and the fusion modules.

The route is an autograd ``Function`` whose inputs are ``x`` and every parameter of ``encoder``, ``fusion_out`` and ``fusion_skip``, so
``.grad`` accumulation, tensor hooks and DDP see ordinary leaves.  Its forward runs the inference kernels and keeps what the backward
reads: the encoder records of :mod:`encoder_grad`, and per generator level the input, both StyledConv activations (the gate is
``out > 0``; the last level keeps its conv2 activation too) and, on VToonify-D, Fusion's ``m_E``, ``f_E * m_E`` (the fusion route that
writes it) and the AdaIN statistics and gamma|beta rows of its mask head.

The backward stays NHWC and follows ``set_precision`` for every input gradient:
  * ToRGB + conv2's gate: ``ops.torgb_gate_grad`` adds ``w_rgb[b]^T g_rgb`` to the activation's gradient reading the planar image
    gradient directly; the skip image's gradient is the adjoint of its Upsample, ``upfirdn2d`` with down 2;
  * conv2 (3x3, per-sample modulated weights): ``conv_transpose_nhwc`` on the transposed modulated weights (the taps flip through
    ``tap_w``);
  * conv1 (Blur o conv_transpose stride 2): Blur's adjoint ``fir_nhwc(pad (2, 2))``, then a stride-2 3x3 convolution with the
    transposed, unflipped modulated weights;
  * Fusion (T): input and weight gradients of both concat halves on the existing cores;
  * Fusion (D): ``ops.fusion_mask_grad`` (g_z and conv2's bias gradient), ``ops.fusion_adain_grad_stats`` (the AdaIN-backward sums
    over the virtual concat, also dgamma and dbeta) and ``ops.fusion_input_grad`` (g_{f_G}, g_{f_E}); conv2's weight gradient on the
    re-applied AdaIN; the label MLP (``linear``, ``norm.style``, [B, <= 4C] rows) by torch autograd;
  * the encoder: :func:`encoder_grad._backward` with the fusion's gradients injected at ``encoder_features`` and ``skip``.
No gradient reaches ``generator.*``, ``res.*`` or ``style`` (requiring one raises); no double backward.
"""
import torch
import torch.nn.functional as F
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import encoder_grad, ops
from .op.conv2d_gradfix import _pad_rows, conv_transpose_nhwc, weight_grad_nhwc

_S2_TAPS = [(ky, kx, ky * 3 + kx) for ky in range(3) for kx in range(3)]     # stride-2 3x3 on the (2H+1)^2 blur-adjoint grid


def trained_params(model):
    """The Function's parameter inputs, in a fixed order."""
    return tuple(model.encoder.parameters()) + tuple(model.fusion_out.parameters()) + tuple(model.fusion_skip.parameters())


def takes_autograd(model, x) -> bool:
    """Grad mode is on and ``x`` or a parameter of ``encoder``, ``fusion_out`` or ``fusion_skip`` requires grad."""
    return torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in trained_params(model)))


def _check_frozen(model, style):
    named = [("style", style)] + [(n, p) for n, p in model.named_parameters() if n.startswith(("generator.", "res."))]
    for name, t in named:
        if t.requires_grad:
            raise NotImplementedError(
                f"VToonify.forward trains the encoder and the fusion modules only and propagates no gradient into the frozen generator "
                f"path, but `{name}` requires grad: call `{name}.requires_grad_(False)` (train_vtoonify_d.py and train_vtoonify_t.py "
                f"freeze `generator` and `res` this way)")


def _cached(owner, name, key, make):
    hit = getattr(owner, name, None)
    if hit is None or hit[0] != key:
        hit = (key, make())
        setattr(owner, name, hit)
    return hit[1]


# ------------------------------------------------------------------------------------------------ forward
def _forward_train(model, x, adastyles, resstyles, d_s):
    """The generator-tail forward on NHWC ``x`` -> (image, [m_E], records)."""
    D = model.backbone == "dualstylegan"
    feat, skip, erec = encoder_grad._forward_train(model, x, resstyles, d_s)
    enc_out = [r[4] for r in erec if r[0] == "conv"][1::2][::-1]      # encoder_features: each block's output, deepest first
    G = model.stylegan()
    out, levels, m_Es = feat, [], []
    for lvl, (conv1, conv2, to_rgb) in enumerate(zip(G.convs[6::2], G.convs[7::2], G.to_rgbs[3:])):
        i = 2 * lvl + 1
        fr = None
        if 2 ** (5 + lvl) <= model.in_size:
            f_E = enc_out[lvl]
            fr = {"f_G": out, "f_E": f_E, "skip": skip}
            if D:
                out, m_E, fEm = model.fusion_out[lvl].forward_nhwc(out, f_E, d_s, rec=fr)
                skip = model.fusion_skip[lvl].forward_smalln(fEm, planar=skip)
                fr.update(m=m_E, fEm=fEm)
                m_Es.append(m_E)
            else:
                out = model.fusion_out[lvl].forward_nhwc(out, x2=f_E)
                skip = model.fusion_skip[lvl].forward_smalln(f_E, planar=skip)
        s1, s2, s3 = adastyles[:, i + 6], adastyles[:, i + 7], adastyles[:, i + 8]
        a1 = conv1.forward_nhwc(out, s1, zero_noise=True)
        a2, img = conv2.forward_nhwc(a1, s2, zero_noise=True, to_rgb=(to_rgb, s3, skip))
        levels.append({"fusion": fr, "x": out, "a1": a1, "a2": a2, "styles": (s1, s2, s3)})
        out, skip = a2, img
    return skip, m_Es, {"feat": feat, "erec": erec, "levels": levels, "d_s": d_s}


# ------------------------------------------------------------------------------------------------ backward
def _transposed(conv, part, cin_pad, scale=1.0):
    """Prepared transposed weight of the input channels ``part`` (a slice) of a plain 3x3 ``Conv2d``, output rows padded to 32."""
    w = conv.weight
    return _cached(conv, f"_wt_{part.start}_{part.stop}_{cin_pad}", (w.data_ptr(), w._version, ops.get_precision()),
                   lambda: ops.prep_weights(_pad_rows(w.detach()[:, part].transpose(0, 1), 32), None, scale, False, cin_pad))


def _conv_transpose3(g, wt, H, W, res=None):
    return conv_transpose_nhwc(g, wt, 3, 3, 1, (1, 1), (1, 1), H, W, res=res)


def _wgrad_halves(conv, g, halves):
    """Weight gradient of a 3x3 convolution on a virtual concat: one weight-gradient launch per half ``(src NHWC, channels)``."""
    M = conv.weight.shape[0]
    parts = [weight_grad_nhwc(g, s, M, n, 3, 3, 1, (1, 1), (1, 1)).reshape(M, n, 3, 3) for s, n in halves]
    return torch.cat(parts, dim=1)


def _label_mlp_grads(fusion, d_s, dgb, need, grads):
    """Fusion.linear / norm.style on [B, <= 4C] rows: torch autograd on the recomputed rows (train_vtoonify_d.py feeds one d_s)."""
    ps = [fusion.linear[0].weight, fusion.linear[0].bias, fusion.linear[2].weight, fusion.linear[2].bias,
          fusion.norm.style.weight, fusion.norm.style.bias]
    if not any(need(p) for p in ps):
        return
    with torch.enable_grad():
        leaves = [p.detach().requires_grad_() for p in ps]
        label = torch.full((dgb.shape[0], 1), float(d_s), device=dgb.device, dtype=torch.float32)
        h = F.leaky_relu(F.linear(label, leaves[0], leaves[1]), 0.2)
        h = F.leaky_relu(F.linear(h, leaves[2], leaves[3]), 0.2)
        gs = torch.autograd.grad(F.linear(h, leaves[4], leaves[5]), leaves, dgb)
    for p, g in zip(ps, gs):
        if need(p):
            grads[p] = g


def _fusion_backward(model, lvl, fr, d_s, g_out, g_skip, g_m, need, grads):
    """-> (gradient of f_G, of f_E, of the skip image before the level) from those of the fusion conv's output and of the skip image."""
    D = model.backbone == "dualstylegan"
    fo, fs = model.fusion_out[lvl], model.fusion_skip[lvl]
    f_G, f_E = fr["f_G"], fr["f_E"]
    B, H, W, C = f_G.shape
    conv = fo.conv if D else fo
    gs32 = ops.to_nhwc(g_skip, 32, round_tf32=False)
    # fusion_skip over cat(skip, P), P = f_E * m_E (D) or f_E (T): the skip half on 32 padded rows, the P half
    g_prev = ops.to_nchw(_conv_transpose3(gs32, _transposed(fs, slice(0, 3), 32), H, W), 3)
    g_P2 = _conv_transpose3(gs32, _transposed(fs, slice(3, 3 + C), 32), H, W)
    # the fusion conv over cat(f_G, P)
    g_fG = _conv_transpose3(g_out, _transposed(conv, slice(0, C), C), H, W)
    g_P = _conv_transpose3(g_out, _transposed(conv, slice(C, 2 * C), C), H, W, res=g_P2)
    P = fr["fEm"] if D else f_E
    if need(fs.weight):
        grads[fs.weight] = _wgrad_halves(fs, gs32, [(ops.to_nhwc(fr["skip"], 32, round_tf32=False), 3), (P, C)])
    if need(fs.bias):
        grads[fs.bias] = ops.channel_sum(g_skip)
    if need(conv.weight):
        grads[conv.weight] = _wgrad_halves(conv, g_out, [(f_G, C), (P, C)])
    if need(conv.bias):
        grads[conv.bias] = ops.channel_sum_nhwc(g_out)
    if not D:
        return g_fG, g_P, g_prev
    stats, gb, m = fr["stats"], fr["gb"], fr["m"]
    g_z, db2 = ops.fusion_mask_grad(g_P, f_E, m, g_m)
    w2 = _cached(fo.conv2, "_w_tapmajor", (fo.conv2.weight.data_ptr(), fo.conv2.weight._version),
                 lambda: fo.conv2.weight.detach().reshape(2 * C, 9).t().contiguous())
    sums = ops.fusion_adain_grad_stats(g_z, w2, f_G, f_E, stats)
    g_fG, g_fE = ops.fusion_input_grad(g_z, w2, f_G, f_E, stats, gb, sums, g_fG, g_P, m)
    if need(fo.conv2.weight):
        gz32 = ops.to_nhwc(g_z, 32, round_tf32=False)
        grads[fo.conv2.weight] = weight_grad_nhwc(gz32, ops.adain_apply(f_G, stats, gb, f_E), 1, 2 * C, 3, 3, 1, (1, 1),
                                                  (1, 1)).reshape(fo.conv2.weight.shape)
    if need(fo.conv2.bias):
        grads[fo.conv2.bias] = db2
    _label_mlp_grads(fo, d_s, torch.cat([sums[:, :, 1], sums[:, :, 0]], dim=1), need, grads)
    return g_fG, g_fE, g_prev


def _backward(model, rec, g_img, g_masks, need, x_channels):
    """-> (gradient of x or None, {parameter: gradient}); ``need(p)``: p wants a gradient; ``x_channels``: None when x wants none."""
    grads = {}
    G = model.stylegan()
    mods = list(zip(G.convs[6::2], G.convs[7::2], G.to_rgbs[3:]))
    g_skip, g_out, g_enc = g_img.contiguous(), None, {}
    for lvl in reversed(range(len(rec["levels"]))):
        L = rec["levels"][lvl]
        conv1, conv2, to_rgb = mods[lvl]
        s1, s2, s3 = L["styles"]
        a1, a2, xin = L["a1"], L["a2"], L["x"]
        B, H2, W2, C = a2.shape
        _, H, W, Cin = xin.shape
        w_rgb = to_rgb.conv.modulated_weights(s3, C, round_tf32=False)
        gz2 = ops.torgb_gate_grad(g_out, g_skip, w_rgb, a2, conv2.activate.negative_slope, conv2.activate.scale)
        up = to_rgb.upsample
        p0, p1 = 3 - up.pad[0], 3 - up.pad[1]          # Upsample(up 2, pad (2, 1)) transposed: down 2, pad (1, 2)
        g_skip = ops.upfirdn2d_planar(g_skip, torch.flip(up.kernel, [0, 1]), (1, 1), (up.factor, up.factor), (p0, p1, p0, p1))
        w2 = conv2.conv.modulated_weights(s2, C)
        ga1 = _conv_transpose3(gz2, w2.transpose(2, 3).contiguous(), H2, W2)
        gz1 = ops.act_grad(ga1, ref=a1, slope=conv1.activate.negative_slope, gain=conv1.activate.scale)
        blur = conv1.conv.blur
        gt = ops.fir_nhwc(gz1, torch.flip(blur.kernel, [0, 1]), (3 - blur.pad[0], 3 - blur.pad[1]))
        w1 = conv1.conv.modulated_weights(s1, Cin)
        g_out = ops.conv2d_nhwc([gt], w1.transpose(2, 3).contiguous(), _S2_TAPS, 2, H, W)
        fr = L["fusion"]
        if fr is not None:
            g_m = g_masks[lvl] if lvl < len(g_masks) else None
            g_out, g_fE, g_skip = _fusion_backward(model, lvl, fr, rec["d_s"], g_out, g_skip, g_m, need, grads)
            g_enc[id(fr["f_E"])] = g_fE
    feat = rec["feat"]
    gx, egrads = encoder_grad._backward(model, rec["erec"], feat, ops.nhwc_as_nchw_view(g_out), g_skip, need, x_channels,
                                        g_inject=g_enc)
    grads.update(egrads)
    return gx, grads


class _VToonifyGrad(Function):
    @staticmethod
    def forward(ctx, model, adastyles, resstyles, d_s, x, *params):
        img, m_Es, rec = _forward_train(model, ops.to_nhwc(x, ops._pad32(x.shape[1])), adastyles, resstyles, d_s)
        ctx.model, ctx.rec, ctx.x_channels = model, rec, x.shape[1]
        return (img,) + tuple(m_Es)

    @staticmethod
    @once_differentiable
    def backward(ctx, g_img, *g_masks):
        params = trained_params(ctx.model)
        wanted = {id(p) for p, n in zip(params, ctx.needs_input_grad[5:]) if n}
        gx, grads = _backward(ctx.model, ctx.rec, g_img, [g.contiguous() for g in g_masks], lambda p: id(p) in wanted,
                              ctx.x_channels if ctx.needs_input_grad[4] else None)
        ctx.rec = None
        return (None, None, None, None, gx) + tuple(grads.get(p) if id(p) in wanted else None for p in params)


def forward_with_grad(model, x, style, d_s, adastyles, resstyles, return_mask):
    """``image`` (and with ``return_mask`` on VToonify-D the list of ``m_E``) of VToonify.forward, with gradients to ``x`` and the
    parameters of ``encoder``, ``fusion_out`` and ``fusion_skip``."""
    _check_frozen(model, style)
    outs = _VToonifyGrad.apply(model, adastyles, resstyles, d_s, x, *trained_params(model))
    if return_mask and model.backbone == "dualstylegan":
        return outs[0], list(outs[1:])
    return outs[0]
