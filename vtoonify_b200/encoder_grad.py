"""Gradients of ``VToonify.forward(x, style, d_s, return_feat=True)``: the student half of encoder pretraining
(train_vtoonify_d.py:81-149), where ``F.mse_loss`` on ``(feat, skip)`` is back-propagated into the encoder.

The route is an autograd ``Function`` whose inputs are ``x`` and every encoder parameter, so ``.grad`` accumulation, tensor hooks
and DDP's reducer see ordinary leaves.  Its forward runs the same NHWC kernels as inference and keeps what the backward reads:
  * every LeakyReLU output (the gate is ``output > 0``, as the reference's in-place ``nn.LeakyReLU`` and ``fused_leaky_relu``
    differentiate); the two convolutions whose epilogue adds a residual after the activation (VToonifyResBlock.conv2,
    AdaResBlock.conv2) run without it and the residual sum is a separate pass, so the activation itself is kept;
  * for each AdaIN of the frozen ModRes blocks (VToonify-D, d_s != 0): the (mean, rstd) table and the gamma|beta rows the forward
    applied; the normalised tensors are never written (the backward recomputes xhat from x and the saved statistics).
The backward stays NHWC: ``ops.act_grad`` applies each gate (with the bias gradient in the same pass, or the AdaIN backward in
front of it), ``conv2d_gradfix.weight_grad_nhwc`` gives the weight gradients (bf16x3 wgmma kernel) and
``conv2d_gradfix.conv_transpose_nhwc`` the input gradients (following ``set_precision``).  No gradient reaches the frozen path
(``res.*``, ``generator.style.*``, ``style``); no double backward.
"""
import math

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ops
from ._lib import ACT_LRELU
from .op.conv2d_gradfix import _pad_rows, conv_transpose_nhwc, weight_grad_nhwc

_R2 = 1.0 / math.sqrt(2.0)


def takes_autograd(model, x) -> bool:
    """The rule of conv2d_gradfix: grad mode is on and ``x`` or an encoder parameter requires grad."""
    return torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in model.encoder.parameters()))


def _check_frozen(model, style, d_s):
    if model.backbone != "dualstylegan" or d_s == 0:
        return
    named = [("style", style)] + [(n, p) for n, p in model.named_parameters()
                                  if n.startswith("generator.style.") or (n.startswith("res.") and not n.startswith("res.0."))]
    for name, t in named:
        if t.requires_grad:
            raise NotImplementedError(
                f"VToonify.forward(return_feat=True) trains the encoder only and propagates no gradient through the frozen "
                f"ModRes path, but `{name}` requires grad: call `{name}.requires_grad_(False)` (train_vtoonify_d.py freezes "
                f"`res` and `generator` this way)")


# ------------------------------------------------------------------------------------------------ forward
def _forward_train(model, x, resstyles, d_s):
    """The return_feat forward on NHWC ``x`` (channels padded to 32) -> (feat NHWC, skip planar, records for the backward)."""
    D = model.backbone == "dualstylegan"
    rec = []
    feat = x
    for block in model.encoder[:-2]:
        mods = list(block)
        for conv, act in zip(mods[0::2], mods[1::2]):
            y = conv.forward_nhwc(feat, act=ACT_LRELU, slope=act.negative_slope, gain=1.0)
            rec.append(("conv", conv, act.negative_slope, feat, y))
            feat = y
    for ii, block in enumerate(model.encoder[-2]):
        o1 = block.conv.forward_nhwc(feat, act=ACT_LRELU, slope=0.2, gain=1.0)
        a2 = block.conv2.forward_nhwc(o1, act=ACT_LRELU, slope=0.2, gain=1.0)
        rec.append(("resblock", block, feat, o1, a2))
        feat = ops.axpby(a2, feat, _R2, _R2)                 # (lrelu(conv2) + x) / sqrt(2)
        if D and d_s != 0:
            feat = _adares_forward(model.res[ii + 1], feat, resstyles[:, ii + 1], float(d_s), rec)
    skip = model.encoder[-1].forward_smalln(feat)
    return feat, skip, rec


def _adares_forward(blk, x, s, w, rec):
    """AdaResBlock.forward_nhwc with the statistics and gamma|beta rows of both AdaINs kept for the backward."""
    B = x.shape[0]
    st1 = ops.instnorm_stats(x)
    gb1, gb2 = blk.norm.gamma_beta(s, B), blk.norm2.gamma_beta(s, B)
    if ops.affine_fusable():
        o1, st2 = blk.conv.forward_nhwc(x, src_affine=ops.adain_affine(st1, gb1), want_stats=True)
        a2 = blk.conv2.forward_nhwc(o1, src_affine=ops.adain_affine(st2, gb2))
    else:
        o1 = blk.conv.forward_nhwc(ops.adain_apply(x, st1, gb1))
        st2 = ops.instnorm_stats(o1)
        a2 = blk.conv2.forward_nhwc(ops.adain_apply(o1, st2, gb2))
    rec.append(("adares", blk, w, x, st1, gb1, o1, st2, gb2, a2))
    return ops.axpby(a2, x, w, 1.0)                          # w * conv2(...) + x


# ------------------------------------------------------------------------------------------------ backward
def _input_grad(conv, scale, g, H, W, stride, pad, dil, res=None, beta=1.0):
    """Input gradient of a k x k convolution from the output gradient ``g`` (NHWC): the transposed op, with ``beta * res``
    added in its epilogue (stride 1)."""
    k = conv.weight.shape[2]
    wt = conv._wt.get(conv.weight.transpose(0, 1), scale, g.shape[3])
    return conv_transpose_nhwc(g, wt, k, k, stride, (pad, pad), (dil, dil), H, W, res=res, beta=beta)


def _weight_grad(conv, g_pre, x, stride, pad, dil):
    Cout, Cin, k, _ = conv.weight.shape
    return weight_grad_nhwc(g_pre, x, Cout, Cin, k, k, stride, (pad, pad), (dil, dil)).reshape(conv.weight.shape)


def _backward(model, rec, feat, g_feat, g_skip, need, x_channels, g_inject=None):
    """-> (grad of x or None, {parameter: grad}) for the records of :func:`_forward_train`; ``need(p)``: p wants a gradient.
    ``g_inject`` {id(activation): NHWC gradient}: more gradient reaching an encoder block's output from outside the encoder (the
    fusion modules read ``encoder_features``), added before that block's gate."""
    grads = {}
    enc5 = model.encoder[-1]
    B, H, W, C = feat.shape
    gf = ops.to_nhwc(g_feat, round_tf32=False)                # zero-copy for the channels_last gradient of a channels_last feat
    gs = ops.to_nhwc(g_skip, ops._pad32(g_skip.shape[1]), round_tf32=False)
    # encoder.5 (1x1, C -> 3): feat receives both gradients, added in the transposed op's epilogue
    g = _input_grad(enc5, 1.0, gs, H, W, 1, 0, 1, res=gf.contiguous(), beta=1.0)
    if need(enc5.weight):
        grads[enc5.weight] = _weight_grad(enc5, gs, feat, 1, 0, 1)
    if need(enc5.bias):
        grads[enc5.bias] = ops.channel_sum(g_skip)
    gx = None
    for r in reversed(rec):
        kind = r[0]
        if kind == "adares":
            _, blk, w, x, st1, gb1, o1, st2, gb2, a2 = r
            c1, l1, c2, l2 = blk.conv[0], blk.conv[1], blk.conv2[0], blk.conv2[1]
            gp2 = ops.act_grad(g, ref=a2, slope=l2.negative_slope, gain=l2.scale * w)
            gn2 = _input_grad(c2, c2.scale, gp2, H, W, 1, c2.padding, c2.dilation)
            gp1 = ops.act_grad(gn2, ref=o1, slope=l1.negative_slope, gain=l1.scale,
                               adain=(o1, st2, gb2, ops.adain_grad_stats(gn2, o1, st2)))
            gn1 = _input_grad(c1, c1.scale, gp1, H, W, 1, c1.padding, c1.dilation)
            g = ops.act_grad(gn1, res=g, beta=1.0, adain=(x, st1, gb1, ops.adain_grad_stats(gn1, x, st1)))
        elif kind == "resblock":
            _, blk, x, o1, a2 = r
            gp2, db2 = ops.act_grad(g, ref=a2, slope=0.2, gain=_R2, bias_grad=True)
            if need(blk.conv2.weight):
                grads[blk.conv2.weight] = _weight_grad(blk.conv2, gp2, o1, 1, 1, 1)
            gp1, db1 = ops.act_grad(_input_grad(blk.conv2, 1.0, gp2, H, W, 1, 1, 1), ref=o1, slope=0.2, gain=1.0, bias_grad=True)
            if need(blk.conv.weight):
                grads[blk.conv.weight] = _weight_grad(blk.conv, gp1, x, 1, 1, 1)
            grads[blk.conv2.bias], grads[blk.conv.bias] = db2, db1
            g = _input_grad(blk.conv, 1.0, gp1, H, W, 1, 1, 1, res=g, beta=_R2)   # + the skip term g / sqrt(2)
        else:
            _, conv, slope, x, y = r
            if g_inject and id(y) in g_inject:
                g = ops.axpby(g, g_inject[id(y)], 1.0, 1.0, round_tf32=False)
            gp, db = ops.act_grad(g, ref=y, slope=slope, gain=1.0, bias_grad=True)
            grads[conv.bias] = db
            if need(conv.weight):
                grads[conv.weight] = _weight_grad(conv, gp, x, conv.stride, conv.padding, 1)
            _, H, W, _ = x.shape
            if r is not rec[0]:
                g = _input_grad(conv, 1.0, gp, H, W, conv.stride, conv.padding, 1)
            elif x_channels is not None:
                # encoder.0.0: 22 input channels padded to 32, so the transposed op's output rows are padded too
                k = conv.kernel_size
                wt = ops.prep_weights(_pad_rows(conv.weight.detach().transpose(0, 1), 32), cin_pad=gp.shape[3])
                gx = ops.to_nchw(conv_transpose_nhwc(gp, wt, k, k, conv.stride, (conv.padding,) * 2, (1, 1), H, W), x_channels)
    return gx, grads


class _FeatGrad(Function):
    @staticmethod
    def forward(ctx, model, resstyles, d_s, x, *params):
        feat, skip, rec = _forward_train(model, ops.to_nhwc(x, ops._pad32(x.shape[1])), resstyles, d_s)
        ctx.model, ctx.rec, ctx.feat, ctx.x_channels = model, rec, feat, x.shape[1]
        return ops.nhwc_as_nchw_view(feat), skip

    @staticmethod
    @once_differentiable
    def backward(ctx, g_feat, g_skip):
        params = tuple(ctx.model.encoder.parameters())       # the order of the inputs
        wanted = {id(p) for p, n in zip(params, ctx.needs_input_grad[4:]) if n}
        gx, grads = _backward(ctx.model, ctx.rec, ctx.feat, g_feat, g_skip, lambda p: id(p) in wanted,
                              ctx.x_channels if ctx.needs_input_grad[3] else None)
        ctx.rec = ctx.feat = None
        return (None, None, None, gx) + tuple(grads.get(p) if id(p) in wanted else None for p in params)


def feat_with_grad(model, x, style, d_s, resstyles):
    """``(feat, skip)`` of VToonify.forward(return_feat=True) with gradients to ``x`` and the encoder parameters."""
    _check_frozen(model, style, d_s)
    params = tuple(model.encoder.parameters())
    return _FeatGrad.apply(model, resstyles, d_s, x, *params)
