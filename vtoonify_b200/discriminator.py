"""Forward and gradients of ``ConditionalDiscriminator`` (model/vtoonify.py:10-89), the discriminator of both VToonify training
scripts: its D step differentiates into the parameters, its G step into the input image.

One route.  The forward runs NHWC on the library's kernels: ``convs.0`` and every ``conv1`` on the convolution kernel with bias +
FusedLeakyReLU in the epilogue; per ResBlock two pad (2, 2) blurs (of conv1's output for conv2, of the block input for the skip),
conv2 at stride 2 and the skip at stride 2 whose epilogue forms the block output; ``vt_mbstd_nhwc_f32`` writes ``final_conv``'s
padded 544-channel input; ``final_linear`` on ``vt_linear_f32``, with its weight's columns permuted once to the NHWC flattening.
Under autograd the same launches keep what the backward reads (the gate references and both blurred tensors per block).

The autograd ``Function``'s inputs are ``x`` and every parameter of ``convs``, ``final_conv`` and ``final_linear``, so ``.grad``
accumulation, hooks and DDP see ordinary leaves.  The backward, by piece:
  * gates and bias gradients: ``ops.act_grad`` (block output (a2 + skip)/sqrt2 with a2 = lrelu(z2)*sqrt2: dz2 = gate * g; the
    skip's 1/sqrt2 is folded into its transposed weight's scale);
  * weight gradients: ``weight_grad_nhwc`` on the kept tensors (conv2 and the skip at stride 2 on their blurred inputs);
  * conv2's input gradient: the adjoint of Blur(pad (2, 2)) o conv(stride 2) is the generator's up-convolution with the blur
    kernel K (not 4K): ``fold_upconv_weights`` + ``conv_up2_folded_nhwc``, one launch, no (2H+1)^2 intermediate;
  * the skip's input gradient: the transposed 1x1 stride-2 conv onto the odd pixels of the (H+1)^2 grid, then the blur's adjoint
    ``fir_nhwc(pad (1, 1))``; it is added in the epilogue of conv1's transposed convolution;
  * the minibatch standard deviation: ``vt_mbstd_grad_nhwc_f32``;
  * ``final_linear``: input gradients with ``vt_linear_f32`` on the cached transposed weights, weight gradients as 1x1 weight
    gradients over ``[B, 1, 1, C]`` maps.
Gradients follow ``ctx.needs_input_grad``: without a parameter requiring grad (G step) no weight- or bias-gradient launch runs; without
``x`` requiring grad (D step) ``convs.0`` computes no input gradient.  No double backward.
"""
import math

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ops
from .op.conv2d_gradfix import _pad_rows, conv_transpose_nhwc

_R2 = 1.0 / math.sqrt(2.0)


def stddev_group(D, B):
    """The reference's ``group = min(B, 4)``; a batch it does not divide is rejected, as the reference's ``view`` rejects it."""
    group = min(B, D.stddev_group)
    if B % group:
        raise ValueError(f"ConditionalDiscriminator: batch {B} is not a multiple of the minibatch-stddev group {group}")
    return group


def trained_params(D):
    """The Function's parameter inputs, in a fixed order."""
    return tuple(D.convs.parameters()) + tuple(D.final_conv.parameters()) + tuple(D.final_linear.parameters())


def takes_autograd(D, x) -> bool:
    return torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in trained_params(D)))


def _cached(owner, name, key, make):
    hit = getattr(owner, name, None)
    if hit is None or hit[0] != key:
        hit = (key, make())
        setattr(owner, name, hit)
    return hit[1]


def _wkey(*ts):
    return tuple((t.data_ptr(), t._version) for t in ts) + (ops.get_precision(),)


def _lin0_weight(D, C, H, W):
    """final_linear.0's weight with its columns in NHWC flattening order (h, w, c) instead of the reference's (c, h, w)."""
    w = D.final_linear[0].weight
    return _cached(D.final_linear[0], "_w_nhwc", _wkey(w),
                   lambda: w.detach().reshape(w.shape[0], C, H, W).permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous())


# ------------------------------------------------------------------------------------------------ forward
def forward_nhwc(D, x, rec=None):
    """``x`` NCHW [B, 3, H, W] -> ``final_linear`` output [B, condition_dim]; ``rec`` (a dict): filled with what the backward reads."""
    B = x.shape[0]
    group = stddev_group(D, B)
    xin = ops.to_nhwc(x, ops._pad32(x.shape[1]))
    h = D.convs[0].forward_nhwc(xin)
    blocks = [] if rec is not None else None
    for blk in D.convs[1:]:
        h = blk.forward_nhwc(h, blocks)
    f = ops.mbstd(h, group)
    af = D.final_conv.forward_nhwc(f)
    _, Hf, Wf, Cf = af.shape
    l0, l1 = D.final_linear
    flat = af.reshape(B, -1)
    o0 = ops.linear(flat, _lin0_weight(D, Cf, Hf, Wf), l0.bias, l0.scale, l0.lr_mul, 1)
    out = ops.linear(o0, l1.weight, l1.bias, l1.scale, l1.lr_mul, 1 if l1.activation else 0)
    if rec is not None:
        rec.update(group=group, xin=xin, blocks=blocks, h=h, f=f, af=af, flat=flat, o0=o0, out=out)
    return out


# ------------------------------------------------------------------------------------------------ backward
def _scaled(t, s):
    return t if s == 1.0 else ops.axpby(t, None, s, round_tf32=False)


def _bias_grad(db, lr_mul):
    return _scaled(db, lr_mul)


def _conv_wgrad(conv, g_pre, src, stride, taps):
    Cout, Cin, k, _ = conv.weight.shape
    wg = ops.conv_wgrad_nhwc(g_pre, src, Cout, Cin, taps, stride, False)
    return _scaled(wg, conv.scale).reshape(conv.weight.shape)


def _taps(k, off):
    return [(ky + off, kx + off) for ky in range(k) for kx in range(k)]


def _linear_backward(lin, g, src, need, grads, act_ref=None):
    """EqualLinear ``y = act(src @ (scale W)^T + lr_mul b)``: ``g`` [B, out] -> input gradient [B, in]."""
    if act_ref is not None:
        g4 = g.reshape(g.shape[0], 1, 1, g.shape[1])
        if need(lin.bias):
            g4, db = ops.act_grad(g4, ref=act_ref.reshape(g4.shape), slope=0.2, gain=math.sqrt(2.0), bias_grad=True)
            grads[lin.bias] = _bias_grad(db, lin.lr_mul)
        else:
            g4 = ops.act_grad(g4, ref=act_ref.reshape(g4.shape), slope=0.2, gain=math.sqrt(2.0))
        g = g4.reshape(g.shape)
    elif need(lin.bias):
        grads[lin.bias] = _bias_grad(ops.channel_sum(g), lin.lr_mul)
    if need(lin.weight):
        M, N = g.shape[1], src.shape[1]
        a = g.reshape(g.shape[0], 1, 1, M)
        if M % 32:
            a = ops.to_nhwc(g.reshape(g.shape[0], M, 1, 1), ops._pad32(M), round_tf32=False)
        s4 = src.reshape(src.shape[0], 1, 1, N).contiguous()
        grads[lin.weight] = _scaled(ops.conv_wgrad_nhwc(a, s4, M, N, [(0, 0)], 1, False), lin.scale).reshape(M, N)
    return g


def _block_backward(blk, r, g, need, grads):
    """ResBlock backward: ``g`` = gradient of the block output -> gradient of the block input."""
    _, x, a1, a1b, a2, xb = r
    c1, l1 = blk.conv1[0], blk.conv1[1]
    c2, l2 = blk.conv2[1], blk.conv2[2]
    cs = blk.skip[1]
    K = blk.conv2[0].kernel
    B, H, W, Cin = x.shape
    want_w = need(c2.weight) or need(l2.bias)
    if want_w:
        gp2, db2 = ops.act_grad(g, ref=a2, slope=l2.negative_slope, gain=l2.scale * _R2, bias_grad=True)
        grads[l2.bias] = db2
    else:
        gp2 = ops.act_grad(g, ref=a2, slope=l2.negative_slope, gain=l2.scale * _R2)
    if need(c2.weight):
        grads[c2.weight] = _conv_wgrad(c2, gp2, a1b, 2, _taps(3, 0))
    if need(cs.weight):
        wg = ops.conv_wgrad_nhwc(g, xb, cs.weight.shape[0], Cin, [(1, 1)], 2, False)
        grads[cs.weight] = _scaled(wg, cs.scale * _R2).reshape(cs.weight.shape)
    # conv2's input gradient: Blur(pad (2, 2)) o conv(stride 2) transposed = the folded up-convolution with kernel K
    wf = _cached(c2, "_wt_folded", _wkey(c2.weight, K), lambda: ops.fold_upconv_weights(
        ops.prep_weights(c2.weight.detach().transpose(0, 1), None, c2.scale, False, g.shape[3], round_tf32=False), K))
    ga1 = ops.conv_up2_folded_nhwc(gp2, wf)
    if need(c1.weight) or need(l1.bias):
        gp1, db1 = ops.act_grad(ga1, ref=a1, slope=l1.negative_slope, gain=l1.scale, bias_grad=True)
        grads[l1.bias] = db1
    else:
        gp1 = ops.act_grad(ga1, ref=a1, slope=l1.negative_slope, gain=l1.scale)
    if need(c1.weight):
        grads[c1.weight] = _conv_wgrad(c1, gp1, x, 1, _taps(3, -1))
    # the skip's input gradient: transposed 1x1 stride-2 conv onto the odd pixels of the (H+1)^2 blur grid, then the blur's adjoint
    wts = cs._wt.get(cs.weight.transpose(0, 1), cs.scale * _R2, g.shape[3])
    gxb = conv_transpose_nhwc(g, wts, 1, 1, 2, (-1, -1), (1, 1), H + 1, W + 1)
    gskip = ops.fir_nhwc(gxb, K, (1, 1))
    wt1 = c1._wt.get(c1.weight.transpose(0, 1), c1.scale, gp1.shape[3])
    return conv_transpose_nhwc(gp1, wt1, 3, 3, 1, (1, 1), (1, 1), H, W, res=gskip, beta=1.0)


def backward_nhwc(D, rec, g_out, need, x_channels):
    """-> (gradient of x or None, {parameter: gradient}); ``need(p)``: p wants a gradient; ``x_channels``: None when x wants none."""
    grads = {}
    l0, l1 = D.final_linear
    B = g_out.shape[0]
    g_out = g_out.contiguous()
    g0 = _linear_backward(l1, g_out, rec["o0"], need, grads, act_ref=rec["out"] if l1.activation else None)
    w1t = _cached(l1, "_wt_lin", _wkey(l1.weight), lambda: l1.weight.detach().t().contiguous())
    go0 = ops.linear(g0, w1t, None, l1.scale)
    af = rec["af"]
    _, Hf, Wf, Cf = af.shape
    gp0 = _linear_backward(l0, go0, rec["flat"], need, grads, act_ref=rec["o0"])
    if need(l0.weight):   # computed in NHWC column order: back to the reference's (c, h, w)
        grads[l0.weight] = grads[l0.weight].reshape(-1, Hf, Wf, Cf).permute(0, 3, 1, 2).reshape(l0.weight.shape).contiguous()
    w0t = _cached(l0, "_wt_lin", _wkey(l0.weight), lambda: _lin0_weight(D, Cf, Hf, Wf).t().contiguous())
    gaf = ops.linear(gp0, w0t, None, l0.scale).reshape(af.shape)
    # final_conv (3x3 on the 544-channel stddev tensor)
    fc, fl = D.final_conv[0], D.final_conv[1]
    f = rec["f"]
    if need(fc.weight) or need(fl.bias):
        gpf, dbf = ops.act_grad(gaf, ref=af, slope=fl.negative_slope, gain=fl.scale, bias_grad=True)
        grads[fl.bias] = dbf
    else:
        gpf = ops.act_grad(gaf, ref=af, slope=fl.negative_slope, gain=fl.scale)
    if need(fc.weight):
        grads[fc.weight] = _conv_wgrad(fc, gpf, f, 1, _taps(3, -1))
    wtf = _cached(fc, "_wt_pad", _wkey(fc.weight), lambda: ops.prep_weights(
        _pad_rows(fc.weight.detach().transpose(0, 1), 32), None, fc.scale, False, gpf.shape[3]))
    gf = conv_transpose_nhwc(gpf, wtf, 3, 3, 1, (1, 1), (1, 1), Hf, Wf)          # [B, 4, 4, 544]: the padded stddev layout
    g = ops.mbstd_grad(gf, rec["h"], rec["group"])
    for r in reversed(rec["blocks"]):
        g = _block_backward(r[0], r, g, need, grads)
    # convs.0: 1x1, 3 -> C on the 32-channel padded input
    c0, a0 = D.convs[0][0], D.convs[0][1]
    xin = rec["xin"]
    h0 = rec["blocks"][0][1] if rec["blocks"] else rec["h"]
    if need(c0.weight) or need(a0.bias):
        gp, db = ops.act_grad(g, ref=h0, slope=a0.negative_slope, gain=a0.scale, bias_grad=True)
        grads[a0.bias] = db
    else:
        gp = ops.act_grad(g, ref=h0, slope=a0.negative_slope, gain=a0.scale)
    if need(c0.weight):
        grads[c0.weight] = _conv_wgrad(c0, gp, xin, 1, [(0, 0)])
    gx = None
    if x_channels is not None:
        wt = ops.prep_weights(_pad_rows(c0.weight.detach().transpose(0, 1), 32), None, c0.scale, False, gp.shape[3])
        _, H, W, _ = xin.shape
        gx = ops.to_nchw(conv_transpose_nhwc(gp, wt, 1, 1, 1, (0, 0), (1, 1), H, W), x_channels)
    return gx, grads


class _DiscGrad(Function):
    @staticmethod
    def forward(ctx, D, x, *params):
        rec = {}
        out = forward_nhwc(D, x, rec)
        ctx.D, ctx.rec, ctx.x_channels = D, rec, x.shape[1]
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out):
        params = trained_params(ctx.D)
        wanted = {id(p) for p, n in zip(params, ctx.needs_input_grad[2:]) if n}
        gx, grads = backward_nhwc(ctx.D, ctx.rec, g_out, lambda p: id(p) in wanted,
                                  ctx.x_channels if ctx.needs_input_grad[1] else None)
        ctx.rec = None
        return (None, gx) + tuple(grads.get(p) if id(p) in wanted else None for p in params)


def final_linear_out(D, x):
    """``final_linear`` output of the discriminator on NCHW ``x``: through the Function when autograd needs it."""
    if takes_autograd(D, x):
        return _DiscGrad.apply(D, x, *trained_params(D))
    return forward_nhwc(D, x)

