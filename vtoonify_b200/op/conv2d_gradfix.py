"""``conv2d_gradfix.conv2d`` / ``conv_transpose2d`` — same call signatures as model/stylegan/op/conv2d_gradfix.py:22-75.
In the reference these forward to cuDNN (F.conv2d / F.conv_transpose2d) on any modern torch; here they run the
library's NHWC convolution kernels (wgmma when shapes allow, fp32 FFMA otherwise).

Supported
  * ``conv2d``: kernels of up to 36 taps (any kh x kw), per-axis padding / dilation, stride s (same on both axes),
    ``groups == 1`` or the form ``ModulatedConv2d`` uses (model/stylegan/model.py:291-301): ``input [1, G*Cin, H, W]``,
    ``weight [G*Cout, Cin, kh, kw]``, ``groups = G`` — the groups are the samples of the batch, so the call is the same
    implicit GEMM with per-sample weight tiles (``wB = G``, selected by the TMA batch coordinate), not a grouped conv.
  * ``conv_transpose2d``: stride 2, padding 0, 3x3 (the only form the reference uses, model.py:236-238, 281-283), with
    ``groups == 1`` or ``groups = G`` as above (``weight [G*Cin, Cout, 3, 3]``).
Everything else raises ``NotImplementedError`` (never a silently wrong shape).  Inputs / outputs are planar NCHW like
``F.conv2d``'s (a channels_last view is returned when the layout allows it without a copy).

Differentiable like the reference (conv2d_gradfix.py:104-227): when grad mode is on and ``input``, ``weight`` or ``bias`` requires
grad, the call goes through a custom autograd ``Function`` with a double backward; every other call runs the forward kernels
directly, with bit-identical results either way.
  * input gradient: the transposed op, run on the forward kernels (and following ``set_precision``): a stride-1 convolution with
    the per-tap transposed weight at taps ``pad - k*dil``, or for stride 2 one such convolution per output phase writing a strided
    view of the gradient (a phase no tap reaches is zero);
  * weight gradient: the wgmma weight-gradient kernel (``ops.conv_wgrad_nhwc``, bf16x3 arithmetic whatever the precision setting),
    skipped inside ``no_weight_gradients()`` (the R1 penalty, util.py:75-80);
  * bias gradient: ``ops.channel_sum`` of the output gradient;
  * second derivatives: the weight gradient's own backward is the forward op with the weight gradient's gradient as weight, plus
    the transposed op.
The transposed op used internally takes stride 1 or 2, any padding, output padding and dilation; the public ``conv_transpose2d``
keeps the limits above."""
import contextlib

import torch
from torch.autograd import Function

from .. import ops

enabled = True
weight_gradients_disabled = False


@contextlib.contextmanager
def no_weight_gradients():
    global weight_gradients_disabled
    old = weight_gradients_disabled
    weight_gradients_disabled = True
    yield
    weight_gradients_disabled = old


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(int(t) for t in v)


def _taps(kh, kw, pad, dil):
    return [(ky * dil[0] - pad[0], kx * dil[1] - pad[1], ky * kw + kx) for ky in range(kh) for kx in range(kw)]


def _group_view(input, groups):
    """``[N, G*C, H, W]`` seen as ``G`` samples of ``C`` channels (N must be 1, as in ModulatedConv2d.forward)."""
    N, GC, H, W = input.shape
    if groups == 1:
        return input, N
    if N != 1 or GC % groups:
        raise NotImplementedError("vtoonify_b200 conv2d_gradfix: groups > 1 is supported in the ModulatedConv2d form only "
                                  "(input [1, groups*Cin, H, W]: one group per sample of the batch)")
    return input.reshape(groups, GC // groups, H, W), groups


def _prep_grouped(weight5, cin_pad):
    """``[G, Cout, Cin, kh, kw]`` -> kernel layout ``[G, kh*kw, Cout, cin_pad]`` (one re-layout launch per group)."""
    G, Cout, Cin, kh, kw = weight5.shape
    out = torch.empty((G, kh * kw, Cout, cin_pad), device=weight5.device, dtype=torch.float32)
    for g in range(G):
        ops.prep_weights(weight5[g], cin_pad=cin_pad, out=out[g:g + 1])
    return out


def _pad_rows(weight, mult):
    """zero-pad dim 0 (output channels) of a ``[Cout, ...]`` weight to a multiple of ``mult``"""
    cout = weight.shape[0]
    cpad = (cout + mult - 1) // mult * mult
    if cpad == cout:
        return weight.contiguous()
    wp = torch.zeros((cpad,) + tuple(weight.shape[1:]), device=weight.device, dtype=weight.dtype)
    wp[:cout] = weight
    return wp


def _conv2d_forward(input, weight, bias, s, p, d, groups):
    GCout, Cin, kh, kw = weight.shape
    if kh * kw > 36:
        raise NotImplementedError("vtoonify_b200 conv2d: kernels of up to 36 taps")
    x4, B = _group_view(input, groups)
    if x4.shape[1] != Cin:
        raise ValueError(f"conv2d: weight expects {Cin} input channels per group, input has {x4.shape[1]}")
    if GCout % groups:
        raise ValueError("conv2d: out_channels not divisible by groups")
    Cout = GCout // groups
    _, C, H, W = x4.shape
    Ho = ops.conv_out_size(H, kh, s[0], p[0], d[0])
    Wo = ops.conv_out_size(W, kw, s[0], p[1], d[1])
    if Ho < 1 or Wo < 1:
        raise ValueError("conv2d: empty output")
    x = ops.to_nhwc(x4, ops._pad32(C) if C % 32 else None)
    taps = _taps(kh, kw, p, d)
    same = (Ho, Wo) == (H, W) and s[0] == 1
    if groups == 1 and Cout <= 4 and same:
        # planar-output CUDA-core head (always writes [B, Cout, H, W] with zero padding: 'same' geometry only)
        w = ops.prep_weights(weight, cin_pad=x.shape[3], round_tf32=False)
        return ops.smalln_conv(x, w, taps, Cout, B, H, W, bias=bias)
    cpad = ops._pad32(Cout) if Cout >= 32 or Cout % 4 else Cout        # tensor cores want Cout % 32 == 0; FFMA kernel % 4
    if groups == 1:
        w = ops.prep_weights(_pad_rows(weight, cpad), cin_pad=x.shape[3])
        b = bias
    else:
        w5 = weight.reshape(groups, Cout, Cin, kh, kw)
        if cpad != Cout:
            w5 = torch.cat([w5, w5.new_zeros((groups, cpad - Cout, Cin, kh, kw))], dim=1)
        w = _prep_grouped(w5.contiguous(), x.shape[3])
        b = None                                                        # a grouped bias is per (group, channel): added below
    if b is not None and cpad != Cout:
        b = torch.cat([b, b.new_zeros(cpad - Cout)])
    y = ops.conv2d_nhwc([x], w, taps, s[0], Ho, Wo, bias=b)             # [B, Ho, Wo, cpad]
    if groups == 1:
        out = ops.nhwc_as_nchw_view(y)
        return out if cpad == Cout else out[:, :Cout]
    # [G, Ho, Wo, Cout] -> the reference's [1, G*Cout, Ho, Wo] (needs planar memory: one transposing pass)
    out = ops.to_nchw(y, Cout).reshape(1, groups * Cout, Ho, Wo)
    if bias is not None:
        out = ops.fused_bias_act(out, bias, 1.0, 1.0)                   # slope 1, gain 1: x + bias[c]
    return out


def _conv_transpose2d_s2_k3_forward(input, weight, bias, groups):
    x4, B = _group_view(input, groups)
    GCin, Cout = weight.shape[:2]                       # F.conv_transpose2d weight is [G*Cin, Cout, kh, kw]
    Cin = GCin // groups
    if x4.shape[1] != Cin:
        raise ValueError(f"conv_transpose2d: weight expects {Cin} input channels per group, input has {x4.shape[1]}")
    x = ops.to_nhwc(x4, ops._pad32(Cin) if Cin % 32 else None)
    cpad = ops._pad32(Cout) if Cout >= 32 or Cout % 4 else Cout
    w5 = weight.reshape(groups, Cin, Cout, 3, 3).transpose(1, 2)        # [G, Cout, Cin, 3, 3]
    if cpad != Cout:
        w5 = torch.cat([w5, w5.new_zeros((groups, cpad - Cout, Cin, 3, 3))], dim=1)
    w = _prep_grouped(w5.contiguous(), x.shape[3]) if groups > 1 else ops.prep_weights(w5[0].contiguous(), cin_pad=x.shape[3])
    y = ops.conv_transpose2d_s2_k3_nhwc(x, w)          # [B, 2H+1, 2W+1, cpad]
    if groups == 1:
        out = ops.nhwc_as_nchw_view(y)
        out = out if cpad == Cout else out[:, :Cout]
    else:
        out = ops.to_nchw(y, Cout).reshape(1, groups * Cout, y.shape[1], y.shape[2])
    if bias is not None:
        out = ops.fused_bias_act(out, bias, 1.0, 1.0)                   # slope 1, gain 1: x + bias[c]
    return out


def _conv_transpose2d_forward(input, weight, bias, s, p, op, d, groups):
    """F.conv_transpose2d with stride 1 or 2 (same on both axes), any padding / output padding / dilation: one stride-1
    convolution per output phase (py, px), each writing the strided view out[:, py::s, px::s] of the result.  Output row
    o = s*j + py receives input row j + (py + pad - ky*dil) / s through tap ky wherever that division is exact."""
    if s == (2, 2) and p == (0, 0) and op == (0, 0) and d == (1, 1) and tuple(weight.shape[2:]) == (3, 3):
        return _conv_transpose2d_s2_k3_forward(input, weight, bias, groups)
    if s[0] != s[1] or s[0] not in (1, 2):
        raise NotImplementedError("vtoonify_b200 conv_transpose2d: stride 1 or 2, the same on both axes")
    st = s[0]
    x4, B = _group_view(input, groups)
    GCin, Cout, kh, kw = weight.shape
    Cin = GCin // groups
    if x4.shape[1] != Cin:
        raise ValueError(f"conv_transpose2d: weight expects {Cin} input channels per group, input has {x4.shape[1]}")
    if kh * kw > 36:
        raise NotImplementedError("vtoonify_b200 conv_transpose2d: kernels of up to 36 taps")
    _, _, H, W = x4.shape
    Ho = (H - 1) * st - 2 * p[0] + d[0] * (kh - 1) + op[0] + 1
    Wo = (W - 1) * st - 2 * p[1] + d[1] * (kw - 1) + op[1] + 1
    if Ho < 1 or Wo < 1:
        raise ValueError("conv_transpose2d: empty output")
    x = ops.to_nhwc(x4, ops._pad32(Cin) if Cin % 32 else None)
    cpad = ops._pad32(Cout) if Cout >= 32 or Cout % 4 else Cout
    w5 = weight.reshape(groups, Cin, Cout, kh, kw).transpose(1, 2)        # [G, Cout, Cin, kh, kw]
    if cpad != Cout:
        w5 = torch.cat([w5, w5.new_zeros((groups, cpad - Cout, Cin, kh, kw))], dim=1)
    w = _prep_grouped(w5.contiguous(), x.shape[3]) if groups > 1 else ops.prep_weights(w5[0].contiguous(), cin_pad=x.shape[3])
    y = conv_transpose_nhwc(x, w, kh, kw, st, p, d, Ho, Wo)
    out = ops.to_nchw(y, Cout)
    if groups > 1:
        out = out.reshape(1, groups * Cout, Ho, Wo)
    if bias is not None:
        out = ops.fused_bias_act(out, bias, 1.0, 1.0)
    return out


def conv_transpose_nhwc(x, w, kh, kw, st, p, d, Ho, Wo, res=None, beta=1.0):
    """The NHWC core of the transposed op: ``x`` [B, H, W, cin_pad], ``w`` [wB, kh*kw, Cout, cin_pad] from ``prep_weights`` of the
    [Cout, Cin, kh, kw] view of a transposed-conv weight (slab ky*kw + kx, not flipped) -> [B, Ho, Wo, Cout].  One stride-1
    convolution per output phase (py, px) writes the strided view y[:, py::st, px::st]: output row o = st*j + py receives input row
    j + (py + pad - ky*dil) / st through tap ky wherever that division is exact.  ``res`` (stride 1 only): ``beta * res`` is
    added in the convolution's epilogue."""
    B, cout = x.shape[0], w.shape[2]
    if res is not None and st != 1:
        raise NotImplementedError("conv_transpose_nhwc: a residual needs stride 1")
    y = torch.empty((B, Ho, Wo, cout), device=x.device, dtype=torch.float32)
    for py in range(st):
        for px in range(st):
            Hp, Wp = (Ho - py + st - 1) // st, (Wo - px + st - 1) // st
            if Hp < 1 or Wp < 1:
                continue
            taps = [((py + p[0] - ky * d[0]) // st, (px + p[1] - kx * d[1]) // st, ky * kw + kx)
                    for ky in range(kh) for kx in range(kw)
                    if (py + p[0] - ky * d[0]) % st == 0 and (px + p[1] - kx * d[1]) % st == 0]
            if not taps:
                y[:, py::st, px::st].zero_()
                continue
            if st == 1:
                ops.conv2d_nhwc([x], w, taps, 1, Hp, Wp, out=y, res=res, beta=beta)
            else:
                view = ((py * Wo + px) * cout, Ho * Wo * cout, st * Wo * cout, st * cout)
                ops.conv2d_nhwc([x], w, taps, 1, Hp, Wp, out=y, out_view=view)
    return y


def weight_grad_nhwc(a, src, M, N, kh, kw, s, p, d, per_sample=False):
    """Weight gradient of a convolution with stride ``s``, padding ``p`` and dilation ``d`` on NHWC operands (channel strides that
    are multiples of 32): ``a`` holds the M output-side channels, ``src`` the N input-side ones -> [nb * M, N, kh*kw]."""
    taps = [(ky * d[0] - p[0], kx * d[1] - p[1]) for ky in range(kh) for kx in range(kw)]
    return ops.conv_wgrad_nhwc(a, src, M, N, taps, s, per_sample)


def _weight_grad(transpose, weight_shape, grad_output, input, s, p, d, groups):
    """conv2d: sum over pixels of grad_output[o] (x) input[s*o + k*dil - pad]; conv_transpose2d: input[i] (x)
    grad_output[s*i + k*dil - pad].  Both are the [M][N][kh][kw] reduction of the weight-gradient kernel."""
    kh, kw = weight_shape[2], weight_shape[3]
    go4, _ = _group_view(grad_output, groups)
    x4, _ = _group_view(input, groups)
    a4, s4 = (x4, go4) if transpose else (go4, x4)
    M, N = a4.shape[1], s4.shape[1]
    a = ops.to_nhwc(a4, ops._pad32(M), round_tf32=False)
    src = ops.to_nhwc(s4, ops._pad32(N), round_tf32=False)
    return weight_grad_nhwc(a, src, M, N, kh, kw, s[0], p, d, groups > 1).reshape(weight_shape)


class _ChannelSum(Function):
    """grad_bias = grad_output.sum((0, 2, 3)), differentiable (its gradient is a broadcast)"""

    @staticmethod
    def forward(ctx, x):
        ctx.shape = tuple(x.shape)
        return ops.channel_sum(x)

    @staticmethod
    def backward(ctx, g):
        return g.reshape((1, -1) + (1,) * (len(ctx.shape) - 2)).expand(ctx.shape)


_gradfix_cache = dict()


def _conv2d_gradfix(transpose, weight_shape, stride, padding, output_padding, dilation, groups):
    """The reference's autograd pair (conv2d_gradfix.py:104-227) on this library's kernels, cached per configuration."""
    key = (transpose, weight_shape, stride, padding, output_padding, dilation, groups)
    if key in _gradfix_cache:
        return _gradfix_cache[key]

    def calc_output_padding(input_shape, output_shape):
        if transpose:
            return (0, 0)
        return tuple(input_shape[i + 2] - (output_shape[i + 2] - 1) * stride[i] - (1 - 2 * padding[i])
                     - dilation[i] * (weight_shape[i + 2] - 1) for i in range(2))

    def transposed_op(input_shape, output_shape):
        return _conv2d_gradfix(not transpose, weight_shape, stride, padding, calc_output_padding(input_shape, output_shape),
                               dilation, groups)

    class Conv2d(Function):
        @staticmethod
        def forward(ctx, input, weight, bias):
            if transpose:
                out = _conv_transpose2d_forward(input, weight, bias, stride, padding, output_padding, dilation, groups)
            else:
                out = _conv2d_forward(input, weight, bias, stride, padding, dilation, groups)
            ctx.save_for_backward(input, weight)
            return out

        @staticmethod
        def backward(ctx, grad_output):
            input, weight = ctx.saved_tensors
            grad_input = grad_weight = grad_bias = None
            if ctx.needs_input_grad[0]:
                grad_input = transposed_op(input.shape, grad_output.shape).apply(grad_output, weight, None).contiguous()
            if ctx.needs_input_grad[1] and not weight_gradients_disabled:
                grad_weight = Conv2dGradWeight.apply(grad_output, input)
            if ctx.needs_input_grad[2]:
                grad_bias = _ChannelSum.apply(grad_output)
            return grad_input, grad_weight, grad_bias

    class Conv2dGradWeight(Function):
        @staticmethod
        def forward(ctx, grad_output, input):
            grad_weight = _weight_grad(transpose, weight_shape, grad_output, input, stride, padding, dilation, groups)
            ctx.save_for_backward(grad_output, input)
            return grad_weight

        @staticmethod
        def backward(ctx, grad_grad_weight):
            grad_output, input = ctx.saved_tensors
            grad_grad_output = grad_grad_input = None
            if ctx.needs_input_grad[0]:
                grad_grad_output = Conv2d.apply(input, grad_grad_weight, None)
            if ctx.needs_input_grad[1]:
                grad_grad_input = transposed_op(input.shape, grad_output.shape).apply(grad_output, grad_grad_weight, None)
            return grad_grad_output, grad_grad_input

    _gradfix_cache[key] = Conv2d
    return Conv2d


def _needs_grad(*ts):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    s, p, d = _pair(stride), _pair(padding), _pair(dilation)
    if s[0] != s[1]:
        raise NotImplementedError("vtoonify_b200 conv2d: the stride must be the same on both axes")
    if _needs_grad(input, weight, bias):
        return _conv2d_gradfix(False, tuple(weight.shape), s, p, (0, 0), d, groups).apply(input, weight, bias)
    return _conv2d_forward(input, weight, bias, s, p, d, groups)


def conv_transpose2d(input, weight, bias=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
    if _pair(stride) != (2, 2) or _pair(padding) != (0, 0) or _pair(output_padding) != (0, 0) \
            or _pair(dilation) != (1, 1) or tuple(weight.shape[2:]) != (3, 3):
        raise NotImplementedError("vtoonify_b200 conv_transpose2d: only stride=2, padding=0, 3x3")
    if _needs_grad(input, weight, bias):
        return _conv2d_gradfix(True, tuple(weight.shape), (2, 2), (0, 0), (0, 0), (1, 1), groups).apply(input, weight, bias)
    return _conv_transpose2d_s2_k3_forward(input, weight, bias, groups)
