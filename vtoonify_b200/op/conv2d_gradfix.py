"""``conv2d_gradfix.conv2d`` / ``conv_transpose2d`` — same call signatures as model/stylegan/op/conv2d_gradfix.py:22-75.
In the reference these forward to cuDNN (F.conv2d / F.conv_transpose2d) on any modern torch; here they run the
library's NHWC convolution kernels (wgmma when shapes allow, fp32 FFMA otherwise).  Forward only.

Supported
  * ``conv2d``: kernels of up to 36 taps (any kh x kw), per-axis padding / dilation, stride s (same on both axes),
    ``groups == 1`` or the form ``ModulatedConv2d`` uses (model/stylegan/model.py:291-301): ``input [1, G*Cin, H, W]``,
    ``weight [G*Cout, Cin, kh, kw]``, ``groups = G`` — the groups are the samples of the batch, so the call is the same
    implicit GEMM with per-sample weight tiles (``wB = G``, selected by the TMA batch coordinate), not a grouped conv.
  * ``conv_transpose2d``: stride 2, padding 0, 3x3 (the only form the reference uses, model.py:236-238, 281-283), with
    ``groups == 1`` or ``groups = G`` as above (``weight [G*Cin, Cout, 3, 3]``).
Everything else raises ``NotImplementedError`` (never a silently wrong shape).  Inputs / outputs are planar NCHW like
``F.conv2d``'s (a channels_last view is returned when the layout allows it without a copy)."""
import contextlib

import torch

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


def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    s, p, d = _pair(stride), _pair(padding), _pair(dilation)
    if s[0] != s[1]:
        raise NotImplementedError("vtoonify_b200 conv2d: the stride must be the same on both axes")
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


def conv_transpose2d(input, weight, bias=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
    if _pair(stride) != (2, 2) or _pair(padding) != (0, 0) or _pair(output_padding) != (0, 0) \
            or _pair(dilation) != (1, 1) or tuple(weight.shape[2:]) != (3, 3):
        raise NotImplementedError("vtoonify_b200 conv_transpose2d: only stride=2, padding=0, 3x3")
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
