"""StyleGAN2 modules with the reference's constructor signatures, forward signatures and state_dict keys
(model/stylegan/model.py), running on the library's sm_90a kernels.

Differences in *how* (not what):
  * activations travel NHWC (channels_last); modules accept any NCHW tensor and return logical-NCHW
    channels_last views, so chained modules never transpose;
  * ``ModulatedConv2d`` never builds a grouped convolution: the per-sample modulated+demodulated weights
    (model.py:259-267) are written once in the GEMM's K-major layout and the convolution is one shared
    implicit GEMM over the batch (per-sample weight tile selected by the TMA coordinate);
  * ``StyledConv`` fuses noise + bias + leaky-relu into the conv epilogue (or into the FIR pass after the
    transposed conv); ``ToRGB`` fuses the 1x1 modulated conv, bias, skip ``Upsample`` and add in one kernel.
Forward-only (inference), CUDA only; the discriminator's ResBlock / ConvLayer(downsample=True) have gradients through
vtoonify_b200.discriminator.
"""
import math
import random

import torch
from torch import nn

from . import ops
from .op import FusedLeakyReLU, fused_leaky_relu, upfirdn2d, conv2d_gradfix  # noqa: F401
from ._lib import ACT_LRELU, ACT_NONE

_R2 = 1.0 / math.sqrt(2.0)


class PixelNorm(nn.Module):
    """model/stylegan/model.py:13-18: normalises over dim 1, for any rank >= 2 (the kernel normalises the last dim, so dim 1
    is moved last and back)."""

    def forward(self, input):
        if input.dim() <= 2:
            return ops.pixelnorm(input)
        return ops.pixelnorm(input.movedim(1, -1)).movedim(-1, 1)


def make_kernel(k):
    """model/stylegan/model.py:21-29: outer product of a 1-D FIR, normalised to sum 1."""
    k = torch.tensor(k, dtype=torch.float32)
    if k.ndim == 1:
        k = k[None, :] * k[:, None]
    k /= k.sum()
    return k


class Upsample(nn.Module):
    """model/stylegan/model.py:32-50"""

    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        kernel = make_kernel(kernel) * (factor ** 2)
        self.register_buffer("kernel", kernel)
        p = kernel.shape[0] - factor
        self.pad = ((p + 1) // 2 + factor - 1, p // 2)

    def forward(self, input):
        return upfirdn2d(input, self.kernel, up=self.factor, down=1, pad=self.pad)


class Downsample(nn.Module):
    """model/stylegan/model.py:53-71"""

    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        kernel = make_kernel(kernel)
        self.register_buffer("kernel", kernel)
        p = kernel.shape[0] - factor
        self.pad = ((p + 1) // 2, p // 2)

    def forward(self, input):
        return upfirdn2d(input, self.kernel, up=1, down=self.factor, pad=self.pad)


class Blur(nn.Module):
    """model/stylegan/model.py:74-90"""

    def __init__(self, kernel, pad, upsample_factor=1):
        super().__init__()
        kernel = make_kernel(kernel)
        if upsample_factor > 1:
            kernel = kernel * (upsample_factor ** 2)
        self.register_buffer("kernel", kernel)
        self.pad = pad

    def forward(self, input):
        return upfirdn2d(input, self.kernel, pad=self.pad)


class _PreppedWeight:
    """Cache of a plain conv weight in the kernels' [1, taps, Cout, cin_pad] layout, invalidated on in-place updates."""

    def __init__(self):
        self.key = None
        self.value = None

    def get(self, weight, scale, cin_pad, round_tf32=None):
        key = (weight.data_ptr(), weight._version, float(scale), cin_pad, ops.get_precision(), weight.device, round_tf32)
        if key != self.key:
            self.value = ops.prep_weights(weight.detach(), None, scale, False, cin_pad, round_tf32=round_tf32)
            self.key = key
        return self.value


def _conv_plain_nhwc(x, weight, wcache, scale, bias, stride, padding, dilation, act=ACT_NONE, slope=0.2, gain=1.0,
                     res=None, alpha=1.0, beta=1.0, src_affine=None, want_stats=False):
    """Shared body of EqualConv2d / Conv2d on an NHWC tensor.  ``want_stats``: returns ``(out, stats)`` with the instance-norm
    statistics of the output (ops.conv2d_nhwc)."""
    B, H, W, Cs = x.shape
    Cout, Cin, k, _ = weight.shape
    w = wcache.get(weight, scale, Cs)
    Ho = ops.conv_out_size(H, k, stride, padding, dilation)
    Wo = ops.conv_out_size(W, k, stride, padding, dilation)
    return ops.conv2d_nhwc([x], w, ops.conv_taps(k, padding, dilation), stride, Ho, Wo, bias=bias, act=act, slope=slope,
                           gain=gain, res=res, alpha=alpha, beta=beta,
                           src_affine=None if src_affine is None else [src_affine], want_stats=want_stats)


class EqualConv2d(nn.Module):
    """model/stylegan/model.py:93-130 (with the reference's added ``dilation``)."""

    def __init__(self, in_channel, out_channel, kernel_size, stride=1, padding=0, bias=True, dilation=1):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_channel, in_channel, kernel_size, kernel_size))
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.stride = stride
        self.padding = padding
        self.dilation = dilation
        self.bias = nn.Parameter(torch.zeros(out_channel)) if bias else None
        self._w = _PreppedWeight()
        self._wt = _PreppedWeight()          # transposed weight of the input gradient (encoder_grad)

    def forward_nhwc(self, x, **epi):
        return _conv_plain_nhwc(x, self.weight, self._w, self.scale, epi.pop("bias", self.bias), self.stride,
                                self.padding, self.dilation, **epi)

    def forward(self, input):
        C = input.shape[1]
        x = ops.to_nhwc(input, ops._pad32(C) if C % 32 else None)
        return ops.nhwc_as_nchw_view(self.forward_nhwc(x))

    def __repr__(self):
        return (f"{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]},"
                f" {self.weight.shape[2]}, stride={self.stride}, padding={self.padding}, dilation={self.dilation})")


class EqualLinear(nn.Module):
    """model/stylegan/model.py:133-167"""

    def __init__(self, in_dim, out_dim, bias=True, bias_init=0, lr_mul=1, activation=None):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_dim, in_dim).div_(lr_mul))
        self.bias = nn.Parameter(torch.zeros(out_dim).fill_(bias_init)) if bias else None
        self.activation = activation
        self.scale = (1 / math.sqrt(in_dim)) * lr_mul
        self.lr_mul = lr_mul

    def forward(self, input):
        return ops.linear(input, self.weight, self.bias, self.scale, self.lr_mul, 1 if self.activation else 0)

    def __repr__(self):
        return f"{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]})"


class ModulatedConv2d(nn.Module):
    """model/stylegan/model.py:170-306.  ``forward(input, style, externalweight=None)``."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, demodulate=True, upsample=False,
                 downsample=False, blur_kernel=[1, 3, 3, 1], fused=True):
        super().__init__()
        self.eps = 1e-8
        self.kernel_size = kernel_size
        self.in_channel = in_channel
        self.out_channel = out_channel
        self.upsample = upsample
        self.downsample = downsample
        if upsample:
            factor = 2
            p = (len(blur_kernel) - factor) - (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2 + factor - 1, p // 2 + 1), upsample_factor=factor)
        if downsample:
            factor = 2
            p = (len(blur_kernel) - factor) + (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2, p // 2))
        fan_in = in_channel * kernel_size ** 2
        self.scale = 1 / math.sqrt(fan_in)
        self.padding = kernel_size // 2
        self.weight = nn.Parameter(torch.randn(1, out_channel, in_channel, kernel_size, kernel_size))
        self.modulation = EqualLinear(style_dim, in_channel, bias_init=1)
        self.demodulate = demodulate
        self.fused = fused  # both reference branches compute the same function; kept for API parity

    def __repr__(self):
        return (f"{self.__class__.__name__}({self.in_channel}, {self.out_channel}, {self.kernel_size}, "
                f"upsample={self.upsample}, downsample={self.downsample})")

    def modulated_weights(self, style, cin_pad, externalweight=None, round_tf32=None, folded=False):
        """[B, k*k, Cout, cin_pad] = scale * (W [+ ext]) * s[b] * demod[b]  (model.py:259-267); ``folded``: the up-conv's
        [B, 9, 4*Cout, cin_pad] phase kernels (Blur o conv_transpose).  Inside a style scope the result (and its bf16 split,
        which is attached to the tensor) is computed once per style."""
        def make():
            s = self.modulation(style)
            W = self.weight[0] if externalweight is None else (self.weight + externalweight)[0]
            w = ops.prep_weights(W.detach(), s, self.scale, self.demodulate, cin_pad, round_tf32=round_tf32)
            return ops.fold_upconv_weights(w, self.blur.kernel) if folded else w
        if externalweight is not None:
            return make()
        return ops.style_cached(self, "w", make, extra=(cin_pad, round_tf32, folded, self.weight._version, self.weight.data_ptr(),
                                                            self.modulation.weight._version, self.modulation.bias._version))

    def forward_nhwc(self, x, style, externalweight=None, bias=None, noise=None, noise_w=None, act=False,
                     slope=0.2, gain=ops.SQRT2, rgb=None, want_stats=False):
        """x NHWC -> NHWC.  Optional fused StyledConv epilogue (noise, bias, leaky relu) and fused ToRGB tail
        (``rgb`` dict, plain 3x3 form only: returns ``(out, rgb_image)``).  ``want_stats``: returns ``(out, instance-norm
        statistics of out)``; the plain form takes them from the convolution's epilogue, the resampling forms from a separate
        statistics pass."""
        if want_stats and (self.upsample or self.downsample):
            out = self.forward_nhwc(x, style, externalweight, bias, noise, noise_w, act, slope, gain)
            return out, ops.instnorm_stats(out)
        B, H, W, Cs = x.shape
        k = self.kernel_size
        a = ACT_LRELU if act else ACT_NONE
        if self.upsample:
            if k != 3:
                raise NotImplementedError("upsampling ModulatedConv2d is 3x3 in StyleGAN2")
            if externalweight is None and Cs == self.in_channel and ops.rsu_eligible(self.in_channel, self.out_channel, W, self.blur.kernel, self.blur.pad):
                w9 = self.modulated_weights(style, Cs, None, round_tf32=False)
                return ops.conv_up2_rs_nhwc(x, w9, self.blur.kernel, bias=bias, noise=noise, noise_w=noise_w, act=a, slope=slope, gain=gain)
            if tuple(self.blur.kernel.shape) == (4, 4) and tuple(self.blur.pad) == (1, 1) and ops.use_folded_upconv(self.in_channel):
                # Blur o conv_transpose folded into 4 phase-specific 3x3 kernels: one launch, no intermediate tensor
                wf = self.modulated_weights(style, Cs, externalweight, round_tf32=False, folded=True)
                return ops.conv_up2_folded_nhwc(x, wf, bias=bias, noise=noise, noise_w=noise_w, act=a, slope=slope, gain=gain)
            w = self.modulated_weights(style, Cs, externalweight)
            t = ops.conv_transpose2d_s2_k3_nhwc(x, w)
            return ops.fir_nhwc(t, self.blur.kernel, self.blur.pad, bias=bias, noise=noise, noise_w=noise_w, act=act,
                                slope=slope, gain=gain)
        w = self.modulated_weights(style, Cs, externalweight)
        if self.downsample:
            xb = ops.fir_nhwc(x, self.blur.kernel, self.blur.pad)
            Ho = ops.conv_out_size(xb.shape[1], k, 2, 0, 1)
            Wo = ops.conv_out_size(xb.shape[2], k, 2, 0, 1)
            return ops.conv2d_nhwc([xb], w, ops.conv_taps(k, 0), 2, Ho, Wo, bias=bias, noise=noise, noise_w=noise_w,
                                   act=a, slope=slope, gain=gain)
        return ops.conv2d_nhwc([x], w, ops.conv_taps(k, self.padding), 1, H, W, bias=bias, noise=noise,
                               noise_w=noise_w, act=a, slope=slope, gain=gain, rgb=rgb, want_stats=want_stats)

    def forward(self, input, style, externalweight=None):
        C = input.shape[1]
        x = ops.to_nhwc(input, ops._pad32(C) if C % 32 else None)
        if self.out_channel <= 4 and self.kernel_size == 1 and not (self.upsample or self.downsample):
            w = self.modulated_weights(style, x.shape[3], externalweight, round_tf32=False)
            B, H, W, _ = x.shape
            return ops.smalln_conv(x, w, [(0, 0, 0)], self.out_channel, B, H, W)
        return ops.nhwc_as_nchw_view(self.forward_nhwc(x, style, externalweight))


class NoiseInjection(nn.Module):
    """model/stylegan/model.py:309-320"""

    def __init__(self):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(1))

    def forward(self, image, noise=None):
        if noise is None:
            batch, _, height, width = image.shape
            noise = image.new_empty(batch, 1, height, width).normal_()
        # standalone use only (StyledConv fuses this into the conv epilogue)
        return image + self.weight * noise


class ConstantInput(nn.Module):
    """model/stylegan/model.py:323-333"""

    def __init__(self, channel, size=4):
        super().__init__()
        self.input = nn.Parameter(torch.randn(1, channel, size, size))

    def forward(self, input):
        return self.input.repeat(input.shape[0], 1, 1, 1)


def _planar_noise(noise, B, H, W):
    if noise.shape[-2:] != (H, W):
        raise ValueError(f"noise spatial size {tuple(noise.shape[-2:])} does not match output {(H, W)}")
    if noise.shape[0] != B:
        noise = noise.expand(B, *noise.shape[1:])
    return noise.contiguous()


class StyledConv(nn.Module):
    """model/stylegan/model.py:336-370.  ``forward(input, style, noise=None, externalweight=None)``."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, upsample=False, blur_kernel=[1, 3, 3, 1],
                 demodulate=True):
        super().__init__()
        self.conv = ModulatedConv2d(in_channel, out_channel, kernel_size, style_dim, upsample=upsample,
                                    blur_kernel=blur_kernel, demodulate=demodulate)
        self.noise = NoiseInjection()
        self.activate = FusedLeakyReLU(out_channel)

    def forward_nhwc(self, x, style, noise=None, externalweight=None, zero_noise=False, to_rgb=None, rgb_only=False,
                     want_stats=False):
        """``to_rgb`` = (ToRGB module, its style, skip image or None): also returns the RGB image, computed in this
        conv's epilogue when possible (the activation is then never re-read for the 1x1 ToRGB conv).  ``rgb_only``: the
        caller drops the activation (last layer of the synthesis network): the returned ``out`` may be ``None`` and a fused
        launch does not write it to HBM at all.  ``want_stats`` (without ``to_rgb``): returns ``(out, instance-norm
        statistics of out)`` for an AdaIN consumer (ModulatedConv2d.forward_nhwc)."""
        B, H, W, _ = x.shape
        Ho, Wo = (2 * H, 2 * W) if self.conv.upsample else (H, W)
        if zero_noise:
            noise = None  # VToonify feeds an all-zero noise tensor (model/vtoonify.py:266-270): exact no-op
        else:
            if noise is None:
                noise = torch.empty((B, 1, Ho, Wo), device=x.device, dtype=torch.float32).normal_()
            noise = _planar_noise(noise, B, Ho, Wo)
        kw = dict(bias=self.activate.bias, noise=noise, noise_w=None if noise is None else self.noise.weight, act=True,
                  slope=self.activate.negative_slope, gain=self.activate.scale)
        if to_rgb is None:
            return self.conv.forward_nhwc(x, style, externalweight, want_stats=want_stats, **kw)
        if want_stats:
            raise ValueError("StyledConv.forward_nhwc: want_stats and to_rgb are exclusive")
        trgb, style_rgb, skip = to_rgb
        Cout = self.conv.out_channel
        fuse = (ops.rgb_fusable(Cout) and not self.conv.upsample and not self.conv.downsample and trgb.fusable_skip(skip, H, W))
        if not fuse:
            out = self.conv.forward_nhwc(x, style, externalweight, **kw)
            return out, trgb.forward_nhwc(out, style_rgb, skip)
        w_rgb = trgb.conv.modulated_weights(style_rgb, Cout, round_tf32=False)      # [B, 1, 3, Cout]
        rgb = {"w": w_rgb, "bias": trgb.bias.view(3), "skip": skip,
               "kernel": trgb.upsample.kernel if skip is not None else None, "only": rgb_only}
        return self.conv.forward_nhwc(x, style, externalweight, rgb=rgb, **kw)

    def forward(self, input, style, noise=None, externalweight=None):
        C = input.shape[1]
        x = ops.to_nhwc(input, ops._pad32(C) if C % 32 else None)
        return ops.nhwc_as_nchw_view(self.forward_nhwc(x, style, noise, externalweight))


class ToRGB(nn.Module):
    """model/stylegan/model.py:373-392.  ``forward(input, style, skip=None, externalweight=None)``."""

    def __init__(self, in_channel, style_dim, upsample=True, blur_kernel=[1, 3, 3, 1]):
        super().__init__()
        if upsample:
            self.upsample = Upsample(blur_kernel)
        self.conv = ModulatedConv2d(in_channel, 3, 1, style_dim, demodulate=False)
        self.bias = nn.Parameter(torch.zeros(1, 3, 1, 1))

    def fusable_skip(self, skip, H, W):
        """True if ``upfirdn2d(skip)`` is the standard up=2 / 4x4 / pad (2,1) form the fused kernels implement."""
        return skip is None or (hasattr(self, "upsample") and self.upsample.factor == 2
                                and tuple(self.upsample.kernel.shape) == (4, 4) and tuple(self.upsample.pad) == (2, 1)
                                and skip.shape[2] * 2 == H and skip.shape[3] * 2 == W)

    def forward_nhwc(self, x, style, skip=None, externalweight=None):
        """x NHWC -> planar NCHW [B,3,H,W] (+ fused skip upsample/add)."""
        B, H, W, Cs = x.shape
        w = self.conv.modulated_weights(style, Cs, externalweight, round_tf32=False)   # CUDA-core kernel: keep fp32
        fuse = skip is not None and self.fusable_skip(skip, H, W)
        out = ops.smalln_conv(x, w, [(0, 0, 0)], 3, B, H, W, bias=self.bias.view(3),
                              skip=skip if fuse else None, skip_kernel=self.upsample.kernel if fuse else None)
        if skip is not None and not fuse:
            out = ops.axpby(out, self.upsample(skip), 1.0, 1.0, round_tf32=False)
        return out

    def forward(self, input, style, skip=None, externalweight=None):
        C = input.shape[1]
        x = ops.to_nhwc(input, ops._pad32(C) if C % 32 else None)
        return self.forward_nhwc(x, style, skip, externalweight)


class Generator(ops.WeightsEpochMixin, nn.Module):
    """model/stylegan/model.py:395-590 — same constructor, attributes and ``forward`` keyword interface."""

    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=[1, 3, 3, 1], lr_mlp=0.01):
        super().__init__()
        self.size = size
        self.style_dim = style_dim
        layers = [PixelNorm()]
        for _ in range(n_mlp):
            layers.append(EqualLinear(style_dim, style_dim, lr_mul=lr_mlp, activation="fused_lrelu"))
        self.style = nn.Sequential(*layers)
        self.channels = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * channel_multiplier,
                         128: 128 * channel_multiplier, 256: 64 * channel_multiplier,
                         512: 32 * channel_multiplier, 1024: 16 * channel_multiplier}
        self.input = ConstantInput(self.channels[4])
        self.conv1 = StyledConv(self.channels[4], self.channels[4], 3, style_dim, blur_kernel=blur_kernel)
        self.to_rgb1 = ToRGB(self.channels[4], style_dim, upsample=False)
        self.log_size = int(math.log(size, 2))
        self.num_layers = (self.log_size - 2) * 2 + 1
        self.convs = nn.ModuleList()
        self.upsamples = nn.ModuleList()
        self.to_rgbs = nn.ModuleList()
        self.noises = nn.Module()
        in_channel = self.channels[4]
        for layer_idx in range(self.num_layers):
            res = (layer_idx + 5) // 2
            self.noises.register_buffer(f"noise_{layer_idx}", torch.randn(1, 1, 2 ** res, 2 ** res))
        for i in range(3, self.log_size + 1):
            out_channel = self.channels[2 ** i]
            self.convs.append(StyledConv(in_channel, out_channel, 3, style_dim, upsample=True, blur_kernel=blur_kernel))
            self.convs.append(StyledConv(out_channel, out_channel, 3, style_dim, blur_kernel=blur_kernel))
            self.to_rgbs.append(ToRGB(out_channel, style_dim))
            in_channel = out_channel
        self.n_latent = self.log_size * 2 - 2

    def make_noise(self):
        device = self.input.input.device
        noises = [torch.randn(1, 1, 4, 4, device=device)]
        for i in range(3, self.log_size + 1):
            for _ in range(2):
                noises.append(torch.randn(1, 1, 2 ** i, 2 ** i, device=device))
        return noises

    def mean_latent(self, n_latent):
        latent_in = torch.randn(n_latent, self.style_dim, device=self.input.input.device)
        return self.style(latent_in).mean(0, keepdim=True)

    def get_latent(self, input):
        return self.style(input)

    def _latent(self, styles, inject_index):
        """Build the [B, n_latent, 512] W+ code from one or two style tensors (model.py:547-565)."""
        def widen(s, n):
            return s.unsqueeze(1).repeat(1, n, 1) if s.ndim < 3 else s
        if len(styles) < 2:
            return widen(styles[0], self.n_latent)
        if inject_index is None:
            inject_index = random.randint(1, self.n_latent - 1)
        if styles[0].ndim < 3:
            return torch.cat([widen(styles[0], inject_index), widen(styles[1], self.n_latent - inject_index)], 1)
        return torch.cat([styles[0][:, :inject_index], styles[1][:, inject_index:]], 1)

    def _prepare(self, styles, inject_index, truncation, truncation_latent, input_is_latent, noise, randomize_noise,
                 z_plus_latent):
        """Head of ``forward`` (model.py:517-565): mapping network, noise list, truncation, W+ code -> ``(latent, noise,
        cacheable)``.  ``cacheable``: the latent is the caller's own tensor and nothing else shapes it (single style input
        already in W+, no truncation / mixing), so per-latent caching keyed on that tensor object is valid."""
        if not input_is_latent:
            if not z_plus_latent:
                styles = [self.style(s) for s in styles]
            else:
                styles = [self.style(s.reshape(-1, s.shape[-1])).reshape(s.shape) for s in styles]
        if noise is None:
            if randomize_noise:
                noise = [None] * self.num_layers
            else:
                noise = [getattr(self.noises, f"noise_{i}") for i in range(self.num_layers)]
        if truncation < 1:
            styles = [truncation_latent + truncation * (s - truncation_latent) for s in styles]
        latent = self._latent(styles, inject_index)
        cacheable = len(styles) == 1 and input_is_latent and truncation >= 1 and latent is styles[0]
        return latent, noise, cacheable

    def forward(self, styles, return_latents=False, inject_index=None, truncation=1, truncation_latent=None,
                input_is_latent=False, noise=None, randomize_noise=True, z_plus_latent=False,
                return_feature_ind=999):
        latent, noise, cacheable = self._prepare(styles, inject_index, truncation, truncation_latent, input_is_latent, noise,
                                                 randomize_noise, z_plus_latent)
        # per-latent caching of the modulated weights: valid while the caller passes the same (unmodified) tensor object again
        token = ops.style_token(self, latent)[0] if cacheable else None
        with ops.style_scope(token):
            return self._synthesis(latent, noise, return_latents, return_feature_ind)

    def _synthesis(self, latent, noise, return_latents, return_feature_ind):
        out = ops.to_nhwc(self.input(latent))
        out = self.conv1.forward_nhwc(out, latent[:, 0], noise=noise[0])
        skip = self.to_rgb1.forward_nhwc(out, latent[:, 1])
        i = 1
        n_levels = len(self.to_rgbs)
        for lvl, (conv1, conv2, noise1, noise2, to_rgb) in enumerate(zip(self.convs[::2], self.convs[1::2], noise[1::2], noise[2::2],
                                                                         self.to_rgbs)):
            out = conv1.forward_nhwc(out, latent[:, i], noise=noise1)
            last = lvl == n_levels - 1 and i + 2 <= return_feature_ind     # nobody reads the last activation (model.py:549-556)
            out, skip = conv2.forward_nhwc(out, latent[:, i + 1], noise=noise2, to_rgb=(to_rgb, latent[:, i + 2], skip), rgb_only=last)
            i += 2
            if i > return_feature_ind:
                return ops.nhwc_as_nchw_view(out), skip
        image = skip
        if return_latents:
            return image, latent
        return image, None


class ConvLayer(nn.Sequential):
    """model/stylegan/model.py:593-637: [Blur] + EqualConv2d + [FusedLeakyReLU]; keys ``0.weight`` / ``1.bias``."""

    def __init__(self, in_channel, out_channel, kernel_size, downsample=False, blur_kernel=[1, 3, 3, 1], bias=True,
                 activate=True, dilation=1):
        layers = []
        if downsample:
            factor = 2
            p = (len(blur_kernel) - factor) + (kernel_size - 1)
            layers.append(Blur(blur_kernel, pad=((p + 1) // 2, p // 2)))
            stride = 2
            self.padding = 0
        else:
            stride = 1
            self.padding = kernel_size // 2 + dilation - 1
        layers.append(EqualConv2d(in_channel, out_channel, kernel_size, padding=self.padding, stride=stride,
                                  bias=bias and not activate, dilation=dilation))
        if activate:
            layers.append(FusedLeakyReLU(out_channel, bias=bias))
        super().__init__(*layers)

    def forward_nhwc(self, x, res=None, alpha=1.0, beta=1.0, src_affine=None, want_stats=False, blurred=None):
        """Fused conv + FusedLeakyReLU (+ ``v*alpha + beta*res``); ``src_affine``: AdaIN table applied to the input inside the
        convolution; ``want_stats``: ``(out, instance-norm statistics of out)`` (non-downsampling form).

        The downsampling form (discriminator) is a stride-2 convolution on ``blurred`` = ``blur_pad2(x)`` (computed here when not
        given): the 4x4 Blur with pad (2, 2), ``[B, H+1, W+1, C]``.  The reference's blur pad (p0, p1) with p0 <= 2 reads that tensor
        shifted by 2 - p0 (the 1x1 skip's pad (1, 1) blur is its tap (1, 1)), so one blur serves every downsampling layer on x."""
        mods = list(self)
        if isinstance(mods[0], Blur):
            if src_affine is not None or want_stats:
                raise NotImplementedError("ConvLayer(downsample=True): no src_affine / want_stats")
            conv = mods[1]
            k, (p0, p1) = conv.weight.shape[2], mods[0].pad
            if tuple(mods[0].kernel.shape) != (4, 4) or p0 > 2:
                raise NotImplementedError("ConvLayer(downsample=True) supports the 4-tap blur kernel")
            xb = blur_pad2(x, mods[0].kernel) if blurred is None else blurred
            B, H, W, _ = x.shape
            Ho = (H + p0 + p1 - 3 - k) // 2 + 1
            Wo = (W + p0 + p1 - 3 - k) // 2 + 1
            off = 2 - p0
            taps = [(ky + off, kx + off, ky * k + kx) for ky in range(k) for kx in range(k)]
            w = conv._w.get(conv.weight, conv.scale, xb.shape[3])
            epi = dict(act=ACT_LRELU, bias=mods[2].bias, slope=mods[2].negative_slope, gain=mods[2].scale) if len(mods) > 2 else {}
            return ops.conv2d_nhwc([xb], w, taps, 2, Ho, Wo, res=res, alpha=alpha, beta=beta, **epi)
        conv = mods[0]
        if len(mods) > 1:
            act = mods[1]
            return conv.forward_nhwc(x, bias=act.bias, act=ACT_LRELU, slope=act.negative_slope, gain=act.scale,
                                     res=res, alpha=alpha, beta=beta, src_affine=src_affine, want_stats=want_stats)
        return conv.forward_nhwc(x, res=res, alpha=alpha, beta=beta, src_affine=src_affine, want_stats=want_stats)


def blur_pad2(x, kernel):
    """``Blur(kernel, pad=(2, 2))`` of NHWC ``x``: ``[B, H+1, W+1, C]``, the input of every downsampling ConvLayer."""
    return ops.fir_nhwc(x, kernel, (2, 2))


class ResBlock(nn.Module):
    """model/stylegan/model.py:640-658: ``(conv2(conv1(x)) + skip(x)) / sqrt(2)``, both halves downsampling by 2.

    NHWC: conv1 with bias + FusedLeakyReLU in its epilogue; conv2 (3x3, stride 2) on the pad (2, 2) blur of conv1's output with its
    bias + FusedLeakyReLU; the skip (1x1, stride 2, tap (1, 1)) on the pad (2, 2) blur of x, whose epilogue adds conv2's output:
    ``(a2 + skip) / sqrt(2)`` with ``alpha = beta = 1/sqrt(2)``, so the block output costs no extra pass and ``a2`` (the gate's
    reference in the backward) is kept."""

    def __init__(self, in_channel, out_channel, blur_kernel=[1, 3, 3, 1]):
        super().__init__()
        self.conv1 = ConvLayer(in_channel, in_channel, 3)
        self.conv2 = ConvLayer(in_channel, out_channel, 3, downsample=True, blur_kernel=blur_kernel)
        self.skip = ConvLayer(in_channel, out_channel, 1, downsample=True, activate=False, bias=False, blur_kernel=blur_kernel)

    def forward_nhwc(self, x, rec=None):
        """NHWC ``x`` -> NHWC block output; ``rec`` (a list): appends what the backward reads."""
        a1 = self.conv1.forward_nhwc(x)
        a1b = blur_pad2(a1, self.conv2[0].kernel)
        a2 = self.conv2.forward_nhwc(a1, blurred=a1b)
        xb = blur_pad2(x, self.skip[0].kernel)
        out = self.skip.forward_nhwc(x, blurred=xb, res=a2, alpha=_R2, beta=_R2)
        if rec is not None:
            rec.append((self, x, a1, a1b, a2, xb))
        return out

    def forward(self, input):
        C = input.shape[1]
        x = ops.to_nhwc(input, ops._pad32(C) if C % 32 else None)
        return ops.nhwc_as_nchw_view(self.forward_nhwc(x))
