"""VToonify (model/vtoonify.py:92-286) — same constructor, ``forward(x, style, d_s=None, return_mask=False,
return_feat=False)``, ``stylegan()``, ``zplus2wplus()`` and state_dict keys, on the library's sm_90a kernels.

The forward keeps every activation NHWC and issues, per layer, one wgmma implicit-GEMM convolution with the layer's
elementwise tail fused in the epilogue:
  encoder convs            bias + LeakyReLU(0.2)                       (model/vtoonify.py:160-176)
  VToonifyResBlock         conv2: bias + LeakyReLU, (out + x)/sqrt(2)   (:92-104)
  AdaResBlock (dilated)    AdaIN -> conv(+FusedLeakyReLU) x2, *d_s + skip
  Fusion (D)               stats of cat(f_G,|f_G-f_E|) without materialising the concat; the mask conv (2C->1) also
                           writes f_E*m_E; the fusion conv reads (f_G, f_E*m_E) as a virtual concat (two TMA sources)
  StyledConv / ToRGB       see stylegan.py; the all-zero noise of :266-270 is elided (exact no-op)
"""
import math

import numpy as np
import torch
from torch import nn

from . import discriminator, encoder_grad, ops, vtoonify_grad
from ._lib import ACT_LRELU, ACT_NONE, ACT_RELU_TANH
from .dualstylegan import AdaptiveInstanceNorm, AdaResBlock, DualStyleGAN, Linear
from .stylegan import ConvLayer, EqualLinear, Generator, ResBlock, _PreppedWeight


class ConditionalDiscriminator(nn.Module):
    """model/vtoonify.py:10-89 — same constructor, ``forward(input, degree_label=None, style_ind=None)``, return value and
    state_dict keys.  The convolutional trunk, the minibatch standard deviation and ``final_linear`` run NHWC on the library's
    kernels, with gradients into ``input`` and every parameter of ``convs``, ``final_conv`` and ``final_linear``
    (vtoonify_b200.discriminator); ``label_mapper``, ``style_mapper`` and the conditioning product are ordinary torch modules."""

    def __init__(self, size, channel_multiplier=2, blur_kernel=[1, 3, 3, 1], use_condition=False, style_num=None):
        super().__init__()
        channels = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * channel_multiplier, 128: 128 * channel_multiplier,
                    256: 64 * channel_multiplier, 512: 32 * channel_multiplier, 1024: 16 * channel_multiplier}
        convs = [ConvLayer(3, channels[size], 1)]
        log_size = int(math.log(size, 2))
        in_channel = channels[size]
        for i in range(log_size, 2, -1):
            out_channel = channels[2 ** (i - 1)]
            convs.append(ResBlock(in_channel, out_channel, blur_kernel))
            in_channel = out_channel
        self.convs = nn.Sequential(*convs)
        self.stddev_group = 4
        self.stddev_feat = 1
        self.use_condition = use_condition
        if self.use_condition:
            self.condition_dim = 128
            self.label_mapper = nn.Sequential(
                nn.Linear(1, 64),
                nn.LeakyReLU(negative_slope=0.2, inplace=True),
                nn.Linear(64, 64),
                nn.LeakyReLU(negative_slope=0.2, inplace=True),
                nn.Linear(64, self.condition_dim // 2),
            )
            self.style_mapper = nn.Embedding(style_num, self.condition_dim - self.condition_dim // 2)
        else:
            self.condition_dim = 1
        self.final_conv = ConvLayer(in_channel + 1, channels[4], 3)
        self.final_linear = nn.Sequential(
            EqualLinear(channels[4] * 4 * 4, channels[4], activation="fused_lrelu"),
            EqualLinear(channels[4], self.condition_dim),
        )

    def forward(self, input, degree_label=None, style_ind=None):
        h = discriminator.final_linear_out(self, input)
        if self.use_condition:
            condition = torch.cat((self.label_mapper(degree_label), self.style_mapper(style_ind)), dim=1)
            return (h * condition).sum(dim=1, keepdim=True) * (1 / np.sqrt(self.condition_dim))
        return h


class Conv2d(nn.Module):
    """nn.Conv2d replacement (keys ``weight`` [Cout,Cin,k,k], ``bias``; PyTorch default init)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, bias=True):
        super().__init__()
        self.stride, self.padding, self.kernel_size = stride, padding, kernel_size
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels, kernel_size, kernel_size))
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if bias:
            bound = 1 / math.sqrt(in_channels * kernel_size ** 2)
            self.bias = nn.Parameter(torch.empty(out_channels).uniform_(-bound, bound))
        else:
            self.bias = None
        self._w = _PreppedWeight()
        self._wp = _PreppedWeight()
        self._wt = _PreppedWeight()          # transposed weight of the input gradient (encoder_grad)

    def forward_nhwc(self, x, act=ACT_NONE, slope=0.2, gain=1.0, res=None, alpha=1.0, beta=1.0, x2=None, x2_scale=None,
                     want_stats=False):
        """x (and optional second concat source x2, optionally multiplied per pixel by the planar map x2_scale) NHWC -> NHWC;
        ``want_stats``: ``(out, instance-norm statistics of out)`` (ops.conv2d_nhwc)."""
        B, H, W, Cs = x.shape
        k = self.kernel_size
        cin = Cs + (0 if x2 is None else x2.shape[3])
        w = self._w.get(self.weight, 1.0, cin)
        Ho = ops.conv_out_size(H, k, self.stride, self.padding, 1)
        Wo = ops.conv_out_size(W, k, self.stride, self.padding, 1)
        srcs = [x] if x2 is None else [x, x2]
        return ops.conv2d_nhwc(srcs, w, ops.conv_taps(k, self.padding), self.stride, Ho, Wo, bias=self.bias, act=act,
                               slope=slope, gain=gain, res=res, alpha=alpha, beta=beta,
                               src_scale=None if x2_scale is None else [None, x2_scale], want_stats=want_stats)

    def forward_smalln(self, x, planar=None, act=ACT_NONE, mul_src=None, src_mask=None):
        """Cout <= 4 form: input channels = [planar (NCHW, first) | x (NHWC)] -> planar NCHW output."""
        B, H, W, Cs = x.shape
        k = self.kernel_size
        npl = 0 if planar is None else planar.shape[1]
        key = (self.weight.data_ptr(), self.weight._version, npl)
        if getattr(self, "_split_key", None) != key:
            wt = self.weight.detach()
            self._w_nhwc_part = wt[:, npl:].contiguous()
            self._w_planar = wt[:, :npl].permute(2, 3, 0, 1).reshape(k * k, wt.shape[0], npl).contiguous() if npl else None
            self._split_key = key
        w = self._wp.get(self._w_nhwc_part, 1.0, Cs, round_tf32=False)
        n_out = self.weight.shape[0]
        if (ops.scale_fusable() and ops.get_option("smalln_via_tc") and k == 3 and 9 * n_out <= 32 and Cs % 32 == 0
                and act == ACT_NONE and mul_src is None):
            # The 9*n_out per-tap dot products of every pixel are a [pixels x C] . [C x 32] GEMM: run it as a 1x1 convolution on
            # the tensor cores (each input read once, at HBM speed), then sum the 9 shifted partial products per output pixel.
            wkey = (w.data_ptr(), w._version)
            if getattr(self, "_wT_key", None) != wkey:
                wT = torch.zeros((1, 1, 32, w.shape[3]), device=w.device, dtype=torch.float32)
                wT[0, 0, :9 * n_out] = w.reshape(9 * n_out, w.shape[3])
                self._wT, self._wT_key = wT, wkey
            T = ops.conv2d_nhwc([x], self._wT, [(0, 0, 0)], 1, H, W, src_scale=None if src_mask is None else [src_mask])
            return ops.smalln_conv(None, None, ops.conv_taps(k, self.padding), n_out, B, H, W, planar=planar,
                                   planar_weight=self._w_planar, bias=self.bias, tsum=T)
        return ops.smalln_conv(x, w, ops.conv_taps(k, self.padding), self.weight.shape[0], B, H, W, planar=planar,
                               planar_weight=self._w_planar, bias=self.bias, act=act, mul_src=mul_src, src_mask=src_mask)

    def forward(self, input):
        C = input.shape[1]
        x = ops.to_nhwc(input, ops._pad32(C) if C % 32 else None)
        if self.weight.shape[0] <= 4:
            if self.stride == 1 and 2 * self.padding == self.kernel_size - 1:
                return self.forward_smalln(x)            # planar head: 'same' geometry only
            from .op import conv2d_gradfix               # any other geometry: generic entry point (FFMA kernel)
            return conv2d_gradfix.conv2d(input, self.weight, self.bias, stride=self.stride, padding=self.padding)
        return ops.nhwc_as_nchw_view(self.forward_nhwc(x))


class LeakyReLU(nn.Module):
    """Placeholder keeping nn.Sequential indices (``encoder.N.{0,2}``); fused into the preceding conv on the fast path."""

    def __init__(self, negative_slope=0.2, inplace=True):
        super().__init__()
        self.negative_slope = negative_slope

    def forward(self, input):
        return ops.fused_bias_act(input, None, self.negative_slope, 1.0)


class _ConvBlock(nn.Sequential):
    """Sequential(Conv2d, LeakyReLU, Conv2d, LeakyReLU) with a fused NHWC path."""

    def forward_nhwc(self, x):
        mods = list(self)
        i = 0
        while i < len(mods):
            conv = mods[i]
            fused = i + 1 < len(mods) and isinstance(mods[i + 1], LeakyReLU)
            x = conv.forward_nhwc(x, act=ACT_LRELU if fused else ACT_NONE,
                                  slope=mods[i + 1].negative_slope if fused else 0.2, gain=1.0)
            i += 2 if fused else 1
        return x


class VToonifyResBlock(nn.Module):
    """model/vtoonify.py:92-104"""

    def __init__(self, fin):
        super().__init__()
        self.conv = Conv2d(fin, fin, 3, 1, 1)
        self.conv2 = Conv2d(fin, fin, 3, 1, 1)
        self.lrelu = LeakyReLU(negative_slope=0.2, inplace=True)

    def forward_nhwc(self, x, want_stats=False):
        """``want_stats``: ``(out, instance-norm statistics of out)`` for an AdaIN consumer (the dilated ModRes block that follows
        every encoder res block in VToonify-D, model/vtoonify.py:239)."""
        out = self.conv.forward_nhwc(x, act=ACT_LRELU, slope=0.2, gain=1.0)
        r = 1.0 / math.sqrt(2)
        return self.conv2.forward_nhwc(out, act=ACT_LRELU, slope=0.2, gain=1.0, res=x, alpha=r, beta=r, want_stats=want_stats)

    def forward(self, x):
        return ops.nhwc_as_nchw_view(self.forward_nhwc(ops.to_nhwc(x)))


class Fusion(nn.Module):
    """model/vtoonify.py:106-128"""

    def __init__(self, in_channels, skip_channels, out_channels):
        super().__init__()
        self.conv = Conv2d(in_channels + skip_channels, out_channels, 3, 1, 1, bias=True)
        self.norm = AdaptiveInstanceNorm(in_channels + skip_channels, 128)
        self.conv2 = Conv2d(in_channels + skip_channels, 1, 3, 1, 1, bias=True)
        # same indices / keys as the reference's Sequential(Linear, LeakyReLU, Linear, LeakyReLU); calling ``self.linear(x)``
        # applies each LeakyReLU once, the fast path below fuses them into the Linear launches (act=2)
        self.linear = nn.Sequential(Linear(1, 64), LeakyReLU(0.2), Linear(64, 128), LeakyReLU(0.2))

    def forward_nhwc(self, f_G, f_E, d_s=1, rec=None):
        """``rec`` (a dict): take the route that writes ``f_E * m_E`` and keep the statistics and gamma|beta rows of the AdaIN for the
        backward (vtoonify_grad)."""
        B = f_G.shape[0]

        def make_gb():   # depends on d_s only: once per (style, d_s) scope
            label = torch.full((B, 1), float(d_s), device=f_G.device, dtype=torch.float32)
            label = self.linear[2](self.linear[0](label, act=2), act=2)   # LeakyReLU(0.2) fused into the Linear launches
            return self.norm.style(label)
        gb = ops.style_cached(self, "gb", make_gb, extra=(B, float(d_s)) + tuple(p._version for p in self.parameters()))
        # AdaIN(cat(f_G, |f_G - f_E|)) is never materialised: plane statistics in one pass over (f_G, f_E), the affine
        # folded into per-sample mask-conv weights, and the mask conv reads f_G / f_E directly (virtual concat)
        stats = ops.instnorm_stats(f_G, f_E)
        C2 = 2 * f_G.shape[3]
        w_plain = self.conv2._wp.get(self.conv2.weight, 1.0, C2, round_tf32=False)          # [1, 9, 1, 2C]
        w_fold, k_fold = ops.affine_fold_weights(w_plain, stats, gb)
        B, H, W, _ = f_G.shape
        if rec is not None:
            rec.update(stats=stats, gb=gb)
        if ops.scale_fusable() and rec is None:
            # f_E * m_E (model/vtoonify.py:127) is never written: the fusion conv multiplies f_E tiles by m_E while it splits
            # them for the tensor cores, and fusion_skip's 3-channel conv scales its loads (VToonify.forward)
            m_E = ops.smalln_conv(f_G, w_fold, ops.conv_taps(3, 1), 1, B, H, W, bias=self.conv2.bias, act=ACT_RELU_TANH,
                                  src2=f_E, tap_const=k_fold)
            return self.conv.forward_nhwc(f_G, x2=f_E, x2_scale=m_E), m_E, None
        m_E, fEm = ops.smalln_conv(f_G, w_fold, ops.conv_taps(3, 1), 1, B, H, W, bias=self.conv2.bias, act=ACT_RELU_TANH,
                                   mul_src=f_E, src2=f_E, tap_const=k_fold)
        f_out = self.conv.forward_nhwc(f_G, x2=fEm)
        return f_out, m_E, fEm

    def forward(self, f_G, f_E, d_s=1):
        f_out, m_E, _ = self.forward_nhwc(ops.to_nhwc(f_G), ops.to_nhwc(f_E), d_s)
        return ops.nhwc_as_nchw_view(f_out), m_E


class VToonify(ops.WeightsEpochMixin, nn.Module):
    """model/vtoonify.py:130-286"""

    def __init__(self, in_size=256, out_size=1024, img_channels=3, style_channels=512, num_mlps=8,
                 channel_multiplier=2, num_res_layers=6, backbone='dualstylegan'):
        super().__init__()
        self.backbone = backbone
        if self.backbone == 'dualstylegan':
            self.generator = DualStyleGAN(out_size, style_channels, num_mlps, channel_multiplier)
        else:
            self.generator = Generator(out_size, style_channels, num_mlps, channel_multiplier)
        self.in_size = in_size
        self.style_channels = style_channels
        channels = self.generator.channels

        encoder_res = [2 ** i for i in range(int(np.log2(in_size)), 4, -1)]
        self.encoder = nn.ModuleList()
        self.encoder.append(_ConvBlock(Conv2d(img_channels + 19, 32, 3, 1, 1), LeakyReLU(0.2),
                                       Conv2d(32, channels[in_size], 3, 1, 1), LeakyReLU(0.2)))
        for res in encoder_res:
            in_channels = channels[res]
            if res > 32:
                out_channels = channels[res // 2]
                self.encoder.append(_ConvBlock(Conv2d(in_channels, out_channels, 3, 2, 1), LeakyReLU(0.2),
                                               Conv2d(out_channels, out_channels, 3, 1, 1), LeakyReLU(0.2)))
            else:
                self.encoder.append(nn.Sequential(*[VToonifyResBlock(in_channels) for _ in range(num_res_layers)]))
                self.encoder.append(Conv2d(in_channels, img_channels, 1, 1, 0))

        self.fusion_out = nn.ModuleList()
        self.fusion_skip = nn.ModuleList()
        for res in encoder_res[::-1]:
            num_channels = channels[res]
            if self.backbone == 'dualstylegan':
                self.fusion_out.append(Fusion(num_channels, num_channels, num_channels))
            else:
                self.fusion_out.append(Conv2d(num_channels * 2, num_channels, 3, 1, 1))
            self.fusion_skip.append(Conv2d(num_channels + 3, 3, 3, 1, 1))

        if self.backbone == 'dualstylegan':
            self.res = nn.ModuleList()
            self.res.append(AdaResBlock(self.generator.channels[2 ** 2]))
            for i in range(3, 6):
                out_channel = self.generator.channels[2 ** i]
                self.res.append(AdaResBlock(out_channel, dilation=2 ** (5 - i)))
                self.res.append(AdaResBlock(out_channel, dilation=2 ** (5 - i)))

    # -------------------------------------------------------------------------------------------
    def _styles(self, style):
        """W+ codes: (adastyles, resstyles) — model/vtoonify.py:212-224."""
        D = self.backbone == 'dualstylegan'
        resstyles = None
        if style.ndim < 3:
            if D:
                resstyles = self.generator.style(style).unsqueeze(1).repeat(1, self.generator.n_latent, 1)
            adastyles = style.unsqueeze(1).repeat(1, self.generator.n_latent, 1)
        else:
            nB, nL, nD = style.shape
            if D:
                resstyles = self.generator.style(style.reshape(nB * nL, nD)).reshape(nB, nL, nD)
            adastyles = style
        if D:
            adastyles = adastyles.clone()
            for i in range(7, self.generator.n_latent):
                adastyles[:, i] = self.generator.res[i](adastyles[:, i])
        return adastyles, resstyles

    def forward(self, x, style, d_s=None, return_mask=False, return_feat=False):
        # One video = one style (style_transfer.py:138-150, 176): everything that depends on the style alone is computed once
        # per style tensor and, when all batch rows carry the same code, as a single shared row (per-sample weights wB = 1).
        token, shared = ops.style_token(self, style, (None if d_s is None else float(d_s),))
        with ops.style_scope(token):
            return self._forward(x, style[:1] if shared else style, d_s, return_mask, return_feat)

    def _forward(self, x, style, d_s, return_mask, return_feat):
        D = self.backbone == 'dualstylegan'
        adastyles, resstyles = ops.style_cached(self, "styles", lambda: self._styles(style))
        if return_feat and encoder_grad.takes_autograd(self, x):
            return encoder_grad.feat_with_grad(self, x, style, d_s, resstyles)
        if not return_feat and vtoonify_grad.takes_autograd(self, x):
            return vtoonify_grad.forward_with_grad(self, x, style, d_s, adastyles, resstyles, return_mask)

        # encoder: downsampling conv blocks, then the res blocks (interleaved with dilated ModRes for D)
        feat = ops.to_nhwc(x, ops._pad32(x.shape[1]))
        encoder_features = []
        for bi, block in enumerate(self.encoder[:-2]):
            with ops.nvtx_range(f"vtoonify/encoder.{bi}"):
                feat = block.forward_nhwc(feat)
            encoder_features.append(feat)
        encoder_features = encoder_features[::-1]
        for ii, block in enumerate(self.encoder[-2]):
            with ops.nvtx_range(f"vtoonify/resblock.{ii}"):
                if D and ops.affine_fusable():
                    feat, st = block.forward_nhwc(feat, want_stats=True)
                    feat = self.res[ii + 1].forward_nhwc(feat, resstyles[:, ii + 1], d_s, x_stats=st)
                else:
                    feat = block.forward_nhwc(feat)
                    if D:
                        feat = self.res[ii + 1].forward_nhwc(feat, resstyles[:, ii + 1], d_s)
        out = feat
        skip = self.encoder[-1].forward_smalln(feat)
        if return_feat:
            return ops.nhwc_as_nchw_view(out), skip

        G = self.stylegan()
        _index = 1
        m_Es = []
        levels = list(zip(G.convs[6::2], G.convs[7::2], G.to_rgbs[3:]))
        for lvl, (conv1, conv2, to_rgb) in enumerate(levels):
            if 2 ** (5 + ((_index - 1) // 2)) <= self.in_size:
                fi = (_index - 1) // 2
                f_E = encoder_features[fi]
                with ops.nvtx_range(f"vtoonify/fusion.{fi}"):
                    if D:
                        out, m_E, fEm = self.fusion_out[fi].forward_nhwc(out, f_E, d_s)
                        if fEm is None:
                            skip = self.fusion_skip[fi].forward_smalln(f_E, planar=skip, src_mask=m_E)
                        else:
                            skip = self.fusion_skip[fi].forward_smalln(fEm, planar=skip)
                        m_Es.append(m_E)
                    else:
                        out = self.fusion_out[fi].forward_nhwc(out, x2=f_E)
                        skip = self.fusion_skip[fi].forward_smalln(f_E, planar=skip)
            with ops.nvtx_range(f"vtoonify/generator.level{(_index - 1) // 2}"):
                out = conv1.forward_nhwc(out, adastyles[:, _index + 6], zero_noise=True)
                # the activation of the last level has no reader (model/vtoonify.py:273-284): only its image is produced
                out, skip = conv2.forward_nhwc(out, adastyles[:, _index + 7], zero_noise=True,
                                               to_rgb=(to_rgb, adastyles[:, _index + 8], skip), rgb_only=lvl == len(levels) - 1)
            _index += 2

        image = skip
        if return_mask and D:
            return image, m_Es
        return image

    def stylegan(self):
        return self.generator.generator if self.backbone == 'dualstylegan' else self.generator

    def zplus2wplus(self, zplus):
        return self.stylegan().style(zplus.reshape(zplus.shape[0] * zplus.shape[1], zplus.shape[2])).reshape(zplus.shape)
