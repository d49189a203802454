"""DualStyleGAN pieces used by VToonify (model/dualstylegan.py:6-76) with identical state_dict keys."""
import math

import torch
from torch import nn

from . import ops
from .stylegan import ConvLayer, EqualLinear, Generator, PixelNorm


class Linear(nn.Module):
    """nn.Linear replacement (same ``weight``/``bias`` keys and default init) running on vt_linear_f32.
    ``act``: 0 none, 2 LeakyReLU(0.2) fused."""

    def __init__(self, in_features, out_features, act=0):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        self.bias = nn.Parameter(torch.empty(out_features))
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        bound = 1 / math.sqrt(in_features)
        nn.init.uniform_(self.bias, -bound, bound)
        self.act = act

    def forward(self, input, act=None):
        return ops.linear(input, self.weight, self.bias, 1.0, 1.0, self.act if act is None else act)


class AdaptiveInstanceNorm(nn.Module):
    """model/dualstylegan.py:6-21: InstanceNorm2d(affine=False) then gamma * x + beta, [gamma|beta] = Linear(style)."""

    def __init__(self, fin, style_dim=512):
        super().__init__()
        self.style = Linear(style_dim, fin * 2)
        self.style.bias.data[:fin] = 1
        self.style.bias.data[fin:] = 0

    def gamma_beta(self, style, B):
        """[B, 2C] rows (gamma | beta) = Linear(style); style-only, so computed once per style inside a style scope
        (a shared [1, D] style is broadcast to the batch)"""
        def make():
            gb = self.style(style)
            return gb if gb.shape[0] == B else gb.expand(B, -1).contiguous()
        return ops.style_cached(self, "gb", make, extra=(B, self.style.weight._version))

    def forward_nhwc(self, x, style, x2=None):
        gb = self.gamma_beta(style, x.shape[0])
        stats = ops.instnorm_stats(x, x2)
        return ops.adain_apply(x, stats, gb, x2)

    def affine(self, x, style, stats=None):
        """The same AdaIN as a [B, C, 2] (scale, shift) table for a convolution that applies it to its input on the fly.
        ``stats``: (mean, rstd) of ``x`` when the kernel that produced ``x`` already delivered them."""
        return ops.adain_affine(ops.instnorm_stats(x) if stats is None else stats, self.gamma_beta(style, x.shape[0]))

    def forward(self, input, style):
        return ops.nhwc_as_nchw_view(self.forward_nhwc(ops.to_nhwc(input), style))


class AdaResBlock(nn.Module):
    """model/dualstylegan.py:24-45 (ModRes): x + w * conv2(AdaIN(conv(AdaIN(x, s)), s))."""

    def __init__(self, fin, style_dim=512, dilation=1):
        super().__init__()
        self.conv = ConvLayer(fin, fin, 3, dilation=dilation)
        self.conv2 = ConvLayer(fin, fin, 3, dilation=dilation)
        self.norm = AdaptiveInstanceNorm(fin, style_dim)
        self.norm2 = AdaptiveInstanceNorm(fin, style_dim)
        self.conv[0].weight.data *= 0.01
        self.conv2[0].weight.data *= 0.01

    def forward_nhwc(self, x, s, w=1, x_stats=None):
        """``x_stats``: instance-norm statistics of ``x`` from the kernel that produced it (else a statistics pass runs)."""
        if w == 0:
            return x
        if ops.affine_fusable():
            # the normalised tensors are never written: each conv applies its AdaIN (scale, shift per sample and channel) to
            # the pixels it stages, padding stays zero as in the reference (which zero-pads the normalised tensor); the
            # statistics of conv's output come out of conv's own epilogue
            out, st = self.conv.forward_nhwc(x, src_affine=self.norm.affine(x, s, x_stats), want_stats=True)
            return self.conv2.forward_nhwc(out, src_affine=self.norm2.affine(out, s, st), res=x, alpha=float(w), beta=1.0)
        out = self.conv.forward_nhwc(self.norm.forward_nhwc(x, s))
        return self.conv2.forward_nhwc(self.norm2.forward_nhwc(out, s), res=x, alpha=float(w), beta=1.0)

    def forward(self, x, s, w=1):
        return ops.nhwc_as_nchw_view(self.forward_nhwc(ops.to_nhwc(x), s, w))


class DualStyleGAN(ops.WeightsEpochMixin, nn.Module):
    """model/dualstylegan.py:47-203: same constructor, parameters / keys and ``forward`` keyword interface (forward only).
    VToonify uses ``.style``, ``.res[7:]`` and ``.generator`` (model/vtoonify.py:214-224, 279-283); ``forward`` is the
    exemplar-based synthesis with the extrinsic style path, the frozen teacher of VToonify-D training."""

    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, twoRes=True, res_index=6):
        super().__init__()
        layers = [PixelNorm()]
        for _ in range(n_mlp - 6):
            layers.append(EqualLinear(512, 512, lr_mul=0.01, activation="fused_lrelu"))
        self.style = nn.Sequential(*layers)
        self.generator = Generator(size, style_dim, n_mlp, channel_multiplier)
        self.res = nn.ModuleList()
        self.res_index = res_index // 2 * 2
        self.res.append(AdaResBlock(self.generator.channels[2 ** 2]))
        for i in range(3, self.generator.log_size + 1):
            out_channel = self.generator.channels[2 ** i]
            if i < 3 + self.res_index // 2:
                self.res.append(AdaResBlock(out_channel))
                self.res.append(AdaResBlock(out_channel))
            else:
                for _ in range(2):
                    self.res.append(EqualLinear(512, 512))
                    self.res[-1].weight.data = torch.eye(512) * 512.0 ** 0.5 + torch.randn(512, 512) * 0.01
        self.res.append(EqualLinear(512, 512))
        self.res[-1].weight.data = torch.eye(512) * 512.0 ** 0.5 + torch.randn(512, 512) * 0.01
        self.size = self.generator.size
        self.style_dim = self.generator.style_dim
        self.log_size = self.generator.log_size
        self.num_layers = self.generator.num_layers
        self.n_latent = self.generator.n_latent
        self.channels = self.generator.channels

    def forward(self, styles, exstyles, return_latents=False, return_feat=False, inject_index=None, truncation=1,
                truncation_latent=None, input_is_latent=False, noise=None, randomize_noise=True, z_plus_latent=False,
                use_res=True, fuse_index=18, interp_weights=[1] * 18):
        """model/dualstylegan.py:84-194 -> ``(image, latent | None)``, or ``(feat, skip)`` with ``return_feat``."""
        G = self.generator
        latent, noise, cacheable = G._prepare(styles, inject_index, truncation, truncation_latent, input_is_latent, noise,
                                              randomize_noise, z_plus_latent)
        weights = tuple(float(w) for w in interp_weights)
        token = None
        if cacheable:
            # every style-only tensor (extrinsic codes, blended styles, modulated weights, AdaIN rows) is memoised while the caller
            # passes the same unmodified latent and exstyles objects with the same weights and path selection
            ex_token = ops.style_token(self.style, exstyles)[0] if use_res else None
            token = ops.style_token(self, latent, (ex_token, weights, fuse_index, bool(use_res)))[0]
        with ops.style_scope(token):
            feat, image = self._synthesis(latent, exstyles, noise, return_feat, use_res, fuse_index, weights)
        if feat is not None:
            return feat, image
        return image, (latent if return_latents else None)

    def _synthesis(self, latent, exstyles, noise, return_feat, use_res, fuse_index, w):
        """model/dualstylegan.py:147-188 on NHWC activations -> ``(feat, skip image)``; ``feat`` (an NCHW view of the
        activation) is None unless ``return_feat`` stopped the loop after the first level above ``res_index``."""
        G = self.generator
        if use_res:         # the colour transform T_c on the extrinsic code, for the ModRes blocks
            resstyles = ops.style_cached(self, "resstyles",
                                         lambda: self.style(exstyles.reshape(-1, exstyles.shape[-1])).reshape(exstyles.shape))

        def per_layer(t, j):            # a [B, 512] code stands for every layer (the reference repeats it)
            return t if t.ndim == 2 else t[:, j]

        def modres(j):                  # a ModRes block follows conv layer j; weight 0 makes it the identity, so it is absent
            return use_res and fuse_index >= max(j, 1) and j <= self.res_index and w[j] != 0

        def style(j):                   # layer j's style: above res_index, the blend with the structure transform T_s
            if not (use_res and fuse_index >= j and j > self.res_index) or w[j] == 0:
                return latent[:, j]     # (weight 0: exactly the intrinsic code)
            return ops.style_cached(self, f"style{j}", lambda: ops.axpby(self.res[j](per_layer(exstyles, j)), latent[:, j], w[j],
                                                                          1.0 - w[j], round_tf32=False))

        def styled(conv, x, j, n):      # StyledConv j and its ModRes block, which takes the conv's output statistics
            if not modres(j):
                return conv.forward_nhwc(x, style(j), noise=n)
            st = None
            if ops.affine_fusable():
                x, st = conv.forward_nhwc(x, style(j), noise=n, want_stats=True)
            else:
                x = conv.forward_nhwc(x, style(j), noise=n)
            return self.res[j].forward_nhwc(x, per_layer(resstyles, j), w[j], x_stats=st)

        out = styled(G.conv1, ops.to_nhwc(G.input(latent)), 0, noise[0])
        skip = G.to_rgb1.forward_nhwc(out, latent[:, 1])
        i = 1
        n_levels = len(G.to_rgbs)
        for lvl, (conv1, conv2, noise1, noise2, to_rgb) in enumerate(zip(G.convs[::2], G.convs[1::2], noise[1::2], noise[2::2],
                                                                         G.to_rgbs)):
            out = styled(conv1, out, i, noise1)
            feat_here = return_feat and i + 2 > self.res_index
            if modres(i + 1):
                # ToRGB reads the ModRes output: its own launch
                out = styled(conv2, out, i + 1, noise2)
                skip = to_rgb.forward_nhwc(out, style(i + 2), skip)
            else:
                out, skip = conv2.forward_nhwc(out, style(i + 1), noise=noise2, to_rgb=(to_rgb, style(i + 2), skip),
                                               rgb_only=lvl == n_levels - 1 and not feat_here)
            i += 2
            if feat_here:
                return ops.nhwc_as_nchw_view(out), skip
        return None, skip

    def make_noise(self):
        return self.generator.make_noise()

    def mean_latent(self, n_latent):
        return self.generator.mean_latent(n_latent)

    def get_latent(self, input):
        return self.generator.style(input)
