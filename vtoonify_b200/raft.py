"""RAFT optical flow (model/raft/core/raft.py) as ``smooth_parsing_map.py`` runs it: a drop-in ``RAFT(args)`` with the reference's
constructor, submodule names and state_dict keys (179, including the BatchNorm buffers of ``cnet``), ``freeze_bn``,
``initialize_flow``, ``upsample_flow`` and ``forward(image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False)``.

Supported: the full model (``small=False``), ``mixed_precision=False``, ``alternate_corr=False``, dropout 0, eval mode, forward only.
Anything else raises ``NotImplementedError``; ``H`` or ``W`` not a multiple of 8 or below 128 raises ``ValueError`` (below 128 the
coarsest correlation level is one pixel wide or high and the reference's ``bilinear_sampler`` divides by zero).

The forward keeps every activation NHWC on the library's kernels (DESIGN.md section 11):
  * both encoders: the 7x7 / 2 stem as a 4x4 convolution over the space-to-depth tensor of ``2 * (x / 255) - 1`` (normalised before
    the stem's zero padding), ``cnet``'s BatchNorm folded into weights and bias with ReLU and the residual add in the epilogue,
    ``fnet``'s instance norm from the convolution's own statistics, applied with the ReLU (and shortcut) by one elementwise pass;
  * the all-pairs correlation: a 1x1 convolution of ``fmap1`` with per-sample weights ``fmap2`` (``Cout = h*w`` padded to 32), the
    1/16 in the epilogue, then three 2x2 mean pools and the 4 x 81-tap bilinear lookup into the 352-channel input of ``convc1``;
  * per iteration: the motion encoder writes into channels 128..253 of the GRU input ``x = [inp | motion | flow]``; each GRU half
    is one convolution for z|r (stacked weights), the reset gate, one convolution for q and the state update; the flow head ends in
    a planar 2-channel convolution whose output the coordinate update adds;
  * the mask head (its 0.25 folded into the last 1x1) and the convex up-sampling run after every iteration whose up-sampled flow is
    returned: all of them, or in test mode only the last.
"""
import torch
from torch import nn

from . import ops
from ._lib import ACT_LRELU, ACT_NONE, c_int64, c_void_p, check, load
from .bisenet import S2D_TAPS, s2d_stem_weight

HDIM = CDIM = 128
CORR_C = 4 * 81          # lookup channels
CORR_CPAD = 352          # ... padded to the convolution's 32-channel granule
MIN_SIZE = 128


def _relu_epi():
    return dict(act=ACT_LRELU, slope=0.0, gain=1.0)


def rect_taps(kh: int, kw: int):
    """(dy, dx, weight slab) of a kh x kw cross-correlation with 'same' zero padding ((kh - 1) / 2, (kw - 1) / 2)."""
    return [(ky - kh // 2, kx - kw // 2, ky * kw + kx) for ky in range(kh) for kx in range(kw)]


def fold_bn(conv: nn.Conv2d, bn: nn.BatchNorm2d):
    """conv (with bias) followed by eval-mode BatchNorm == conv with weight * a[n] and bias a[n] * b[n] + c[n]."""
    a = bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)
    c = bn.bias.detach() - bn.running_mean * a
    return (conv.weight.detach() * a.view(-1, 1, 1, 1)).contiguous(), (conv.bias.detach() * a + c).contiguous()


def stacked_zr(convz: nn.Conv2d, convr: nn.Conv2d):
    """convz | convr as one convolution with Cout = 2 * hidden: output channels [z logits | r logits]."""
    return (torch.cat([convz.weight.detach(), convr.weight.detach()], 0).contiguous(),
            torch.cat([convz.bias.detach(), convr.bias.detach()], 0).contiguous())


def motion_conv_weights(conv: nn.Conv2d):
    """the motion encoder's 126-channel output convolution padded to 128 output channels (two zero rows: ReLU(0) = 0)."""
    w, b = conv.weight.detach(), conv.bias.detach()
    pad = 128 - w.shape[0]
    return (torch.cat([w, w.new_zeros((pad,) + tuple(w.shape[1:]))], 0).contiguous(), torch.cat([b, b.new_zeros(pad)], 0).contiguous())


def mask_weights(conv: nn.Conv2d):
    """the mask head's last 1x1 with RAFT's ``.25 *`` folded in (an exact power-of-two scale)."""
    return (0.25 * conv.weight.detach()).contiguous(), (0.25 * conv.bias.detach()).contiguous()


def convf1_weights(conv: nn.Conv2d):
    """[Cout, 2, 7, 7] -> the direct kernel's [49, 2, Cout] layout."""
    return conv.weight.detach().permute(2, 3, 1, 0).reshape(49, 2, -1).contiguous()


# ---------------------------------------------------------------------------------------------- parameter holders (reference keys)
def _norm(kind, c):
    return nn.BatchNorm2d(c) if kind == "batch" else nn.InstanceNorm2d(c)


class ResidualBlock(nn.Module):
    """model/raft/core/extractor.py:6-56 (batch or instance norm)."""

    def __init__(self, in_planes, planes, norm_fn, stride=1):
        super().__init__()
        self.conv1 = nn.Conv2d(in_planes, planes, 3, padding=1, stride=stride)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1)
        self.relu = nn.ReLU(inplace=True)
        self.norm1 = _norm(norm_fn, planes)
        self.norm2 = _norm(norm_fn, planes)
        self.stride = stride
        self.downsample = None
        if stride != 1:
            self.norm3 = _norm(norm_fn, planes)
            self.downsample = nn.Sequential(nn.Conv2d(in_planes, planes, 1, stride=stride), self.norm3)


class BasicEncoder(nn.Module):
    """model/raft/core/extractor.py:118-192."""

    def __init__(self, output_dim=128, norm_fn="batch", dropout=0.0):
        super().__init__()
        self.norm_fn = norm_fn
        self.norm1 = _norm(norm_fn, 64)
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3)
        self.relu1 = nn.ReLU(inplace=True)
        self.layer1 = nn.Sequential(ResidualBlock(64, 64, norm_fn, 1), ResidualBlock(64, 64, norm_fn, 1))
        self.layer2 = nn.Sequential(ResidualBlock(64, 96, norm_fn, 2), ResidualBlock(96, 96, norm_fn, 1))
        self.layer3 = nn.Sequential(ResidualBlock(96, 128, norm_fn, 2), ResidualBlock(128, 128, norm_fn, 1))
        self.conv2 = nn.Conv2d(128, output_dim, 1)
        self.dropout = None


class BasicMotionEncoder(nn.Module):
    """model/raft/core/update.py:79-97."""

    def __init__(self, args):
        super().__init__()
        self.convc1 = nn.Conv2d(args.corr_levels * (2 * args.corr_radius + 1) ** 2, 256, 1)
        self.convc2 = nn.Conv2d(256, 192, 3, padding=1)
        self.convf1 = nn.Conv2d(2, 128, 7, padding=3)
        self.convf2 = nn.Conv2d(128, 64, 3, padding=1)
        self.conv = nn.Conv2d(64 + 192, 128 - 2, 3, padding=1)


class SepConvGRU(nn.Module):
    """model/raft/core/update.py:33-59."""

    def __init__(self, hidden_dim=128, input_dim=192 + 128):
        super().__init__()
        c = hidden_dim + input_dim
        self.convz1 = nn.Conv2d(c, hidden_dim, (1, 5), padding=(0, 2))
        self.convr1 = nn.Conv2d(c, hidden_dim, (1, 5), padding=(0, 2))
        self.convq1 = nn.Conv2d(c, hidden_dim, (1, 5), padding=(0, 2))
        self.convz2 = nn.Conv2d(c, hidden_dim, (5, 1), padding=(2, 0))
        self.convr2 = nn.Conv2d(c, hidden_dim, (5, 1), padding=(2, 0))
        self.convq2 = nn.Conv2d(c, hidden_dim, (5, 1), padding=(2, 0))


class FlowHead(nn.Module):
    """model/raft/core/update.py:6-14."""

    def __init__(self, input_dim=128, hidden_dim=256):
        super().__init__()
        self.conv1 = nn.Conv2d(input_dim, hidden_dim, 3, padding=1)
        self.conv2 = nn.Conv2d(hidden_dim, 2, 3, padding=1)
        self.relu = nn.ReLU(inplace=True)


class BasicUpdateBlock(nn.Module):
    """model/raft/core/update.py:114-136."""

    def __init__(self, args, hidden_dim=128, input_dim=128):
        super().__init__()
        self.args = args
        self.encoder = BasicMotionEncoder(args)
        self.gru = SepConvGRU(hidden_dim=hidden_dim, input_dim=128 + hidden_dim)
        self.flow_head = FlowHead(hidden_dim, hidden_dim=256)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 64 * 9, 1))


# ---------------------------------------------------------------------------------------------- the model
def _conv(srcs, wb, taps, stride=1, Ho=None, Wo=None, **epi):
    B, H, W, _ = srcs[0].shape
    return ops.conv2d_nhwc(srcs, wb[0], taps, stride, H if Ho is None else Ho, W if Wo is None else Wo, bias=wb[1], **epi)


def _norm_relu(x, stats, res=None, stats_res=None):
    B, H, W, C = x.shape
    out = torch.empty_like(x)
    check(load().vt_raft_norm_relu_nhwc(x.data_ptr(), stats.data_ptr(), ops._ptr(res), ops._ptr(stats_res), out.data_ptr(), B, H * W, C,
                                        ops._stream()))
    return out


class RAFT(nn.Module):
    """model/raft/core/raft.py:24-144 on the library (see the module docstring for what is supported)."""

    def __init__(self, args):
        super().__init__()
        self.args = args
        if args.small:
            raise NotImplementedError("RAFT: small=True (the small model) is not supported; only the full model is")
        self.hidden_dim = HDIM
        self.context_dim = CDIM
        args.corr_levels = 4
        args.corr_radius = 4
        if "dropout" not in self.args:
            self.args.dropout = 0
        if "alternate_corr" not in self.args:
            self.args.alternate_corr = False
        if getattr(args, "mixed_precision", False):
            raise NotImplementedError("RAFT: mixed_precision=True is not supported")
        if self.args.alternate_corr:
            raise NotImplementedError("RAFT: alternate_corr=True (alt_cuda_corr) is not supported")
        if self.args.dropout:
            raise NotImplementedError("RAFT: dropout > 0 is not supported")
        self.fnet = BasicEncoder(output_dim=256, norm_fn="instance", dropout=args.dropout)
        self.cnet = BasicEncoder(output_dim=HDIM + CDIM, norm_fn="batch", dropout=args.dropout)
        self.update_block = BasicUpdateBlock(self.args, hidden_dim=HDIM)
        self._wcache = {}

    def freeze_bn(self):
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.eval()

    def initialize_flow(self, img):
        """the pixel grids (coords0, coords1), [N, 2, H/8, W/8] with channel 0 = x"""
        N, C, H, W = img.shape
        ys, xs = torch.meshgrid(torch.arange(H // 8, device=img.device), torch.arange(W // 8, device=img.device), indexing="ij")
        coords = torch.stack([xs, ys], dim=0).float()[None].repeat(N, 1, 1, 1)
        return coords, coords.clone()

    def upsample_flow(self, flow, mask):
        """flow [N, 2, H, W] and mask [N, 576, H, W] (planar CUDA fp32) -> the convex up-sampling [N, 2, 8H, 8W]"""
        N, _, H, W = flow.shape
        if tuple(mask.shape) != (N, 576, H, W):
            raise ValueError(f"RAFT.upsample_flow: mask {tuple(mask.shape)} must be [{N}, 576, {H}, {W}]")
        ops._req_cuda(flow, mask)
        coords = torch.empty((N, H, W, 2), device=flow.device, dtype=torch.float32)      # grid + flow, as forward keeps it
        check(load().vt_raft_flow_f32(coords.data_ptr(), flow.contiguous().data_ptr(), 1, None, 2, N, H, W, ops._stream()))
        up = torch.empty((N, 2, 8 * H, 8 * W), device=flow.device, dtype=torch.float32)
        m = ops.to_nhwc(mask, round_tf32=False).contiguous()
        check(load().vt_raft_upsample_f32(m.data_ptr(), 576, coords.data_ptr(), up.data_ptr(), None, N, H, W, ops._stream()))
        return up

    # ------------------------------------------------------------------------------------------ weights
    def _cached(self, name, tensors, fn):
        key = tuple((t.data_ptr(), t._version) for t in tensors) + (ops.get_precision(),)
        hit = self._wcache.get(name)
        if hit is None or hit[0] != key:
            with torch.no_grad():
                hit = (key, fn())
            self._wcache[name] = hit
        return hit[1]

    def _plain(self, name, conv, cin, fold=None, transform=None):
        """(prepared weight, bias) of ``conv`` (optionally BN-folded or transformed), input channels padded to ``cin``."""
        ts = [conv.weight, conv.bias] + ([] if fold is None else [fold.weight, fold.bias, fold.running_mean, fold.running_var])

        def make():
            if fold is not None:
                w, b = fold_bn(conv, fold)
            elif transform is not None:
                w, b = transform(conv)
            else:
                w, b = conv.weight.detach().contiguous(), conv.bias.detach().contiguous()
            return ops.prep_weights(w, cin_pad=cin), b
        return self._cached(name, ts, make)

    def _stem(self, name, enc):
        bn = enc.norm1 if enc.norm_fn == "batch" else None
        ts = [enc.conv1.weight, enc.conv1.bias] + ([] if bn is None else [bn.weight, bn.bias, bn.running_mean, bn.running_var])

        def make():
            w, b = fold_bn(enc.conv1, bn) if bn is not None else (enc.conv1.weight.detach(), enc.conv1.bias.detach().contiguous())
            return ops.prep_weights(s2d_stem_weight(w).contiguous(), cin_pad=32), b
        return self._cached(name, ts, make)

    # ------------------------------------------------------------------------------------------ encoders
    def _encode(self, name, enc, z):
        """BasicEncoder.forward on the space-to-depth input z [n, H/2, W/2, 32] -> NHWC [n, H/8, W/8, out]"""
        inst = enc.norm_fn == "instance"
        n, H2, W2, _ = z.shape
        ws = self._stem(name + ".stem", enc)
        if inst:
            x = _norm_relu(*_conv([z], ws, S2D_TAPS, want_stats=True))
        else:
            x = _conv([z], ws, S2D_TAPS, **_relu_epi())
        for li, layer in enumerate((enc.layer1, enc.layer2, enc.layer3)):
            for bi, blk in enumerate(layer):
                key = f"{name}.{li}.{bi}"
                C = x.shape[3]
                Ho = ops.conv_out_size(x.shape[1], 3, blk.stride, 1, 1)
                Wo = ops.conv_out_size(x.shape[2], 3, blk.stride, 1, 1)
                t3 = ops.conv_taps(3, 1)
                if inst:
                    y = _norm_relu(*_conv([x], self._plain(key + ".c1", blk.conv1, C), t3, blk.stride, Ho, Wo, want_stats=True))
                    y, s2 = _conv([y], self._plain(key + ".c2", blk.conv2, y.shape[3]), t3, want_stats=True)
                    if blk.downsample is not None:
                        sc, s3 = _conv([x], self._plain(key + ".ds", blk.downsample[0], C), ops.conv_taps(1, 0), blk.stride, Ho, Wo,
                                       want_stats=True)
                        x = _norm_relu(y, s2, sc, s3)
                    else:
                        x = _norm_relu(y, s2, x)
                else:
                    y = _conv([x], self._plain(key + ".c1", blk.conv1, C, fold=blk.norm1), t3, blk.stride, Ho, Wo, **_relu_epi())
                    sc = x
                    if blk.downsample is not None:
                        sc = _conv([x], self._plain(key + ".ds", blk.downsample[0], C, fold=blk.norm3), ops.conv_taps(1, 0), blk.stride,
                                   Ho, Wo)
                    # relu(shortcut + relu(bn2(conv2 y))): ReLU and the add in the epilogue, the outer ReLU as one elementwise pass
                    y = _conv([y], self._plain(key + ".c2", blk.conv2, y.shape[3], fold=blk.norm2), t3, res=sc, **_relu_epi())
                    x = ops.fused_bias_act(y, None, 0.0, 1.0)
        return _conv([x], self._plain(name + ".out", enc.conv2, x.shape[3]), ops.conv_taps(1, 0))

    # ------------------------------------------------------------------------------------------ forward
    def _check_model(self):
        """the module-level limits of the forward: eval mode, and no parameter that requires grad in grad mode"""
        if self.training:
            raise NotImplementedError("RAFT: train mode is not supported (BatchNorm would need batch statistics); call .eval()")
        if torch.is_grad_enabled():
            for nm, p in self.named_parameters():
                if p.requires_grad:
                    raise NotImplementedError(f"RAFT: parameter {nm} requires grad; the module is forward only "
                                              "(run it under torch.no_grad())")

    def _check(self, image1, image2, iters, flow_init):
        if self.training:
            raise NotImplementedError("RAFT: train mode is not supported (BatchNorm would need batch statistics); call .eval()")
        if torch.is_grad_enabled():
            for nm, t in (("image1", image1), ("image2", image2), ("flow_init", flow_init)):
                if t is not None and t.requires_grad:
                    raise NotImplementedError(f"RAFT: {nm} requires grad; the module is forward only (run it under torch.no_grad())")
            for nm, p in self.named_parameters():
                if p.requires_grad:
                    raise NotImplementedError(f"RAFT: parameter {nm} requires grad; the module is forward only "
                                              "(run it under torch.no_grad())")
        if image1.dim() != 4 or image1.shape[1] != 3 or tuple(image2.shape) != tuple(image1.shape):
            raise ValueError(f"RAFT: image1 {tuple(image1.shape)} and image2 {tuple(image2.shape)} must both be [B, 3, H, W]")
        B, _, H, W = image1.shape
        if H % 8 or W % 8 or H < MIN_SIZE or W < MIN_SIZE:
            raise ValueError(f"RAFT: H and W must be multiples of 8 and at least {MIN_SIZE} (got {H}x{W}); pad with InputPadder")
        if flow_init is not None and tuple(flow_init.shape) != (B, 2, H // 8, W // 8):
            raise ValueError(f"RAFT: flow_init {tuple(flow_init.shape)} must be [{B}, 2, {H // 8}, {W // 8}]")
        if int(iters) < 1:
            raise ValueError("RAFT: iters must be at least 1")
        ops._req_cuda(image1, image2, flow_init)

    def forward(self, image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False):
        self._check(image1, image2, iters, flow_init)
        with torch.no_grad():
            return self._forward(image1.contiguous(), image2.contiguous(), int(iters), flow_init, test_mode)

    def _forward(self, image1, image2, iters, flow_init, test_mode):
        B = image1.shape[0]
        with ops.nvtx_range("raft.encoders"):
            z = self._input_s2d(image1, image2)
            fmap = self._features(z)                                   # [2B, h, w, 256]: fmap1 | fmap2
            net, x = self._context(z[:B])
        return self._iterate(fmap[:B], fmap[B:], net, x, iters, flow_init, test_mode)

    # the three steps of the forward, also used on their own by smooth_parsing.smooth_parsing_maps, which encodes each frame once
    def _input_s2d(self, image1, image2=None):
        """the space-to-depth stem input [n, H/2, W/2, 32] of 2 * (x / 255) - 1 for image1 (then image2), planar [B, 3, H, W] in 0..255"""
        B, _, H, W = image1.shape
        z = torch.empty(((1 if image2 is None else 2) * B, H // 2, W // 2, 32), device=image1.device, dtype=torch.float32)
        check(load().vt_raft_input_s2d_f32(image1.data_ptr(), ops._ptr(image2), z.data_ptr(), B, H, W, 32, ops._stream()))
        return z

    def _features(self, z):
        """the encoder step: fnet's features NHWC [n, H/8, W/8, 256] of the stem inputs z (instance norm: per sample)"""
        return self._encode("fnet", self.fnet, z)

    def _context(self, z):
        """the context step: cnet on the stem inputs z -> the GRU state net [n, h, w, 128] = tanh and the GRU input buffer
        x [n, h, w, 256] whose channels 0..127 hold inp = relu (the iterations write the rest)"""
        n, H2, W2, _ = z.shape
        h, w = H2 // 4, W2 // 4
        cnet = self._encode("cnet", self.cnet, z)                     # [n, h, w, 256]
        net = torch.empty((n, h, w, HDIM), device=z.device, dtype=torch.float32)
        x = torch.empty((n, h, w, 256), device=z.device, dtype=torch.float32)      # GRU input [inp | motion | flow]
        check(load().vt_raft_context_f32(cnet.data_ptr(), net.data_ptr(), x.data_ptr(), n * h * w, HDIM, 256, ops._stream()))
        return net, x

    def _iterate(self, fmap1, fmap2, net, x, iters, flow_init=None, test_mode=True):
        """the iteration step: correlation pyramid of (fmap1, fmap2) [B, h, w, 256], ``iters`` updates of the GRU state ``net`` and
        input ``x`` (both updated in place), mask head and convex up-sampling; returns what ``forward`` returns"""
        lib, st = load(), ops._stream()
        B, h, w, _ = fmap1.shape
        H, W = 8 * h, 8 * w
        dev = fmap1.device
        ub = self.update_block

        with ops.nvtx_range("raft.correlation"):
            levels = self._pyramid(fmap1, fmap2, B, h, w)

        coords = torch.empty((B, h, w, 2), device=dev, dtype=torch.float32)
        fi = None if flow_init is None else flow_init.contiguous()
        check(lib.vt_raft_flow_f32(coords.data_ptr(), ops._ptr(fi), 1, None, 2, B, h, w, st))
        corr = torch.zeros((B, h, w, CORR_CPAD), device=dev, dtype=torch.float32)
        lv_ptr = (c_void_p * 4)(*[t.data_ptr() for t, _, _, _ in levels])
        lv_stride = (c_int64 * 4)(*[s for _, s, _, _ in levels])
        npix = B * h * w
        x_motion = (128, h * w * 256, w * 256, 256)
        t15, t51, t3, t1 = rect_taps(1, 5), rect_taps(5, 1), ops.conv_taps(3, 1), ops.conv_taps(1, 0)
        enc, gru = ub.encoder, ub.gru
        w_c1 = self._plain("c1", enc.convc1, CORR_CPAD)
        w_c2 = self._plain("c2", enc.convc2, 256)
        w_f1 = self._cached("f1", [enc.convf1.weight], lambda: convf1_weights(enc.convf1))
        w_f2 = self._plain("f2", enc.convf2, 128)
        w_mo = self._plain("mo", enc.conv, 256, transform=motion_conv_weights)
        w_zr = [self._cached(f"zr{i}", [getattr(gru, f"convz{i}").weight, getattr(gru, f"convz{i}").bias,
                                         getattr(gru, f"convr{i}").weight, getattr(gru, f"convr{i}").bias],
                             lambda i=i: (lambda wb: (ops.prep_weights(wb[0], cin_pad=384), wb[1]))(
                                 stacked_zr(getattr(gru, f"convz{i}"), getattr(gru, f"convr{i}"))))
                for i in (1, 2)]
        w_q = [self._plain(f"q{i}", getattr(gru, f"convq{i}"), 384) for i in (1, 2)]
        w_h1 = self._plain("h1", ub.flow_head.conv1, HDIM)
        w_h2 = self._cached("h2", [ub.flow_head.conv2.weight],
                            lambda: ops.prep_weights(ub.flow_head.conv2.weight.detach().contiguous(), cin_pad=256, round_tf32=False))
        w_m0 = self._plain("m0", ub.mask[0], HDIM)
        w_m2 = self._plain("m2", ub.mask[2], 256, transform=mask_weights)
        rh = torch.empty_like(net)
        preds = []
        low = None
        with ops.nvtx_range("raft.iterations"):
            for itr in range(iters):
                check(lib.vt_raft_corr_lookup_f32(lv_ptr, lv_stride, h, w, coords.data_ptr(), corr.data_ptr(), CORR_CPAD, npix, st))
                c = _conv([corr], w_c1, t1, **_relu_epi())
                c = _conv([c], w_c2, t3, **_relu_epi())
                f = torch.empty((B, h, w, 128), device=dev, dtype=torch.float32)
                check(lib.vt_raft_convf1_f32(coords.data_ptr(), w_f1.data_ptr(), enc.convf1.bias.data_ptr(), f.data_ptr(), B, h, w, 128, st))
                f = _conv([f], w_f2, t3, **_relu_epi())
                ops.conv2d_nhwc([c, f], w_mo[0], t3, 1, h, w, out=x, out_view=x_motion, bias=w_mo[1], **_relu_epi())
                check(lib.vt_raft_flow_f32(coords.data_ptr(), None, 0, x[..., 254:].data_ptr(), 256, B, h, w, st))
                for half, taps in ((0, t15), (1, t51)):
                    zr = _conv([net, x], w_zr[half], taps)
                    check(lib.vt_raft_gru_reset_f32(zr.data_ptr(), net.data_ptr(), rh.data_ptr(), npix, HDIM, st))
                    q = _conv([rh, x], w_q[half], taps)
                    check(lib.vt_raft_gru_update_f32(zr.data_ptr(), q.data_ptr(), net.data_ptr(), npix, HDIM, st))
                fh = _conv([net], w_h1, t3, **_relu_epi())
                delta = ops.smalln_conv(fh, w_h2, t3, 2, B, h, w, bias=ub.flow_head.conv2.bias)
                check(lib.vt_raft_flow_f32(coords.data_ptr(), delta.data_ptr(), 0, None, 2, B, h, w, st))
                last = itr == iters - 1
                if test_mode and not last:
                    continue
                m = _conv([net], w_m0, t3, **_relu_epi())
                m = _conv([m], w_m2, t1)
                up = torch.empty((B, 2, H, W), device=dev, dtype=torch.float32)
                if last and test_mode:
                    low = torch.empty((B, 2, h, w), device=dev, dtype=torch.float32)
                check(lib.vt_raft_upsample_f32(m.data_ptr(), 576, coords.data_ptr(), up.data_ptr(), ops._ptr(low), B, h, w, st))
                preds.append(up)
        if test_mode:
            return low, preds[-1]
        return preds

    def _pyramid(self, fmap1, fmap2, B, h, w):
        """the correlation pyramid: [(tensor, row stride, h_l, w_l)] of the 4 levels, level 0 [B, h, w, pad32(h*w)]"""
        lib, st = load(), ops._stream()
        hw = h * w
        cp = ops._pad32(hw)
        wc = torch.zeros((B, 1, cp, 256), device=fmap1.device, dtype=torch.float32)
        wc[:, 0, :hw].copy_(fmap2.reshape(B, hw, 256))
        c0 = ops.conv2d_nhwc([fmap1], wc, [(0, 0, 0)], 1, h, w, alpha=1.0 / 16.0)   # fmap1 . fmap2 / sqrt(256)
        levels = [(c0, cp, h, w)]
        N = B * hw
        for _ in range(3):
            src, stride, hl, wl = levels[-1]
            out = torch.empty((N, (hl // 2) * (wl // 2)), device=fmap1.device, dtype=torch.float32)
            check(lib.vt_raft_corr_pool_f32(src.data_ptr(), out.data_ptr(), N, hl, wl, stride, st))
            levels.append((out, (hl // 2) * (wl // 2), hl // 2, wl // 2))
        return levels
