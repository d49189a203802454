"""Functional layer over the C-ABI: every function launches hand-written sm_90a kernels from
libvtoonify_b200.so on torch CUDA tensors (torch is used for memory and streams only).

Internal activation layout is NHWC (``[B, H, W, C]`` contiguous fp32); the reference-facing modules
convert at the API boundary (NCHW in / out, or zero-copy when a tensor is channels_last).
"""
import math
import os as _os
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import ACT_LRELU, ACT_NONE, ACT_RELU_TANH, ConvDesc, SmallNDesc, check

SQRT2 = math.sqrt(2.0)

# Convolution arithmetic (set_precision):
# "bf16x3" (default, the product path): wgmma tensor-core convolutions with every fp32 operand split into bf16 hi + lo parts
#   (pixels in shared memory, weights by vt_split_weights_bf16x3) and three MMA products per K step, fp32 accumulate:
#   a_hi*w_hi + a_lo*w_hi + a_hi*w_lo.  Meets the 1e-3 per-pixel parity bar (tests/test_gpu_vtoonify.py, test_gpu_fullsize.py).
# "tf32": the same kernel with TF32 operands: fewer MMA products, but 10-bit mantissas put the ~47-layer VToonify-D output
#   above the parity bar.  Opt-in.
# "fp32": every convolution on the fp32-exact FFMA kernel (used to cross-check the tensor-core paths).
DEFAULT_PRECISION = "bf16x3"
_precision = DEFAULT_PRECISION


def set_precision(p: str) -> str:
    global _precision
    if p not in ("tf32", "bf16x3", "fp32"):
        raise ValueError("precision must be 'tf32', 'bf16x3' or 'fp32'")
    old, _precision = _precision, p
    return old


def get_precision() -> str:
    return _precision


# algorithm switches (kept so tests can compare both formulations on the GPU)
# fold_upconv: True = always fold Blur o conv_transpose into one N = 4*Cout convolution; an int = only when Cin <= that value
# (the folded form issues 4x the MMA work but has no intermediate tensor; tools/upconv_bench.py compares the two; the threshold
# of 128 has not been re-measured on H100).  fuse_mask_mul: Fusion's f_E * m_E is applied inside the consumers instead of being materialised.
# rs_conv: 3x3 / stride 1 / padding 1 layers with Cin, Cout in {32, 64} and at least rs_min_width pixels per row go through the
# row-strip entry point (vt_conv2d_rs), which can also produce the fused ToRGB image alone; rs_fmt: the operand split of the
# tensor-core mode ("bf16" | "f16": fp16 halves carry 11 + 11 mantissa bits instead of 8 + 8, weights pre-scaled by F16_WEIGHT_SCALE).
_options = {"fold_upconv": 128, "fuse_torgb": True, "fuse_mask_mul": True, "smalln_via_tc": True, "bf16x3_nstack": False, "fuse_adain": True,
            "rs_conv": True, "rs_min_width": 256, "rs_fmt": _os.environ.get("VT_SPLIT_FMT", "bf16"), "nvtx": bool(_os.environ.get("VT_NVTX")),
            # rsu_conv: up-convolutions with Cin <= rsu_max_cin and rows of >= rs_min_width pixels go through conv_up2_rs_nhwc
            "rsu_conv": True, "rsu_max_cin": 128,
            # fuse_stats: AdaIN statistics of a conv output come from the producing kernel's epilogue (per-tile partial sums + finalize)
            # instead of a separate pass over the tensor
            "fuse_stats": True,
            # raft_corr: RAFT's correlation lookup from the all-pairs volume ("volume": the pyramid of fmap1 . fmap2, O((h*w)^2) memory)
            # or computed at each lookup from fmap1 and the pooled fmap2 ("on_demand": AlternateCorrBlock, O(h*w*256) memory)
            "raft_corr": "volume"}
if _os.environ.get("VT_FOLD_UPCONV_MAX_CIN"):
    _options["fold_upconv"] = int(_os.environ["VT_FOLD_UPCONV_MAX_CIN"])


def use_folded_upconv(cin: int) -> bool:
    v = _options["fold_upconv"]
    return bool(v) if isinstance(v, bool) else cin <= int(v)


_OPTION_ALIASES = {"split_fmt": "rs_fmt"}


def set_option(name: str, value) -> None:
    name = _OPTION_ALIASES.get(name, name)
    if name not in _options:
        raise KeyError(name)
    if name == "rs_fmt" and value not in ("bf16", "f16"):
        raise ValueError("split_fmt must be 'bf16' or 'f16'")
    if name == "raft_corr" and value not in ("volume", "on_demand"):
        raise ValueError("raft_corr must be 'volume' or 'on_demand'")
    _options[name] = value


def get_option(name: str):
    return _options[_OPTION_ALIASES.get(name, name)]


# fp16 split: weights are multiplied by this power of two before the split so that the low halves of small (demodulated,
# 1/sqrt(fan_in)-sized) weights stay out of fp16's subnormal range; the kernels undo it on the accumulators (acc_scale).
# |weight| must stay below 65504 / 256.
F16_WEIGHT_SCALE = 256.0


# Optional per-launch timing of the tensor-core convolution (bench.py's roofline leg): when set to a list, every
# vt_conv2d_tc_tf32 launch appends (start_event, end_event, algorithmic_flops, algorithmic_bytes, label, issued_mma_flops).
_tc_profile = None


def set_tc_profile(sink):
    global _tc_profile
    old, _tc_profile = _tc_profile, sink
    return old


# ----------------------------------------------------------------------------------------------
# per-style caching (SURVEY.md section 7 step 8): within one video every frame batch carries the same style code
# (style_transfer.py:138-150, 176), so everything that depends on the style only -- the W+ transforms, the 15 modulation
# linears, the modulated / demodulated / folded / split weights, the AdaIN gamma|beta rows -- is computed once per style.
# A *scope* names the style by a token; modules memoise their style-only tensors per token (one entry per site, replaced when
# the token changes).  Tokens are identity based (same tensor object, same version => same content), never content hashed.
# ----------------------------------------------------------------------------------------------
import itertools as _itertools

_token_counter = _itertools.count(1)
_scope_stack = []
_weights_epoch = 0


def bump_weights_epoch():
    """invalidate every style token (called when a model's parameters are (re)loaded or moved)"""
    global _weights_epoch
    _weights_epoch += 1


class WeightsEpochMixin:
    """nn.Module mixin: ``load_state_dict`` / ``.to()`` / ``.cuda()`` invalidate the per-style caches"""

    def load_state_dict(self, *args, **kwargs):
        r = super().load_state_dict(*args, **kwargs)
        bump_weights_epoch()
        return r

    def _apply(self, fn, *args, **kwargs):
        r = super()._apply(fn, *args, **kwargs)
        bump_weights_epoch()
        return r


class style_scope:
    """``with ops.style_scope(token):`` — modules called inside memoise style-only tensors under ``token`` (None: no caching)."""

    def __init__(self, token):
        self.token = token

    def __enter__(self):
        _scope_stack.append(self.token)
        return self

    def __exit__(self, *exc):
        _scope_stack.pop()
        return False


def style_token(owner, style: torch.Tensor, extra=()):
    """-> (token, shared): ``token`` is stable while the caller keeps passing the same tensor object (unmodified) and ``extra``;
    ``shared`` says that all batch rows of ``style`` are equal (one video, one style): an expanded (stride-0) tensor is
    recognised for free, a materialised ``repeat`` by one device comparison when the object is first seen."""
    st = owner.__dict__.get("_vt_style_state")
    key = (style._version, tuple(style.shape), tuple(style.stride()), style.data_ptr(), tuple(extra), _precision, _weights_epoch)
    if st is not None and st[0] is style and st[1] == key:
        return st[2], st[3]
    if style.shape[0] == 1 or style.stride(0) == 0:
        shared = True
    else:
        shared = bool((style == style[:1]).all().item())       # one synchronising check per new style object
    tok = next(_token_counter)
    owner.__dict__["_vt_style_state"] = (style, key, tok, shared)
    return tok, shared


def style_cached(owner, name: str, fn, extra=None):
    """memoise ``fn()`` on ``owner`` under the current style scope (recomputed when the token / ``extra`` / precision change)"""
    tok = _scope_stack[-1] if _scope_stack else None
    if tok is None:
        return fn()
    key = (tok, extra, _precision)
    cache = owner.__dict__.setdefault("_vt_style_cache", {})
    hit = cache.get(name)
    if hit is not None and hit[0] == key:
        return hit[1]
    val = fn()
    cache[name] = (key, val)
    return val


class nvtx_range:
    """NVTX range around a stage / layer when ``set_option("nvtx", True)`` (or VT_NVTX=1): names the launches of a stage for
    ``ncu --nvtx --nvtx-include "<name>/"`` and for timeline tools; free when disabled."""

    def __init__(self, name: str):
        self.name = name
        self.on = _options["nvtx"]

    def __enter__(self):
        if self.on:
            torch.cuda.nvtx.range_push(self.name)
        return self

    def __exit__(self, *exc):
        if self.on:
            torch.cuda.nvtx.range_pop()
        return False


def _round_flag() -> int:
    return 1 if _precision == "tf32" else 0


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _req_cuda(*ts):
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.VtError("vtoonify_b200 ops need CUDA tensors: there is no CPU fallback "
                               "(use the reference's op_cpu or oracle/ for CPU)")
        if t.dtype != torch.float32:
            raise _lib.VtError(f"vtoonify_b200 ops are fp32 I/O (got {t.dtype})")


def _ptr(t):
    return None if t is None else t.data_ptr()


# ----------------------------------------------------------------------------------------------
# layout
# ----------------------------------------------------------------------------------------------
def is_channels_last_view(x: torch.Tensor) -> bool:
    """True if logical-NCHW ``x`` is physically NHWC-contiguous."""
    if x.dim() != 4:
        return False
    B, C, H, W = x.shape
    return x.stride() == (H * W * C, 1, W * C, C) or (B == 1 and x.stride()[1:] == (1, W * C, C))


def to_nhwc(x: torch.Tensor, c_pad: Optional[int] = None, round_tf32: Optional[bool] = None) -> torch.Tensor:
    """NCHW (any strides) -> NHWC ``[B,H,W,c_pad]`` with zero-filled pad channels."""
    _req_cuda(x)
    B, C, H, W = x.shape
    c_pad = C if c_pad is None else c_pad
    if c_pad == C and is_channels_last_view(x):
        return x.permute(0, 2, 3, 1)
    x = x.contiguous()
    out = torch.empty((B, H, W, c_pad), device=x.device, dtype=torch.float32)
    rt = _round_flag() if round_tf32 is None else int(round_tf32)
    check(_lib.load().vt_nchw_to_nhwc_f32(x.data_ptr(), out.data_ptr(), B, C, H, W, c_pad, rt, _stream()))
    return out


def to_nchw(x: torch.Tensor, C: Optional[int] = None) -> torch.Tensor:
    """NHWC ``[B,H,W,Cs]`` -> contiguous NCHW ``[B,C,H,W]`` (first C channels)."""
    _req_cuda(x)
    B, H, W, Cs = x.shape
    C = Cs if C is None else C
    out = torch.empty((B, C, H, W), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_nhwc_to_nchw_f32(x.data_ptr(), out.data_ptr(), B, C, H, W, Cs, _stream()))
    return out


def nhwc_as_nchw_view(x: torch.Tensor) -> torch.Tensor:
    """Zero-copy: NHWC tensor seen as a logical NCHW (channels_last) tensor."""
    return x.permute(0, 3, 1, 2)


# ----------------------------------------------------------------------------------------------
# a1 / a2: the reference's two custom ops (planar NCHW API)
# ----------------------------------------------------------------------------------------------
def upfirdn2d_planar(x: torch.Tensor, kernel: torch.Tensor, up: Tuple[int, int], down: Tuple[int, int],
                     pad: Tuple[int, int, int, int]) -> torch.Tensor:
    _req_cuda(x, kernel)
    B, C, H, W = x.shape
    kh, kw = kernel.shape
    lib = _lib.load()
    oh, ow = _lib.c_int(), _lib.c_int()
    check(lib.vt_upfirdn2d_out_size(H, W, kh, kw, up[0], up[1], down[0], down[1], pad[0], pad[1], pad[2], pad[3], oh, ow))
    if oh.value < 1 or ow.value < 1:
        raise _lib.VtError(f"upfirdn2d: empty output {oh.value}x{ow.value}")
    x = x.contiguous()
    kernel = kernel.contiguous()
    out = torch.empty((B, C, oh.value, ow.value), device=x.device, dtype=torch.float32)
    check(lib.vt_upfirdn2d_f32(x.data_ptr(), kernel.data_ptr(), out.data_ptr(), B * C, H, W, kh, kw, up[0], up[1],
                               down[0], down[1], pad[0], pad[1], pad[2], pad[3], _stream()))
    return out


def fused_bias_act(x: torch.Tensor, bias: Optional[torch.Tensor], negative_slope: float, scale: float) -> torch.Tensor:
    _req_cuda(x, bias)
    x = x.contiguous()
    out = torch.empty_like(x)
    n = x.numel()
    if bias is not None:
        if x.dim() < 2 or bias.dim() != 1 or bias.shape[0] != x.shape[1]:
            raise _lib.VtError(f"fused_leaky_relu: bias {tuple(bias.shape)} does not match dim 1 of {tuple(x.shape)}")
        step_b = 1
        for s in x.shape[2:]:
            step_b *= s
        bias = bias.contiguous()
        check(_lib.load().vt_fused_bias_act_f32(x.data_ptr(), bias.data_ptr(), out.data_ptr(), n, step_b, x.shape[1],
                                                negative_slope, scale, _stream()))
    else:
        check(_lib.load().vt_fused_bias_act_f32(x.data_ptr(), None, out.data_ptr(), n, 1, 1, negative_slope, scale, _stream()))
    return out


def fused_bias_act_grad(grad: torch.Tensor, ref_out: torch.Tensor, negative_slope: float, scale: float,
                        bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """backward of :func:`fused_bias_act` w.r.t. its input: ``(ref_out > 0 ? g : g * slope) * scale`` with ``g = grad (+ bias[c])``
    (op/fused_act.py:20-53; ``bias`` is the second backward's ``gradgrad_bias``)"""
    _req_cuda(grad, ref_out, bias)
    grad, ref_out = grad.contiguous(), ref_out.contiguous()
    if grad.shape != ref_out.shape:
        raise _lib.VtError("fused_bias_act_grad: grad and the forward output must have the same shape")
    out = torch.empty_like(grad)
    step_b = 1
    for s in grad.shape[2:]:
        step_b *= s
    check(_lib.load().vt_fused_bias_act_grad_f32(grad.data_ptr(), _ptr(None if bias is None else bias.contiguous()), ref_out.data_ptr(),
                                                 out.data_ptr(), grad.numel(), step_b, grad.shape[1] if grad.dim() > 1 else 1,
                                                 negative_slope, scale, _stream()))
    return out


def channel_sum(x: torch.Tensor) -> torch.Tensor:
    """``x.sum(dim=[0, 2, 3, ...])`` of a contiguous ``[B, C, ...]`` tensor (deterministic two-stage reduction)"""
    _req_cuda(x)
    x = x.contiguous()
    B, C = x.shape[0], x.shape[1]
    inner = x.numel() // (B * C)
    lib = _lib.load()
    ws = torch.empty((lib.vt_channel_sum_ws_floats(C),), device=x.device, dtype=torch.float32)
    out = torch.empty((C,), device=x.device, dtype=torch.float32)
    check(lib.vt_channel_sum_f32(x.data_ptr(), out.data_ptr(), ws.data_ptr(), B, C, inner, _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# small dense layers
# ----------------------------------------------------------------------------------------------
def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], w_scale: float = 1.0,
           b_scale: float = 1.0, act: int = 0) -> torch.Tensor:
    """``act``: 0 none, 1 fused_leaky_relu (0.2, *sqrt2), 2 LeakyReLU(0.2), 3 ReLU, 4 sigmoid."""
    if weight.dim() != 2 or x.dim() < 1 or weight.shape[1] != x.shape[-1]:
        raise _lib.VtError(f"linear: weight {tuple(weight.shape)} does not match input {tuple(x.shape)}: "
                           "it must be [out_dim, in_dim] with in_dim the last dim of the input")
    if bias is not None and bias.numel() != weight.shape[0]:
        raise _lib.VtError(f"linear: bias has {bias.numel()} elements, out_dim is {weight.shape[0]}")
    _req_cuda(x, weight, bias)
    shp = x.shape
    x2 = x.reshape(-1, shp[-1]).contiguous()
    out = torch.empty((x2.shape[0], weight.shape[0]), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_linear_f32(x2.data_ptr(), weight.contiguous().data_ptr(), _ptr(None if bias is None else bias.contiguous()),
                                    out.data_ptr(), x2.shape[0], x2.shape[1], weight.shape[0], w_scale, b_scale, act, _stream()))
    return out.reshape(*shp[:-1], weight.shape[0])


def pixelnorm(x: torch.Tensor) -> torch.Tensor:
    _req_cuda(x)
    x2 = x.reshape(-1, x.shape[-1]).contiguous()
    out = torch.empty_like(x2)
    check(_lib.load().vt_pixelnorm_f32(x2.data_ptr(), out.data_ptr(), x2.shape[0], x2.shape[1], _stream()))
    return out.reshape(x.shape)


# ----------------------------------------------------------------------------------------------
# a3: weights
# ----------------------------------------------------------------------------------------------
def _pad32(c: int) -> int:
    return (c + 31) // 32 * 32


def prep_weights(W: torch.Tensor, style: Optional[torch.Tensor] = None, scale: float = 1.0, demodulate: bool = False,
                 cin_pad: Optional[int] = None, round_tf32: Optional[bool] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``W`` [Cout,Cin,kh,kw] (+ optional per-sample ``style`` [B,Cin]) -> conv-kernel layout
    ``[wB, kh*kw, Cout, cin_pad]`` = (scale*W)*style*demod (model/stylegan/model.py:259-267)."""
    if W.dim() != 4:
        raise _lib.VtError(f"prep_weights: W must be [Cout, Cin, kh, kw] (got {tuple(W.shape)})")
    if style is not None and (style.dim() != 2 or style.shape[1] != W.shape[1]):
        raise _lib.VtError(f"prep_weights: style {tuple(style.shape)} must be [wB, Cin] with Cin = {W.shape[1]}")
    _req_cuda(W, style)
    Cout, Cin, kh, kw = W.shape
    cin_pad = _pad32(Cin) if cin_pad is None else cin_pad
    wB = 1 if style is None else style.shape[0]
    if out is None:
        out = torch.empty((wB, kh * kw, Cout, cin_pad), device=W.device, dtype=torch.float32)
    elif tuple(out.shape) != (wB, kh * kw, Cout, cin_pad) or not out.is_contiguous() or out.dtype != torch.float32:
        raise _lib.VtError("prep_weights: bad out tensor")
    check(_lib.load().vt_modulate_weights_f32(W.contiguous().data_ptr(), _ptr(None if style is None else style.contiguous()),
                                              out.data_ptr(), wB, Cout, Cin, kh, kw, cin_pad, float(scale),
                                              int(demodulate), _round_flag() if round_tf32 is None else int(round_tf32),
                                              _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# convolution
# ----------------------------------------------------------------------------------------------
def conv_taps(k: int, padding: int, dilation: int = 1):
    """(dy, dx, weight-slab) of a k x k cross-correlation with zero padding."""
    return [(ky * dilation - padding, kx * dilation - padding, ky * k + kx) for ky in range(k) for kx in range(k)]


def conv2d_nhwc(srcs: Sequence[torch.Tensor], weight: torch.Tensor, taps, stride: int, Ho: int, Wo: int,
                out: Optional[torch.Tensor] = None, out_view: Optional[Tuple[int, int, int, int]] = None,
                src_c: Optional[Sequence[int]] = None, phase_offs: Optional[Sequence[int]] = None,
                bias: Optional[torch.Tensor] = None, noise: Optional[torch.Tensor] = None,
                noise_w: Optional[torch.Tensor] = None, act: int = ACT_NONE, slope: float = 0.2, gain: float = 1.0,
                res: Optional[torch.Tensor] = None, alpha: float = 1.0, beta: float = 1.0,
                precision: Optional[str] = None, rgb: Optional[dict] = None,
                slope_vec: Optional[torch.Tensor] = None, src_scale: Optional[Sequence] = None,
                src_affine: Optional[Sequence] = None, want_stats: bool = False, stats_eps: float = 1e-5) -> torch.Tensor:
    """General NHWC convolution (virtual channel-concat of ``srcs``).

    ``want_stats``: also return the instance-norm statistics ``[B, Cout, 2]`` = (mean, rstd) of the OUTPUT (what
    :func:`instnorm_stats` would compute from it): the tensor-core kernel's epilogue warps write per-tile centred partials of the values
    they store and only the finalize pass runs afterwards; other routes fall back to the separate statistics pass.

    ``weight``: ``[wB, w_taps, Cout, w_cstride]`` from :func:`prep_weights`.
    ``out_view``: (offset_elems, sb, sy, sx) strided view into ``out`` (used for polyphase transposed conv).
    ``phase_offs``: 4 element offsets -> one launch computes 4 output phases: ``weight`` rows are phase-major
    ``[n_phase * Cout]`` per tap and phase ``ph`` is stored through the strided view ``out_view`` shifted by ``phase_offs[ph]``.
    """
    prec = precision or _precision
    B, H, W, _ = srcs[0].shape
    wB, w_taps, Cout, w_cs = weight.shape
    if phase_offs is not None:
        Cout //= len(phase_offs)          # weight rows are phase-major [n_phase * Cout]
    _req_cuda(weight, bias, noise, noise_w, res, *srcs)
    d = ConvDesc()
    d.struct_size = _lib.ctypes.sizeof(ConvDesc)
    d.n_src = len(srcs)
    for i, s in enumerate(srcs):
        if not s.is_contiguous() or s.shape[:3] != (B, H, W):
            raise _lib.VtError("conv2d_nhwc: sources must be contiguous NHWC with equal B,H,W")
        d.src[i] = s.data_ptr()
        d.src_c[i] = s.shape[3] if src_c is None else src_c[i]
        d.src_cstride[i] = s.shape[3]
    d.B, d.H, d.W, d.Ho, d.Wo = B, H, W, Ho, Wo
    d.stride = stride
    d.taps = len(taps)
    for t, tap in enumerate(taps):
        d.tap_dy[t], d.tap_dx[t], d.tap_w[t] = tap[0], tap[1], tap[2]
    d.n_phase = 1 if phase_offs is None else len(phase_offs)
    d.weight = weight.data_ptr()
    d.wB, d.w_taps, d.w_cstride, d.Cout = wB, w_taps, w_cs, Cout
    # rgb["only"]: the caller has no use for the activation (last generator layer) -> a kernel that supports it gets out = NULL
    # and only produces the image; every other route allocates the activation as usual and drops it on return
    rgb_only = rgb is not None and bool(rgb.get("only")) and out is None and out_view is None
    if out is None:
        out = torch.empty((B, Ho, Wo, Cout), device=srcs[0].device, dtype=torch.float32) if not rgb_only else None
    if rgb_only:
        off, sb, sy, sx = 0, Ho * Wo * Cout, Wo * Cout, Cout
    elif out_view is None:
        off, sb, sy, sx = 0, Ho * Wo * Cout, Wo * Cout, Cout
        if out.shape != (B, Ho, Wo, Cout) or not out.is_contiguous():
            raise _lib.VtError("conv2d_nhwc: bad out tensor")
    else:
        off, sb, sy, sx = out_view
    d.out = out.data_ptr() if out is not None else None
    d.out_cpitch = out.shape[-1] if out is not None else Cout
    if phase_offs is None:
        d.phase_off[0] = off
    else:
        for i, po in enumerate(phase_offs):
            d.phase_off[i] = off + po
    d.out_sb, d.out_sy, d.out_sx = sb, sy, sx
    d.bias = _ptr(bias)
    d.noise = _ptr(noise)
    d.noise_w = _ptr(noise_w)
    d.act, d.slope, d.gain = act, slope, gain
    if slope_vec is not None:
        _req_cuda(slope_vec)
        d.slope_vec = slope_vec.contiguous().data_ptr()
    if res is not None:
        if out_view is not None or res.shape != (B, Ho, Wo, Cout) or not res.is_contiguous():
            raise _lib.VtError("conv2d_nhwc: residual must match a dense output")
        d.res = res.data_ptr()
    d.alpha, d.beta = alpha, beta
    d.round_tf32 = _round_flag()
    rgb_out = None
    if rgb is not None:
        # fused ToRGB tail: rgb = {"w": [wB,3,Cout] or [wB,1,3,Cout], "bias": [3], "skip": [B,3,Ho/2,Wo/2] or None, "kernel": [4,4]}
        # with wB the conv weight's: the kernels read them by raw pointer, "w" as a dense [wB][3][Cout]
        _req_cuda(rgb["w"], rgb["bias"], rgb.get("skip"), rgb.get("kernel"))
        rw, rb, skip, kern = rgb["w"], rgb["bias"], rgb.get("skip"), rgb.get("kernel")
        if tuple(rw.shape) not in ((wB, 3, Cout), (wB, 1, 3, Cout)) or not rw.is_contiguous() or rw.dtype != torch.float32:
            raise _lib.VtError(f"conv2d_nhwc: rgb['w'] must be a contiguous float32 [wB, 3, Cout] = [{wB}, 3, {Cout}] tensor "
                               f"(got {rw.dtype} {tuple(rw.shape)}{'' if rw.is_contiguous() else ', not contiguous'})")
        if rb.numel() != 3 or not rb.is_contiguous() or rb.dtype != torch.float32:
            raise _lib.VtError("conv2d_nhwc: rgb['bias'] must be a contiguous float32 tensor of 3 elements")
        if skip is not None:
            if tuple(skip.shape) != (B, 3, Ho // 2, Wo // 2) or 2 * (Ho // 2) != Ho or 2 * (Wo // 2) != Wo or skip.dtype != torch.float32:
                raise _lib.VtError(f"conv2d_nhwc: rgb['skip'] must be a float32 [B, 3, Ho/2, Wo/2] = [{B}, 3, {Ho / 2:g}, {Wo / 2:g}] "
                                   f"tensor (got {tuple(skip.shape)})")
            if kern is None or tuple(kern.shape) != (4, 4) or kern.dtype != torch.float32:
                raise _lib.VtError("conv2d_nhwc: rgb['kernel'] must be a float32 4x4 up-sampling kernel when rgb['skip'] is given")
        rgb_out = torch.empty((B, 3, Ho, Wo), device=srcs[0].device, dtype=torch.float32)
        d.rgb_w, d.rgb_bias, d.rgb_out = rgb["w"].data_ptr(), rgb["bias"].data_ptr(), rgb_out.data_ptr()
        if rgb.get("skip") is not None:
            d.rgb_skip, d.rgb_skip_kernel = rgb["skip"].contiguous().data_ptr(), rgb["kernel"].contiguous().data_ptr()
    if src_scale is not None:
        # per-pixel planar [B,H,W] multiplier of a source (bf16x3 tensor-core mode only; see scale_fusable)
        for i, sc in enumerate(src_scale):
            if sc is not None:
                _req_cuda(sc)
                if sc.numel() != B * H * W or not sc.is_contiguous():
                    raise _lib.VtError("conv2d_nhwc: src_scale must be a contiguous [B,H,W] map")
                d.src_scale[i] = sc.data_ptr()
    if src_affine is not None:
        # per-(sample, channel) (scale, shift) table [B, C_i, 2] of a source (AdaIN applied inside the conv; bf16x3 mode only)
        for i, af in enumerate(src_affine):
            if af is not None:
                _req_cuda(af)
                if tuple(af.shape) != (B, int(d.src_c[i]), 2) or not af.is_contiguous():
                    raise _lib.VtError("conv2d_nhwc: src_affine must be a contiguous [B, C, 2] table")
                d.src_affine[i] = af.data_ptr()
    lib = _lib.load()
    if prec == "bf16x3":
        d.weight_bf16x3 = weight.data_ptr()   # marks the mode for the *_supported checks; the split buffer is attached below
    # full-resolution small-channel 3x3 layer: the row-strip entry point (the only route that takes an image-only ToRGB launch)
    rs = (prec == "bf16x3" and _options["rs_conv"] and W >= _options["rs_min_width"] and len(srcs) == 1 and phase_offs is None
          and stride == 1 and len(taps) == 9 and res is None and slope_vec is None and src_scale is None and src_affine is None
          and Cout in (32, 64) and int(d.src_c[0]) in (32, 64) and w_cs == int(d.src_c[0]) and alpha == 1.0
          and act in (ACT_NONE, ACT_LRELU) and bool(lib.vt_conv2d_rs_supported(d)))
    if out is None and not rs:
        out = torch.empty((B, Ho, Wo, Cout), device=srcs[0].device, dtype=torch.float32)
        d.out = out.data_ptr()
    use_tc = rs or (prec in ("tf32", "bf16x3") and lib.vt_conv2d_tc_supported(d))
    d.weight_bf16x3 = None
    if use_tc and prec == "bf16x3":
        # Cout == 32: the N-stacked form needs 4 instead of 6 MMA instructions per tap (and keeps all four hi/lo products) but
        # twice the accumulator columns; off by default.  The row-strip kernel (conv_rs_kernel) reads exactly this form for Cout == 32
        # (its 64 weight rows are the MMA's M), so the rs route gets it with the bf16 split; a launch that also writes instance-norm
        # statistics is one conv_rs_kernel does not take and keeps the plain split
        nstack = Cout == 32 and phase_offs is None and (bool(_options["bf16x3_nstack"]) or
                                                        (rs and _options["rs_fmt"] == "bf16" and not want_stats))
        if _options["rs_fmt"] == "f16" and not nstack:
            d.weight_bf16x3 = split_weights_f16x3(weight).data_ptr()
            d.split_fmt, d.acc_scale = 1, 1.0 / F16_WEIGHT_SCALE
        else:
            d.weight_bf16x3 = split_weights_bf16x3(weight, nstack).data_ptr()
            d.bf16x3_nstack = 1 if nstack else 0
    stats = stats_ws = None
    if want_stats:
        if rgb is not None or out_view is not None or phase_offs is not None:
            raise _lib.VtError("conv2d_nhwc: want_stats needs a dense single-phase output without the fused ToRGB tail")
        chunks = lib.vt_conv2d_tc_stats_chunks(d) if (use_tc and _options["fuse_stats"]) else -1
        if chunks > 0:
            stats_ws = torch.empty((lib.vt_instnorm_partials_floats(chunks, B, Cout),), device=out.device, dtype=torch.float32)
            d.stats_ws, d.stats_ws_floats = stats_ws.data_ptr(), stats_ws.numel()
    if use_tc:
        if _tc_profile is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            cin = sum(int(d.src_c[i]) for i in range(d.n_src))
            flops = 2.0 * B * Ho * Wo * Cout * cin * len(taps)   # algorithmic (the folded up-conv issues 4x this)
            nbytes = 4.0 * (B * H * W * cin + B * Ho * Wo * Cout * d.n_phase + weight.numel())
            e0.record()
            check(lib.vt_conv2d_rs(d, 0.0, _stream()) if rs else lib.vt_conv2d_tc_tf32(d, _stream()))
            e1.record()
            # MMA flops actually issued: 3 bf16 products per algorithmic product in the split-operand mode, and the folded
            # up-convolution evaluates all 4 output phases with full 3x3 support (4x the transposed conv's algorithmic MACs)
            issued = flops * (3.0 if prec == "bf16x3" else 1.0) * (4.0 if d.n_phase == 4 else 1.0)
            _tc_profile.append((e0, e1, flops, nbytes, f"{cin}->{Cout}{'x4up' if d.n_phase > 1 else ''} k{len(taps)} s{stride} {H}x{W}", issued))
        else:
            check(lib.vt_conv2d_rs(d, 0.0, _stream()) if rs else lib.vt_conv2d_tc_tf32(d, _stream()))
    else:
        check(lib.vt_conv2d_direct_f32(d, _stream()))
    if want_stats:
        if stats_ws is not None:
            stats = torch.empty((B, Cout, 2), device=out.device, dtype=torch.float32)
            check(lib.vt_instnorm_finalize_f32(stats_ws.data_ptr(), stats.data_ptr(), B, Cout, chunks, Ho * Wo, stats_eps, _stream()))
        else:
            stats = instnorm_stats(out, eps=stats_eps)
        return out, stats
    return out if rgb is None else (out, rgb_out)


def split_weights_bf16x3(weight: torch.Tensor, nstack: bool = False) -> torch.Tensor:
    """``weight`` (from :func:`prep_weights` / :func:`fold_upconv_weights`, unrounded fp32, channel stride % 32 == 0) ->
    buffer whose 32-channel chunks hold ``[bf16(w) | bf16(w - bf16(w))]``; ``nstack`` (Cout == 32): per tap 32 rows ``[hi|hi]``
    then 32 rows ``[lo|lo]`` (twice the rows). Cached on the tensor object, so cached plain-conv weights are split once;
    per-frame modulated weights are split per call (one tiny launch)."""
    ver = weight._version
    cached = getattr(weight, "_vt_bf16x3", None)
    if cached is not None and cached[0] == ver and cached[1] == weight.data_ptr() and cached[3] == nstack:
        return cached[2]
    if weight.shape[-1] % 32 != 0 or not weight.is_contiguous():
        raise _lib.VtError("split_weights_bf16x3: weight channel stride must be a multiple of 32")
    rows = weight.numel() // weight.shape[-1]
    nrows = weight.shape[-2] if nstack else 0
    out = torch.empty((2 * rows if nstack else rows, weight.shape[-1]), device=weight.device, dtype=torch.float32)
    check(_lib.load().vt_split_weights_bf16x3(weight.data_ptr(), out.data_ptr(), rows, weight.shape[-1], nrows, _stream()))
    weight._vt_bf16x3 = (ver, weight.data_ptr(), out, nstack)
    return out


def split_weights_f16x3(weight: torch.Tensor) -> torch.Tensor:
    """fp16 counterpart of :func:`split_weights_bf16x3`: chunks hold ``[half(w * 256) | half(w * 256 - hi)]``; cached on the tensor."""
    ver = weight._version
    cached = getattr(weight, "_vt_f16x3", None)
    if cached is not None and cached[0] == ver and cached[1] == weight.data_ptr():
        return cached[2]
    if weight.shape[-1] % 32 != 0 or not weight.is_contiguous():
        raise _lib.VtError("split_weights_f16x3: weight channel stride must be a multiple of 32")
    rows = weight.numel() // weight.shape[-1]
    out = torch.empty((rows, weight.shape[-1]), device=weight.device, dtype=torch.float32)
    check(_lib.load().vt_split_weights_f16x3(weight.data_ptr(), out.data_ptr(), rows, weight.shape[-1], F16_WEIGHT_SCALE, _stream()))
    weight._vt_f16x3 = (ver, weight.data_ptr(), out)
    return out


def affine_fusable(precision: Optional[str] = None) -> bool:
    """conv2d_nhwc(src_affine=...) is available and enabled (AdaIN applied by the operand-transform warps)."""
    return (precision or _precision) == "bf16x3" and _options["fuse_adain"]


def scale_fusable(precision: Optional[str] = None) -> bool:
    """conv2d_nhwc(src_scale=...) is available (the split-operand tensor-core mode applies it while converting tiles)."""
    return (precision or _precision) == "bf16x3" and _options["fuse_mask_mul"]


def rgb_fusable(Cout: int, precision: Optional[str] = None) -> bool:
    """The ToRGB tail can ride in the conv epilogue when one N tile (at most 128 channels) holds all channels (tensor-core path only)."""
    return (precision or _precision) in ("tf32", "bf16x3") and Cout % 32 == 0 and Cout <= 128 and (Cout & (Cout - 1)) == 0 and _options["fuse_torgb"]


def conv_out_size(n: int, k: int, stride: int, padding: int, dilation: int) -> int:
    return (n + 2 * padding - dilation * (k - 1) - 1) // stride + 1


def conv_transpose2d_s2_k3_nhwc(x: torch.Tensor, weight: torch.Tensor, precision: Optional[str] = None) -> torch.Tensor:
    """F.conv_transpose2d(x, w, stride=2, padding=0) with a 3x3 kernel as 4 polyphase convolutions
    (model/stylegan/model.py:273-283).  ``weight`` in prep layout with slab index ky*3+kx of the (un-flipped)
    W[cout, cin, ky, kx].  out[2i+ky, 2j+kx] += x[i,j] * W[:, :, ky, kx]  ->  [B, 2H+1, 2W+1, Cout]."""
    B, H, W, _ = x.shape
    Cout = weight.shape[2]
    Hf, Wf = 2 * H + 1, 2 * W + 1
    out = torch.empty((B, Hf, Wf, Cout), device=x.device, dtype=torch.float32)
    for py in (0, 1):
        for px in (0, 1):
            taps = []
            for ky in range(py, 3, 2):
                for kx in range(px, 3, 2):
                    taps.append((-(ky - py) // 2, -(kx - px) // 2, ky * 3 + kx))
            Ho = H + 1 if py == 0 else H
            Wo = W + 1 if px == 0 else W
            view = ((py * Wf + px) * Cout, Hf * Wf * Cout, 2 * Wf * Cout, 2 * Cout)
            conv2d_nhwc([x], weight, taps, 1, Ho, Wo, out=out, out_view=view, precision=precision)
    return out


def conv_wgrad_nhwc(a: torch.Tensor, s: torch.Tensor, M: int, N: int, taps, stride: int, per_sample: bool) -> torch.Tensor:
    """Weight gradient ``out[m, n, t] = sum_{b, p} a[b, p, m] * s[b, stride * p + (dy_t, dx_t), n]`` (zero outside ``s``) on the
    wgmma weight-gradient kernel (bf16x3 arithmetic whatever :func:`set_precision` says).  ``a``, ``s``: contiguous NHWC with channel
    strides that are multiples of 32 (:func:`to_nhwc` with ``c_pad``); ``taps``: [(dy, dx)].  Returns ``[nb * M, N, len(taps)]``,
    nb = B when ``per_sample`` else 1.  Deterministic: the same inputs give bit-identical results."""
    _req_cuda(a, s)
    B, Ha, Wa, ca = a.shape
    Bs, Hs, Ws, cs = s.shape
    if Bs != B or not a.is_contiguous() or not s.is_contiguous():
        raise _lib.VtError("conv_wgrad_nhwc: a and s must be contiguous NHWC tensors with the same batch")
    d = _lib.ConvWgradDesc()
    d.struct_size = _lib.ctypes.sizeof(_lib.ConvWgradDesc)
    d.B, d.per_sample, d.stride = B, int(per_sample), stride
    d.a, d.a_h, d.a_w, d.M, d.a_cstride = a.data_ptr(), Ha, Wa, M, ca
    d.s, d.s_h, d.s_w, d.N, d.s_cstride = s.data_ptr(), Hs, Ws, N, cs
    d.taps = len(taps)
    if d.taps > _lib.VT_MAX_TAPS:
        raise _lib.VtError(f"conv_wgrad_nhwc: at most {_lib.VT_MAX_TAPS} taps")
    for t, (dy, dx) in enumerate(taps):
        d.tap_dy[t], d.tap_dx[t] = dy, dx
    lib = _lib.load()
    n_ws = lib.vt_conv2d_wgrad_ws_floats(d)
    if n_ws < 0:
        check(1)
    out = torch.empty(((B if per_sample else 1) * M, N, len(taps)), device=a.device, dtype=torch.float32)
    ws = torch.empty((n_ws,), device=a.device, dtype=torch.float32) if n_ws > 0 else None
    d.out = out.data_ptr()
    if ws is not None:
        d.ws, d.ws_floats = ws.data_ptr(), n_ws
    check(lib.vt_conv2d_wgrad(d, _stream()))
    return out


def fold_upconv_weights(w: torch.Tensor, blur_kernel: torch.Tensor) -> torch.Tensor:
    """[wB, 9, Cout, cpad] modulated weights (un-rounded) + 4x4 blur -> [wB, 9, 4*Cout, cpad]: per tap the 4 phase kernels
    stacked along the GEMM N dimension."""
    _req_cuda(w, blur_kernel)
    wB, nine, Cout, cpad = w.shape
    if nine != 9 or tuple(blur_kernel.shape) != (4, 4):
        raise _lib.VtError("fold_upconv_weights: needs 3x3 weights and a 4x4 blur kernel")
    out = torch.empty((wB, 9, 4 * Cout, cpad), device=w.device, dtype=torch.float32)
    check(_lib.load().vt_fold_upconv_weights_f32(w.data_ptr(), blur_kernel.contiguous().data_ptr(), out.data_ptr(), wB, Cout,
                                                 cpad, _round_flag(), _stream()))
    return out


_UP2_TAPS = [(dy, dx, (dy + 1) * 3 + (dx + 1)) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]


def conv_up2_folded_nhwc(x: torch.Tensor, w_folded: torch.Tensor, bias=None, noise=None, noise_w=None, act: int = ACT_NONE,
                         slope: float = 0.2, gain: float = 1.0, precision: Optional[str] = None) -> torch.Tensor:
    """Blur(conv_transpose2d(x, w, stride 2)) as ONE 3x3 convolution with N = 4*Cout (the 4 output phases stacked along
    the GEMM N dimension); the (2H+1)x(2W+1) intermediate of model/stylegan/model.py:281-285 never exists.
    Output [B, 2H, 2W, Cout] with the StyledConv tail (noise, bias, leaky relu) in the epilogue."""
    B, H, W, _ = x.shape
    Cout = w_folded.shape[2] // 4
    Hf, Wf = 2 * H, 2 * W
    out = torch.empty((B, Hf, Wf, Cout), device=x.device, dtype=torch.float32)
    view = (0, Hf * Wf * Cout, 2 * Wf * Cout, 2 * Cout)
    offs = [(ry * Wf + rx) * Cout for ry in (0, 1) for rx in (0, 1)]
    conv2d_nhwc([x], w_folded, _UP2_TAPS, 1, H, W, out=out, out_view=view, phase_offs=offs, bias=bias, noise=noise,
                noise_w=noise_w, act=act, slope=slope, gain=gain, precision=precision)
    return out


def rsu_eligible(cin: int, cout: int, W: int, kernel: torch.Tensor, pad, precision: Optional[str] = None) -> bool:
    return ((precision or _precision) == "bf16x3" and _options["rsu_conv"] and cin % 32 == 0 and 32 <= cin <= _options["rsu_max_cin"]
            and cout % 32 == 0 and 32 <= cout <= 128 and W >= _options["rs_min_width"] and tuple(pad) == (1, 1)
            and tuple(kernel.shape) == (4, 4))


def conv_up2_rs_nhwc(x: torch.Tensor, w9: torch.Tensor, blur_kernel: torch.Tensor, bias=None, noise=None, noise_w=None,
                     act: int = ACT_NONE, slope: float = 0.2, gain: float = 1.0) -> torch.Tensor:
    """Blur(conv_transpose2d(x, w, stride 2)) for the full-resolution up-convolutions.  ``w9``: modulated weights ``[wB, 9, Cout, Cin]``
    (un-rounded fp32, slab ky*3+kx).  The blur is folded into the 4 output-phase kernels (cached on the tensor object) and the layer
    runs as one wgmma convolution with N = 4 * Cout (:func:`conv_up2_folded_nhwc`)."""
    _req_cuda(x, w9, bias, noise, noise_w)
    cached = getattr(w9, "_vt_rsu", None)
    if cached is not None and cached[0] == w9._version and cached[1] == w9.data_ptr() and cached[2] is blur_kernel:
        wf = cached[3]
    else:
        wf = fold_upconv_weights(w9, blur_kernel)
        w9._vt_rsu = (w9._version, w9.data_ptr(), blur_kernel, wf)
    return conv_up2_folded_nhwc(x, wf, bias=bias, noise=noise, noise_w=noise_w, act=act, slope=slope, gain=gain)


def fir_nhwc(x: torch.Tensor, kernel: torch.Tensor, pad: Tuple[int, int], bias: Optional[torch.Tensor] = None,
             noise: Optional[torch.Tensor] = None, noise_w: Optional[torch.Tensor] = None, act: bool = False,
             slope: float = 0.2, gain: float = SQRT2) -> torch.Tensor:
    _req_cuda(x, kernel, bias, noise, noise_w)
    B, H, W, C = x.shape
    kh, kw = kernel.shape
    Ho, Wo = H + pad[0] + pad[1] - kh + 1, W + pad[0] + pad[1] - kw + 1
    out = torch.empty((B, Ho, Wo, C), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_fir_nhwc_f32(x.data_ptr(), kernel.contiguous().data_ptr(), out.data_ptr(), B, H, W, C, kh, kw,
                                      pad[0], pad[1], _ptr(bias), _ptr(noise), _ptr(noise_w), int(act), slope, gain,
                                      _round_flag(), _stream()))
    return out


def smalln_conv(src: Optional[torch.Tensor], weight: Optional[torch.Tensor], taps, Cout: int, B: int, H: int, W: int,
                planar: Optional[torch.Tensor] = None, planar_weight: Optional[torch.Tensor] = None,
                bias: Optional[torch.Tensor] = None, act: int = ACT_NONE, skip: Optional[torch.Tensor] = None,
                skip_kernel: Optional[torch.Tensor] = None, mul_src: Optional[torch.Tensor] = None,
                src2: Optional[torch.Tensor] = None, tap_const: Optional[torch.Tensor] = None,
                src_mask: Optional[torch.Tensor] = None, tsum: Optional[torch.Tensor] = None):
    """Cout<=4 convolution with planar NCHW output ``[B,Cout,H,W]``; optionally also returns ``mul_src * out[:,0]``.
    ``src2``: the input is the virtual concat ``[src | abs(src - src2)]`` (weight rows hold 2*C channels);
    ``tap_const`` ``[wB, w_taps, Cout]``: constant added for every in-bounds tap (folded AdaIN affine)."""
    _req_cuda(src, weight, planar, planar_weight, bias, skip, skip_kernel, mul_src, src2, tap_const, tsum)
    dev = next(t for t in (src, planar, tsum) if t is not None).device
    d = SmallNDesc()
    d.struct_size = _lib.ctypes.sizeof(SmallNDesc)
    if planar is not None:
        planar = planar.contiguous()
        d.n_planar = planar.shape[1]
        d.planar = planar.data_ptr()
        d.planar_weight = planar_weight.contiguous().data_ptr()
    if src is not None:
        d.src = src.data_ptr()
        d.src_c = src.shape[3]
        d.src_cstride = src.shape[3]
        d.weight = weight.data_ptr()
        d.wB, d.w_taps, _, d.w_cstride = weight.shape
        if src2 is not None:
            if src2.shape != src.shape or not src2.is_contiguous():
                raise _lib.VtError("smalln_conv: src2 must match src")
            d.src2, d.src2_mode = src2.data_ptr(), 1
        if tap_const is not None:
            d.tap_const = tap_const.contiguous().data_ptr()
        if src_mask is not None:
            _req_cuda(src_mask)
            if src_mask.numel() != B * H * W or not src_mask.is_contiguous():
                raise _lib.VtError("smalln_conv: src_mask must be a contiguous [B,H,W] map")
            d.src_mask = src_mask.data_ptr()
    else:
        d.wB, d.w_taps = 1, (planar_weight.shape[0] if planar_weight is not None else len(taps))
    if tsum is not None:
        # NHWC [B,H,W,Ct] per-tap partial products from a 1x1 tensor-core convolution (rows t*Cout + n)
        if tsum.shape[:3] != (B, H, W) or not tsum.is_contiguous() or tsum.shape[3] < len(taps) * Cout:
            raise _lib.VtError("smalln_conv: bad tsum tensor")
        d.tsum, d.tsum_c = tsum.data_ptr(), tsum.shape[3]
    d.Cout = Cout
    d.B, d.H, d.W = B, H, W
    d.taps = len(taps)
    for t, (dy, dx, tw) in enumerate(taps):
        d.tap_dy[t], d.tap_dx[t], d.tap_w[t] = dy, dx, tw
    d.bias = _ptr(bias)
    d.act = act
    if skip is not None:
        skip = skip.contiguous()
        d.skip = skip.data_ptr()
        d.skip_kernel = skip_kernel.contiguous().data_ptr()
    out = torch.empty((B, Cout, H, W), device=dev, dtype=torch.float32)
    d.out = out.data_ptr()
    mul_out = None
    if mul_src is not None:
        mul_out = torch.empty_like(mul_src)
        d.mul_out, d.mul_src, d.mul_c = mul_out.data_ptr(), mul_src.data_ptr(), mul_src.shape[3]
    d.round_tf32 = _round_flag()
    check(_lib.load().vt_smalln_conv_f32(d, _stream()))
    return (out, mul_out) if mul_src is not None else out


# ----------------------------------------------------------------------------------------------
# a7: AdaIN
# ----------------------------------------------------------------------------------------------
def instnorm_stats(x: torch.Tensor, x2: Optional[torch.Tensor] = None, eps: float = 1e-5) -> torch.Tensor:
    """Per-(b,c) (mean, rstd) of ``x`` (or of cat(x, |x - x2|) when ``x2`` is given)."""
    _req_cuda(x, x2)
    B, H, W, C = x.shape
    mode = 0 if x2 is None else 1
    Cs = C * (2 if mode else 1)
    stats = torch.empty((B, Cs, 2), device=x.device, dtype=torch.float32)
    nbytes = _lib.load().vt_instnorm_ws_bytes(B, H * W, C, mode)
    if nbytes < 0:
        raise _lib.VtError(f"instnorm_stats: unsupported shape C={C}")
    ws = torch.empty((nbytes // 4,), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_instnorm_stats_nhwc(x.data_ptr(), _ptr(x2), mode, B, H * W, C, C, eps, stats.data_ptr(),
                                             ws.data_ptr(), _stream()))
    return stats


def adain_affine(stats: torch.Tensor, gamma_beta: torch.Tensor) -> torch.Tensor:
    """AdaIN as a per-(sample, channel) affine table ``[B, Cs, 2]`` = (gamma*rstd, beta - gamma*mean*rstd) for
    ``conv2d_nhwc(src_affine=...)`` (model/dualstylegan.py:16-21 applied inside the consuming convolution)."""
    _req_cuda(stats, gamma_beta)
    B, Cs, _ = stats.shape
    out = torch.empty((B, Cs, 2), device=stats.device, dtype=torch.float32)
    check(_lib.load().vt_adain_affine_f32(stats.contiguous().data_ptr(), gamma_beta.contiguous().data_ptr(), out.data_ptr(), B, Cs,
                                          _stream()))
    return out


def adain_apply(x: torch.Tensor, stats: torch.Tensor, gamma_beta: torch.Tensor, x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req_cuda(x, x2, stats, gamma_beta)
    B, H, W, C = x.shape
    mode = 0 if x2 is None else 1
    Cs = C * (2 if mode else 1)
    out = torch.empty((B, H, W, Cs), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_adain_apply_nhwc(x.data_ptr(), _ptr(x2), mode, B, H * W, C, C, stats.data_ptr(),
                                          gamma_beta.contiguous().data_ptr(), out.data_ptr(), _round_flag(), _stream()))
    return out


def _grad_ws(B: int, HW: int, C: int, device) -> torch.Tensor:
    nbytes = _lib.load().vt_act_grad_ws_bytes(B, HW, C)
    if nbytes < 0:
        raise _lib.VtError(f"act_grad: unsupported shape C={C}")
    return torch.empty((nbytes // 8,), device=device, dtype=torch.float64)


def _nhwc_check(name, ref, *ts):
    for t in ts:
        if t is not None and (t.shape != ref.shape or not t.is_contiguous()):
            raise _lib.VtError(f"{name}: tensors must be contiguous NHWC of the same shape")


def adain_grad_stats(g: torch.Tensor, x: torch.Tensor, stats: torch.Tensor) -> torch.Tensor:
    """Reduction half of the instance-norm backward: ``[B, C, 2]`` = (sum of g, sum of g * xhat) per plane, xhat = (x - mean) * rstd
    with the statistics ``stats`` [B, C, 2] the forward applied (deterministic, double-precision reduction)."""
    _req_cuda(g, x, stats)
    _nhwc_check("adain_grad_stats", g, g, x)
    B, H, W, C = g.shape
    if tuple(stats.shape) != (B, C, 2) or not stats.is_contiguous():
        raise _lib.VtError("adain_grad_stats: stats must be a contiguous [B, C, 2] table")
    sums = torch.empty((B, C, 2), device=g.device, dtype=torch.float32)
    check(_lib.load().vt_adain_grad_stats_nhwc(g.data_ptr(), x.data_ptr(), stats.data_ptr(), B, H * W, C, sums.data_ptr(),
                                               _grad_ws(B, H * W, C, g.device).data_ptr(), _stream()))
    return sums


def act_grad(g: torch.Tensor, ref: Optional[torch.Tensor] = None, slope: float = 0.2, gain: float = 1.0,
             res: Optional[torch.Tensor] = None, beta: float = 1.0, adain: Optional[Tuple] = None, bias_grad: bool = False):
    """Backward of an activation (and optionally of the AdaIN in front of it) on NHWC tensors:
    ``out = beta * res + gate(ref) * gain * T(g)``, gate(ref) = ref > 0 ? 1 : slope (``ref``: the LeakyReLU's own output),
    T(g) = g, or with ``adain = (x, stats, gamma_beta, sums)`` the instance-norm + affine backward
    ``gamma * rstd * ((g - m_g) - (x - mean) * rstd * m_gx)`` (``sums`` from :func:`adain_grad_stats`).
    ``bias_grad``: also return the per-channel sum of ``out`` ([C]), reduced in the same pass."""
    x, stats, gb, sums = adain if adain is not None else (None, None, None, None)
    _req_cuda(g, ref, res, x, stats, gb, sums)
    _nhwc_check("act_grad", g, g, ref, res, x)
    B, H, W, C = g.shape
    if adain is not None:
        if tuple(stats.shape) != (B, C, 2) or tuple(sums.shape) != (B, C, 2) or tuple(gb.shape) != (B, 2 * C):
            raise _lib.VtError("act_grad: AdaIN tables must be stats/sums [B, C, 2] and gamma_beta [B, 2C]")
        stats, gb, sums = stats.contiguous(), gb.contiguous(), sums.contiguous()
    out = torch.empty_like(g)
    bg = torch.empty((C,), device=g.device, dtype=torch.float32) if bias_grad else None
    ws = _grad_ws(B, H * W, C, g.device) if bias_grad else None
    check(_lib.load().vt_act_grad_nhwc(g.data_ptr(), _ptr(ref), slope, gain, _ptr(res), beta, _ptr(x), _ptr(stats), _ptr(gb),
                                       _ptr(sums), B, H * W, C, out.data_ptr(), _ptr(bg), _ptr(ws), _stream()))
    return (out, bg) if bias_grad else out


def channel_sum_nhwc(g: torch.Tensor) -> torch.Tensor:
    """Per-channel sum ``[C]`` of a contiguous NHWC ``[B, H, W, C]`` tensor (a bias gradient): the reduction of :func:`act_grad`
    without its elementwise output (deterministic, double-precision partials)."""
    _req_cuda(g)
    _nhwc_check("channel_sum_nhwc", g, g)
    B, H, W, C = g.shape
    bg = torch.empty((C,), device=g.device, dtype=torch.float32)
    check(_lib.load().vt_act_grad_nhwc(g.data_ptr(), None, 0.2, 1.0, None, 1.0, None, None, None, None, B, H * W, C, None,
                                       bg.data_ptr(), _grad_ws(B, H * W, C, g.device).data_ptr(), _stream()))
    return bg


def mbstd(x: torch.Tensor, group: int) -> torch.Tensor:
    """Minibatch standard deviation of the StyleGAN discriminator (model/vtoonify.py:67-75) on NHWC ``x`` [B, H, W, C]:
    ``[B, H, W, pad32(C + 1)]`` holding x, then the statistic of the sample's column ``b % (B / group)``, then zeros."""
    _req_cuda(x)
    B, H, W, C = x.shape
    if B % group:
        raise _lib.VtError(f"mbstd: batch {B} is not a multiple of the group size {group}")
    x = x.contiguous()
    out = torch.empty((B, H, W, _pad32(C + 1)), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_mbstd_nhwc_f32(x.data_ptr(), out.data_ptr(), B, group, H * W, C, out.shape[3], _stream()))
    return out


def mbstd_grad(g: torch.Tensor, x: torch.Tensor, group: int) -> torch.Tensor:
    """Backward of :func:`mbstd`: ``g`` [B, H, W, c_pad] (gradient of its output), ``x`` its input -> gradient of ``x``."""
    _req_cuda(g, x)
    B, H, W, C = x.shape
    if B % group:
        raise _lib.VtError(f"mbstd_grad: batch {B} is not a multiple of the group size {group}")
    if g.shape[:3] != x.shape[:3]:
        raise _lib.VtError("mbstd_grad: g and x must have the same batch and map size")
    g, x = g.contiguous(), x.contiguous()
    out = torch.empty_like(x)
    check(_lib.load().vt_mbstd_grad_nhwc_f32(g.data_ptr(), x.data_ptr(), out.data_ptr(), B, group, H * W, C, g.shape[3], _stream()))
    return out


def torgb_gate_grad(g: Optional[torch.Tensor], g_rgb: torch.Tensor, w_rgb: torch.Tensor, ref: torch.Tensor, slope: float = 0.2,
                    gain: float = SQRT2) -> torch.Tensor:
    """Backward of a StyledConv whose activation ``ref`` (NHWC [B, H, W, C]) also feeds a 1x1 ToRGB: ``gate(ref) * gain * (g +
    w_rgb[b]^T g_rgb)``.  ``g``: the activation's other gradient (None: 0); ``g_rgb``: the planar image gradient [B, 3, H, W], read
    as it is; ``w_rgb``: ToRGB's modulated weights [wB, 1, 3, c] (c >= C)."""
    _req_cuda(g, g_rgb, w_rgb, ref)
    _nhwc_check("torgb_gate_grad", ref, g, ref)
    B, H, W, C = ref.shape
    if tuple(g_rgb.shape) != (B, 3, H, W) or w_rgb.dim() != 4 or tuple(w_rgb.shape[1:3]) != (1, 3) or w_rgb.shape[0] not in (1, B):
        raise _lib.VtError("torgb_gate_grad: g_rgb must be [B, 3, H, W] and w_rgb [1 or B, 1, 3, c]")
    w_rgb, g_rgb = w_rgb.contiguous(), g_rgb.contiguous()
    out = torch.empty_like(ref)
    check(_lib.load().vt_torgb_gate_grad_nhwc(_ptr(g), g_rgb.data_ptr(), w_rgb.data_ptr(), w_rgb.shape[0], w_rgb.shape[3],
                                              ref.data_ptr(), slope, gain, B, H * W, C, out.data_ptr(), _stream()))
    return out


def fusion_mask_grad(g_p: torch.Tensor, f_e: torch.Tensor, m: torch.Tensor, g_m: Optional[torch.Tensor] = None):
    """Fusion's mask head ``m = tanh(relu z)`` read by ``f_E * m``: ``g_p`` (gradient of ``f_E * m``), ``f_e`` NHWC [B, H, W, C],
    ``m`` and ``g_m`` (the returned mask's own gradient, may be None) planar [B, 1, H, W] -> (g_z [B, 1, H, W], conv2's bias gradient [1])."""
    _req_cuda(g_p, f_e, m, g_m)
    _nhwc_check("fusion_mask_grad", f_e, g_p, f_e)
    B, H, W, C = f_e.shape
    for t in (m, g_m):
        if t is not None and (t.numel() != B * H * W or not t.is_contiguous()):
            raise _lib.VtError("fusion_mask_grad: m and g_m must be contiguous [B, 1, H, W] maps")
    lib = _lib.load()
    ws = torch.empty((lib.vt_fusion_mask_grad_ws_bytes(B, H * W) // 8,), device=f_e.device, dtype=torch.float64)
    g_z = torch.empty((B, 1, H, W), device=f_e.device, dtype=torch.float32)
    db = torch.empty((1,), device=f_e.device, dtype=torch.float32)
    check(lib.vt_fusion_mask_grad_nhwc(g_p.data_ptr(), f_e.data_ptr(), m.data_ptr(), _ptr(g_m), B, H * W, C, g_z.data_ptr(),
                                       db.data_ptr(), ws.data_ptr(), _stream()))
    return g_z, db


def _fusion_check(name, g_z, w2, f_g, f_e, stats):
    _nhwc_check(name, f_g, f_g, f_e)
    B, H, W, C = f_g.shape
    if (tuple(g_z.shape) != (B, 1, H, W) or not g_z.is_contiguous() or tuple(w2.shape) != (9, 2 * C) or not w2.is_contiguous()
            or tuple(stats.shape) != (B, 2 * C, 2) or not stats.is_contiguous()):
        raise _lib.VtError(f"{name}: g_z must be [B, 1, H, W], w2 [9, 2C] and stats [B, 2C, 2], contiguous")
    return B, H, W, C


def fusion_adain_grad_stats(g_z: torch.Tensor, w2: torch.Tensor, f_g: torch.Tensor, f_e: torch.Tensor, stats: torch.Tensor) -> torch.Tensor:
    """AdaIN-backward sums of Fusion's mask head over the virtual concat ``cat(f_G, |f_G - f_E|)``: ``[B, 2C, 2]`` = (sum of u, sum of
    u * ahat) per plane, u = conv2's input gradient (its transposed 3x3 of ``g_z``, recomputed per pixel), ``w2`` = conv2's weight as
    ``[9, 2C]`` (tap-major).  The two sums are also dbeta and dgamma of the affine."""
    _req_cuda(g_z, w2, f_g, f_e, stats)
    B, H, W, C = _fusion_check("fusion_adain_grad_stats", g_z, w2, f_g, f_e, stats)
    sums = torch.empty((B, 2 * C, 2), device=f_g.device, dtype=torch.float32)
    check(_lib.load().vt_fusion_adain_grad_stats_nhwc(g_z.data_ptr(), w2.data_ptr(), f_g.data_ptr(), f_e.data_ptr(), stats.data_ptr(),
                                                      B, H, W, C, sums.data_ptr(), _grad_ws(B, H * W, 2 * C, f_g.device).data_ptr(),
                                                      _stream()))
    return sums


def fusion_input_grad(g_z: torch.Tensor, w2: torch.Tensor, f_g: torch.Tensor, f_e: torch.Tensor, stats: torch.Tensor,
                      gamma_beta: torch.Tensor, sums: torch.Tensor, g_dir: Optional[torch.Tensor], g_p: torch.Tensor, m: torch.Tensor):
    """-> (g_{f_G}, g_{f_E}) of Fusion's mask head: the AdaIN backward of both concat halves (``sums`` from
    :func:`fusion_adain_grad_stats`, ``gamma_beta`` [B, 4C]), the ``|f_G - f_E|`` split (sign(0) = 0), ``g_dir`` (f_G's gradient from
    the fusion convolution, may be None) and ``g_p * m`` (``g_p``: gradient of ``f_E * m``)."""
    _req_cuda(g_z, w2, f_g, f_e, stats, gamma_beta, sums, g_dir, g_p, m)
    B, H, W, C = _fusion_check("fusion_input_grad", g_z, w2, f_g, f_e, stats)
    _nhwc_check("fusion_input_grad", f_g, g_dir, g_p)
    if tuple(gamma_beta.shape) != (B, 4 * C) or tuple(sums.shape) != (B, 2 * C, 2) or m.numel() != B * H * W or not m.is_contiguous():
        raise _lib.VtError("fusion_input_grad: gamma_beta must be [B, 4C], sums [B, 2C, 2] and m [B, 1, H, W]")
    g_fg, g_fe = torch.empty_like(f_g), torch.empty_like(f_e)
    check(_lib.load().vt_fusion_input_grad_nhwc(g_z.data_ptr(), w2.data_ptr(), f_g.data_ptr(), f_e.data_ptr(), stats.data_ptr(),
                                                gamma_beta.contiguous().data_ptr(), sums.contiguous().data_ptr(), _ptr(g_dir),
                                                g_p.data_ptr(), m.data_ptr(), B, H, W, C, g_fg.data_ptr(), g_fe.data_ptr(), _stream()))
    return g_fg, g_fe


def affine_fold_weights(w: torch.Tensor, stats: torch.Tensor, gamma_beta: torch.Tensor):
    """Fold AdaIN's per-(b,c) affine into conv weights ``w`` [1, taps, N, C2] -> (w' [B, taps, N, C2], k [B, taps, N])."""
    _req_cuda(w, stats, gamma_beta)
    _, taps, N, C2 = w.shape
    B = stats.shape[0]
    out_w = torch.empty((B, taps, N, C2), device=w.device, dtype=torch.float32)
    out_k = torch.empty((B, taps, N), device=w.device, dtype=torch.float32)
    check(_lib.load().vt_affine_fold_weights_f32(w.data_ptr(), stats.data_ptr(), gamma_beta.contiguous().data_ptr(),
                                                 out_w.data_ptr(), out_k.data_ptr(), B, taps * N, C2, _stream()))
    return out_w, out_k


def gate_shortcut_add(x: torch.Tensor, gate: Optional[torch.Tensor], sc: torch.Tensor, sc_stride: int = 1) -> torch.Tensor:
    """``x * gate[b,c] + sc[b, y*s, x*s, c]`` (SE gate and residual shortcut; a MaxPool2d(1, s) shortcut is the strided read)."""
    if x.dim() != 4 or sc.dim() != 4 or not x.is_contiguous() or not sc.is_contiguous():
        raise _lib.VtError(f"gate_shortcut_add: x {tuple(x.shape)} and sc {tuple(sc.shape)} must be contiguous NHWC tensors")
    B, H, W, C = x.shape
    if sc.shape[0] != B or sc.shape[3] != C:
        raise _lib.VtError(f"gate_shortcut_add: sc {tuple(sc.shape)} does not match the batch and channels of x {tuple(x.shape)}")
    if gate is not None and (gate.shape[0] != B or gate.numel() != B * C):
        raise _lib.VtError(f"gate_shortcut_add: gate {tuple(gate.shape)} must hold [B, C] = [{B}, {C}] values")
    _req_cuda(x, gate, sc)
    out = torch.empty_like(x)
    check(_lib.load().vt_gate_shortcut_add_nhwc(x.data_ptr(), _ptr(None if gate is None else gate.contiguous()), sc.data_ptr(),
                                                out.data_ptr(), B, H, W, C, sc.shape[1], sc.shape[2], sc_stride, _round_flag(), _stream()))
    return out


def bilinear_add(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """``F.interpolate(x, size=y.shape[1:3], mode='bilinear', align_corners=True) + y`` on NHWC tensors."""
    if x.dim() != 4 or y.dim() != 4 or not x.is_contiguous() or not y.is_contiguous():
        raise _lib.VtError(f"bilinear_add: x {tuple(x.shape)} and y {tuple(y.shape)} must be contiguous NHWC tensors")
    if x.shape[0] != y.shape[0] or x.shape[3] != y.shape[3]:
        raise _lib.VtError(f"bilinear_add: x {tuple(x.shape)} and y {tuple(y.shape)} differ in batch or channels")
    _req_cuda(x, y)
    B, h, w, C = x.shape
    _, H, W, _ = y.shape
    out = torch.empty_like(y)
    check(_lib.load().vt_bilinear_add_nhwc(x.data_ptr(), y.data_ptr(), out.data_ptr(), B, h, w, H, W, C, _round_flag(), _stream()))
    return out


def axpby(a: torch.Tensor, b: Optional[torch.Tensor], sa: float, sb: float = 0.0, round_tf32: Optional[bool] = None,
          out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out = a * sa + b * sb`` elementwise over ``a.numel()`` elements (``b`` None: ``a * sa``)."""
    if b is not None and b.numel() != a.numel():
        raise _lib.VtError(f"axpby: b has {b.numel()} elements, a has {a.numel()}")
    _req_cuda(a, b, out)
    if not a.is_contiguous() or (b is not None and not b.is_contiguous()):
        a, b = a.contiguous(), (None if b is None else b.contiguous())
    if out is None:
        out = torch.empty_like(a)
    elif out.numel() != a.numel() or not out.is_contiguous():
        raise _lib.VtError("axpby: out must be contiguous with as many elements as a")
    rt = _round_flag() if round_tf32 is None else int(round_tf32)
    check(_lib.load().vt_axpby_f32(a.data_ptr(), _ptr(b), out.data_ptr(), a.numel(), sa, sb, rt, _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# a11: frame transforms
# ----------------------------------------------------------------------------------------------
def frames_u8_to_f32(frames: torch.Tensor, out: Optional[torch.Tensor] = None, swap_rb: bool = False) -> torch.Tensor:
    """uint8 ``[B,H,W,3]`` -> fp32 ``[B,3,H,W]`` in [-1,1] (ToTensor + Normalize(0.5,0.5))."""
    if not frames.is_cuda or frames.dtype != torch.uint8:
        raise _lib.VtError("frames_u8_to_f32 needs a CUDA uint8 tensor")
    B, H, W, _ = frames.shape
    if out is None:
        out = torch.empty((B, 3, H, W), device=frames.device, dtype=torch.float32)
    check(_lib.load().vt_frame_u8_to_f32(frames.contiguous().data_ptr(), out.data_ptr(), B, H, W, int(swap_rb),
                                         out.stride(0), _stream()))
    return out


def f32_to_frames_u8(img: torch.Tensor, swap_rb: bool = True) -> torch.Tensor:
    """fp32 ``[B,3,H,W]`` -> clamp(-1,1) -> uint8 ``[B,H,W,3]`` (util.tensor2cv2 semantics, RGB->BGR by default)."""
    _req_cuda(img)
    B, _, H, W = img.shape
    out = torch.empty((B, H, W, 3), device=img.device, dtype=torch.uint8)
    check(_lib.load().vt_f32_to_frame_u8(img.contiguous().data_ptr(), out.data_ptr(), B, H, W, int(swap_rb), _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# f3: pre-filter + resize of high-resolution frames (style_transfer.py:124-130, 151-156), bit-exact with OpenCV
# ----------------------------------------------------------------------------------------------
def resize_tables(src: int, dst: int, clamp_weights: bool):
    """The (offset, weight0, weight1) int32 table cv::resize(INTER_LINEAR, 8-bit) builds for one axis: source coordinate in float
    like OpenCV, cvFloor, weights cvRound(w * 2048).  Columns (``clamp_weights``): out-of-range neighbours get unit weight on the
    border pixel; rows: the weights stay fractional and the row index is clamped by the kernel."""
    import numpy as np
    scale = np.float64(src) / np.float64(dst)
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_weights:
        lo, hi = s < 0, s >= src - 1
        f = np.where(lo | hi, np.float32(0), f).astype(np.float32)
        s = np.where(lo, 0, np.where(hi, src - 1, s))
    w1 = np.rint(f * np.float32(2048)).astype(np.int32)
    w0 = np.rint((np.float32(1.0) - f) * np.float32(2048)).astype(np.int32)
    return np.stack([s.astype(np.int32), w0, w1], axis=0)


_resize_table_cache = {}


def frame_prefilter_resize(frames: torch.Tensor, n_blur: int, size: Tuple[int, int],
                           crop: Optional[Tuple[int, int, int, int]] = None) -> torch.Tensor:
    """uint8 ``[B,H,W,3]`` frames -> ``cv2.resize(blur^n(frame), size)[top:bottom, left:right]`` on the device, bit-exact with
    the reference's CPU pre-processing (``size`` = (w, h) like cv2; ``crop`` = (top, bottom, left, right))."""
    if not frames.is_cuda or frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
        raise _lib.VtError("frame_prefilter_resize needs a CUDA uint8 [B,H,W,3] tensor")
    if n_blur not in (0, 1, 2):
        raise _lib.VtError("frame_prefilter_resize: the frame loop applies the blur 0, 1 or 2 times")
    frames = frames.contiguous()
    B, H, W, _ = frames.shape
    lib = _lib.load()
    cur = frames
    for _ in range(n_blur):
        nxt = torch.empty_like(cur)
        check(lib.vt_frame_blur4_u8(cur.data_ptr(), nxt.data_ptr(), B, H, W, _stream()))
        cur = nxt
    dw, dh = int(size[0]), int(size[1])
    top, bottom, left, right = (0, dh, 0, dw) if crop is None else (int(c) for c in crop)
    key = (H, W, dh, dw, frames.device)
    tabs = _resize_table_cache.get(key)
    if tabs is None:
        tabs = (torch.from_numpy(resize_tables(W, dw, True)).to(frames.device).contiguous(),
                torch.from_numpy(resize_tables(H, dh, False)).to(frames.device).contiguous())
        _resize_table_cache[key] = tabs
    out = torch.empty((B, bottom - top, right - left, 3), device=frames.device, dtype=torch.uint8)
    check(lib.vt_frame_resize_crop_u8(cur.data_ptr(), out.data_ptr(), B, H, W, dh, dw, top, left, bottom - top, right - left,
                                      tabs[0].data_ptr(), tabs[1].data_ptr(), _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# face-parsing pre-network helpers (model/bisenet/model.py, style_transfer.py:171-174)
# ----------------------------------------------------------------------------------------------
def frame_s2d(x: torch.Tensor, upsample2: bool, cpad: int = 32) -> torch.Tensor:
    """planar ``[B,3,H,W]`` -> NHWC space-to-depth tensor ``[B, ceil(XH/2), ceil(XW/2), cpad]`` of X = x (or of
    ``2 * bilinear_up2(x)``), the input of the stride-2 7x7 stem run as a 4x4 stride-1 convolution."""
    _req_cuda(x)
    x = x.contiguous()
    B, C, H, W = x.shape
    if C != 3:
        raise _lib.VtError("frame_s2d: expected 3 planar channels")
    XH, XW = (2 * H, 2 * W) if upsample2 else (H, W)
    out = torch.empty((B, (XH + 1) // 2, (XW + 1) // 2, cpad), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_frame_s2d_f32(x.data_ptr(), out.data_ptr(), B, H, W, out.shape[1], out.shape[2], cpad, int(bool(upsample2)),
                                       _stream()))
    return out


def maxpool3x3s2(x: torch.Tensor) -> torch.Tensor:
    _req_cuda(x)
    B, H, W, C = x.shape
    out = torch.empty((B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_maxpool3x3s2_nhwc_f32(x.contiguous().data_ptr(), out.data_ptr(), B, H, W, C, _stream()))
    return out


def maxpool2x2(x: torch.Tensor) -> torch.Tensor:
    """``nn.MaxPool2d(2, 2)`` on NHWC ``[B, H, W, C]`` -> ``[B, H // 2, W // 2, C]`` (bit-identical to torch's)."""
    _req_cuda(x)
    B, H, W, C = x.shape
    out = torch.empty((B, H // 2, W // 2, C), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_maxpool2x2_nhwc_f32(x.contiguous().data_ptr(), out.data_ptr(), B, H, W, C, _stream()))
    return out


def maxpool2x2_grad(g: torch.Tensor, x: torch.Tensor, add: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Adjoint of :func:`maxpool2x2`: ``g`` [B, H // 2, W // 2, C] goes to the first maximal element of each window of the pool input
    ``x`` in row-major order (torch's tie rule); ``add`` (``x``'s shape, may be None) is added to the result."""
    _req_cuda(g, x, add)
    _nhwc_check("maxpool2x2_grad", x, x, add)
    B, H, W, C = x.shape
    if tuple(g.shape) != (B, H // 2, W // 2, C) or not g.is_contiguous():
        raise _lib.VtError(f"maxpool2x2_grad: g {tuple(g.shape)} must be contiguous [B, H // 2, W // 2, C] of x {tuple(x.shape)}")
    out = torch.empty_like(x)
    check(_lib.load().vt_maxpool2x2_grad_nhwc_f32(g.data_ptr(), x.data_ptr(), _ptr(add), out.data_ptr(), B, H, W, C, _stream()))
    return out


def lpips_head(taps: Sequence[torch.Tensor], lin_w: Sequence[torch.Tensor]) -> torch.Tensor:
    """LPIPS head over NHWC taps ``[2B, h_k, w_k, C_k]`` (rows ``b`` and ``B + b`` are the two images of pair ``b``) with the ``lin``
    weights ``[C_k]`` -> ``[B]``: the sum over the taps of the spatial mean of ``sum_c w_c (u0_c - u1_c)^2``, u = f / (||f|| + 1e-10).
    Deterministic: reruns are bit-identical."""
    if len(taps) != len(lin_w) or not taps:
        raise _lib.VtError("lpips_head: one lin weight per tap")
    _req_cuda(*taps, *lin_w)
    B2 = taps[0].shape[0]
    if B2 % 2:
        raise _lib.VtError("lpips_head: taps must hold 2B rows")
    for t, w in zip(taps, lin_w):
        if t.dim() != 4 or t.shape[0] != B2 or not t.is_contiguous() or w.numel() != t.shape[3] or not w.is_contiguous():
            raise _lib.VtError("lpips_head: taps must be contiguous NHWC [2B, h, w, C] with contiguous [C] weights")
    n, B = len(taps), B2 // 2
    hw = (_lib.c_int64 * n)(*[t.shape[1] * t.shape[2] for t in taps])
    cs = (_lib.c_int * n)(*[t.shape[3] for t in taps])
    fp = (_lib.c_void_p * n)(*[t.data_ptr() for t in taps])
    wp = (_lib.c_void_p * n)(*[w.data_ptr() for w in lin_w])
    lib = _lib.load()
    nbytes = lib.vt_lpips_head_ws_bytes(B, n, hw)
    if nbytes < 0:
        raise _lib.VtError("lpips_head: bad tap shapes")
    ws = torch.empty((nbytes // 8,), device=taps[0].device, dtype=torch.float64)
    out = torch.empty((B,), device=taps[0].device, dtype=torch.float32)
    check(lib.vt_lpips_head_nhwc(n, fp, wp, hw, cs, B, out.data_ptr(), ws.data_ptr(), _stream()))
    return out


def lpips_head_grad(tap: torch.Tensor, lin_w: torch.Tensor, g_b: torch.Tensor, target: bool, pred: bool):
    """Gradient of :func:`lpips_head` for one tap ``[2B, h, w, C]``, scaled by ``g_b`` [B] (the loss gradient per sample) -> NHWC
    ``[nb * B, h, w, C]``: the target rows (0..B-1) then the pred rows (B..2B-1) of whichever of the two are asked for."""
    _req_cuda(tap, lin_w, g_b)
    B2, h, w, C = tap.shape
    B = B2 // 2
    if B2 % 2 or not tap.is_contiguous() or lin_w.numel() != C or g_b.numel() != B or not (target or pred):
        raise _lib.VtError("lpips_head_grad: tap must be contiguous [2B, h, w, C], lin_w [C] and g_b [B]; ask for a side")
    out = torch.empty(((int(target) + int(pred)) * B, h, w, C), device=tap.device, dtype=torch.float32)
    gt = out[:B] if target else None
    gp = out[B:] if (target and pred) else (out if pred else None)
    check(_lib.load().vt_lpips_head_grad_nhwc(tap.data_ptr(), lin_w.contiguous().data_ptr(), g_b.contiguous().data_ptr(), B, h * w, C,
                                              _ptr(gt), _ptr(gp), _stream()))
    return out


def resize_nearest(x: torch.Tensor, H: int, W: int) -> torch.Tensor:
    _req_cuda(x)
    B, h, w, C = x.shape
    out = torch.empty((B, H, W, C), device=x.device, dtype=torch.float32)
    check(_lib.load().vt_resize_nearest_nhwc_f32(x.contiguous().data_ptr(), out.data_ptr(), B, h, w, H, W, C, _stream()))
    return out


def logits_readout(logits: torch.Tensor, n_classes: int, Hf: int, Wf: int, step: int = 1, scale: float = 1.0,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """NHWC logits ``[B,h,w,Cs]`` -> planar ``[B,n_classes,ceil(Hf/step),ceil(Wf/step)]``: every ``step``-th pixel of the
    ``align_corners=True`` bilinear up-sampling to ``(Hf, Wf)``.  ``out``: optional channel slice ``t[:, c0:c0+n_classes]`` of a
    contiguous planar tensor (written in place)."""
    _req_cuda(logits)
    B, h, w, Cs = logits.shape
    Ho, Wo = (Hf + step - 1) // step, (Wf + step - 1) // step
    if out is None:
        out = torch.empty((B, n_classes, Ho, Wo), device=logits.device, dtype=torch.float32)
    elif tuple(out.shape) != (B, n_classes, Ho, Wo) or out.dtype != torch.float32 or out.stride()[1:] != (Ho * Wo, Wo, 1):
        raise _lib.VtError("logits_readout: out must be a [B,n_classes,Ho,Wo] channel slice of a contiguous planar tensor")
    check(_lib.load().vt_logits_readout_f32(logits.contiguous().data_ptr(), out.data_ptr(), B, h, w, Cs, n_classes, Hf, Wf, Ho, Wo,
                                            step, float(scale), out.stride(0), _stream()))
    return out
