"""conv_tc (csrc/conv_tc.cu) against a float64 reference, instantiation by instantiation and plan knob by plan knob.

Every case of TABLE names the kernel instantiation the planner (conv_tc_run) must pick for it, and the test checks that name
in a torch.profiler trace: together the cases reach every entry of kTcKernels, which test_table_reaches_every_instantiation
reads from the source.  Each case runs one conv2d_nhwc descriptor with a bundle of epilogue features and is compared, element
by element, with the same operation evaluated by F.conv2d in float64.  The error bar of an element is c_mode times the float64
sum of the absolute values of every term that went into it (the same conv of |x| with |w|, plus |bias|, |noise|, ...), so it
scales with what the element sums instead of one max-abs tolerance per layer.

The kernel names come from one child process that runs the table under torch.profiler: traces taken in a process that has
already run many profiler sessions (the rest of the suite) can come back without their kernels.

The knob sweep sets each vt_set_option key of the planner and checks that the result still meets the bar and that it is
bit-identical to the default plan: whatever the staging (halo boxes or one box per tap, taps per weight box, pipeline stage
counts, M tiles per work item, work-item order, transposed view, wide or ping-pong items), every output element gets the same
k16 (or k8) MMA products of the same operands in the same order and the same epilogue arithmetic.

Outputs are written into NaN-filled buffers with guard regions, so an element the kernel does not write, or a write outside the
output, fails the test.
"""
import contextlib
import math
import json
import os
import re
import subprocess
import sys
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

torch.set_grad_enabled(False)
gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONV_TC_SRC = os.path.join(ROOT, "vtoonify_b200", "csrc", "conv_tc.cu")
ACT_NONE, ACT_LRELU, ACT_RELU_TANH = 0, 1, 2

# ---- error model ----------------------------------------------------------------------------------------------------
# bar = (C_OP[mode] + sqrt(K) * 2^-24) * terms + EPI * |ref|, K = input channels x taps.
#   C_OP is the operand rounding: the estimates were tf32 about 2^-11 on each operand (2^-10 per product), the bf16 split
#   (a_lo * w_lo dropped, lo parts rounded) about 2^-16 and the fp16 split about 2^-21; sqrt(K) * 2^-24 is the fp32
#   accumulation over K.  Measured on an H100 (80 GB HBM3, 700 W) over this file's cases, the worst err / terms was 7.6e-4
#   (tf32, K = 32), 4.7e-6 (bf16 split, K = 32) and 8.8e-7 (fp16 split, K = 864, where the accumulation term dominates);
#   the constants below put the bar at about twice that.  Every case prints its worst err / bar (run with -s).
#   EPI covers the fp32 epilogue (bias and noise adds, tanhf, the residual blend).
C_OP = {"tf32": 1.5e-3, "bf16": 2.0 ** -17, "f16": 2.0 ** -23}
EPI = 2.0 ** -22

OPS = {   # operand mode -> (set_precision, split_fmt, bf16x3_nstack option)
    "tf32": ("tf32", "bf16", False),
    "bf16": ("bf16x3", "bf16", False),
    "f16": ("bf16x3", "f16", False),
    "nstack": ("bf16x3", "bf16", True),
}
OP_ENUM = {"tf32": 0, "bf16": 1, "f16": 2, "nstack": 3}
KERNEL_RE = re.compile(r"conv_tc(?:_pingpong)?_kernel<\d+, \d+, \d+>")
GUARD = 1024            # floats of guard region before and after every output buffer
GUARD_VALUE = 1234.5


def kname(nw, mt, op, pp=False):
    return f"conv_tc{'_pingpong' if pp else ''}_kernel<{nw}, {mt}, {OP_ENUM[op] if isinstance(op, str) else op}>"


def ktc_kernels():
    """kernel names of the kTcKernels entries of csrc/conv_tc.cu (constants and the TcOp enum resolved from the same source)"""
    src = open(CONV_TC_SRC).read()
    consts = {m.group(1): int(m.group(2)) for m in re.finditer(r"constexpr int (\w+) = (\d+);", src)}
    enum = re.search(r"enum TcOp : int \{(.*?)\};", src, re.S).group(1)
    consts.update({m.group(1): int(m.group(2)) for m in re.finditer(r"(OP_\w+) = (\d+)", enum)})
    val = lambda s: int(s) if s.isdigit() else consts[s]
    macro = re.search(r"#define VT_TC_OPS\(NW, MT\)(.*?)\n(?!\s)", src, re.S).group(1)
    macro_ops = re.findall(r"\{NW, MT, (OP_\w+), (true|false)", macro)
    table = re.search(r"const TcKernel kTcKernels\[\] = \{(.*?)\n\};", src, re.S).group(1)
    names = []
    for nw, mt in re.findall(r"VT_TC_OPS\((\w+), (\w+)\)", table):
        names += [kname(val(nw), val(mt), consts[op], pp == "true") for op, pp in macro_ops]
    for nw, mt, op, pp in re.findall(r"\{(\w+), (\w+), (OP_\w+), (true|false),", table):
        names.append(kname(val(nw), val(mt), consts[op], pp == "true"))
    return names


# ---- the case table ---------------------------------------------------------------------------------------------------
# Epilogue features: bias, noise, lrelu (scalar slope), slope_vec (per-channel slope, the PReLU of pSp), tanh (ACT_RELU_TANH),
# res (residual, alpha/beta), alpha (alpha without residual), stats (want_stats), affine / scale (src_affine on source 0,
# src_scale on the last source: the split modes at stride 1), rgb / rgb_skip (fused ToRGB), up (four-phase folded up-conv).
FULL = ("bias", "noise", "slope_vec", "res", "stats")
SPLIT_SRC = ("affine", "scale")
TORGB = ("bias", "noise", "tanh", "alpha", "rgb", "rgb_skip")
TORGB_NOSKIP = ("bias", "lrelu", "res", "rgb")
UP = ("up", "bias", "noise", "lrelu")


@dataclass(frozen=True)
class Case:
    name: str
    op: str                  # tf32 | bf16 | f16 | nstack
    B: int
    cin: tuple               # channels of each source (two sources: the virtual concat)
    cout: int
    H: int
    W: int
    feats: tuple
    expect: tuple            # kernel names the launch must run
    k: int = 3
    stride: int = 1
    pad: int = 1
    dil: int = 1
    wB: int = 1
    knobs: tuple = ()        # ((vt_set_option key, value), ...)

    @property
    def Ho(self):
        return self.H if "up" in self.feats else (self.H + 2 * self.pad - self.dil * (self.k - 1) - 1) // self.stride + 1

    @property
    def Wo(self):
        return self.W if "up" in self.feats else (self.W + 2 * self.pad - self.dil * (self.k - 1) - 1) // self.stride + 1

    @property
    def mode(self):
        return "tf32" if self.op == "tf32" else ("f16" if self.op == "f16" else "bf16")


def _split_feats(op, stride=1):
    return SPLIT_SRC if op != "tf32" and stride == 1 else ()


def _table():
    t = []
    for op in ("tf32", "bf16", "f16"):
        o = OP_ENUM[op]
        sf = _split_feats(op)
        t += [
            # N tile 128, one M tile: partial pixel tiles in x and y (19 x 13, handed over transposed), two uneven sources
            Case(f"n128_{op}_full", op, 2, (64, 32), 128, 19, 13, FULL + sf, (kname(128, 1, o),)),
            Case(f"n128_{op}_torgb", op, 2, (64,), 128, 18, 14, TORGB, (kname(128, 1, o),)),
            Case(f"n128_{op}_torgb_noskip_1x1", op, 1, (32,), 128, 20, 10, TORGB_NOSKIP, (kname(128, 1, o),), k=1, pad=0),
            # N tile 64, two M tiles per work item
            Case(f"n64m2_{op}_full", op, 2, (32, 32), 64, 17, 21, FULL + sf, (kname(64, 2, o),)),
            Case(f"n64m2_{op}_torgb", op, 2, (64,), 64, 18, 22, TORGB, (kname(64, 2, o),)),
            Case(f"n64m2_{op}_torgb_noskip", op, 1, (32,), 64, 33, 70, TORGB_NOSKIP, (kname(64, 2, o),)),
            # 4 x 4 maps: one M tile
            Case(f"n64m1_{op}_full", op, 3, (64,), 64, 4, 4, FULL + sf, (kname(64, 1, o),)),
            Case(f"n64m1_{op}_torgb", op, 3, (64,), 64, 4, 4, TORGB, (kname(64, 1, o),)),
            Case(f"n32m1_{op}_full", op, 3, (32, 32), 32, 4, 4, FULL + sf, (kname(32, 1, o),)),
            Case(f"n32m1_{op}_torgb", op, 3, (32,), 32, 4, 4, TORGB, (kname(32, 1, o),)),
            # N tile 32, two and four M tiles (four: the 1x1 small-N halo case)
            Case(f"n32m2_{op}_full", op, 2, (32,), 32, 16, 12, FULL + sf, (kname(32, 2, o),)),
            Case(f"n32m2_{op}_torgb", op, 2, (64,), 32, 16, 12, TORGB, (kname(32, 2, o),)),
            Case(f"n32m4_{op}_full_1x1", op, 1, (128,), 32, 16, 24, FULL + sf, (kname(32, 4, o),), k=1, pad=0),
            Case(f"n32m4_{op}_torgb_1x1", op, 2, (64,), 32, 16, 24, TORGB, (kname(32, 4, o),), k=1, pad=0),
            # four-phase folded up-convolution: N = 4 * Cout = 128
            Case(f"up_{op}", op, 2, (64,), 32, 7, 9, UP, (kname(128, 1, o),)),
        ]
    sf = _split_feats("bf16")
    t += [
        # the N-stacked bf16 split (Cout 32: weight rows [w_hi|w_hi], [w_lo|w_lo], MMA N = 64)
        Case("nstack_m2_full", "nstack", 2, (32,), 32, 16, 12, FULL + sf, (kname(64, 2, 3),)),
        Case("nstack_m2_torgb", "nstack", 2, (64,), 32, 18, 22, TORGB, (kname(64, 2, 3),)),
        Case("nstack_m1_full", "nstack", 3, (32, 32), 32, 4, 4, FULL + sf, (kname(64, 1, 3),)),
        Case("nstack_m1_torgb", "nstack", 3, (32,), 32, 4, 4, TORGB, (kname(64, 1, 3),)),
        # the wide item (128 x 256, bf16 split): the tanh and ToRGB epilogue are left out of it by design
        Case("wide_full", "bf16", 1, (64, 64), 256, 12, 20, FULL + sf, (kname(256, 1, 1),)),
        Case("wide_lrelu_res_512", "bf16", 1, (128,), 512, 9, 16, ("bias", "lrelu", "res"), (kname(256, 1, 1),)),
        Case("wide_up", "bf16", 2, (64,), 64, 6, 10, UP, (kname(256, 1, 1),)),
        Case("wide_excludes_tanh", "bf16", 1, (64,), 256, 12, 20, ("bias", "noise", "tanh", "alpha"), (kname(128, 1, 1),),
             knobs=(("tc_wide", 2),)),
        # the ping-pong item (128 x 128, bf16 split, one consumer warpgroup per item): no tanh or ToRGB either
        Case("pingpong_full", "bf16", 2, (64, 32), 128, 19, 13, FULL + sf, (kname(128, 1, 1, True),), knobs=(("tc_pingpong", 2),)),
        Case("pingpong_lrelu_res_1x1", "bf16", 1, (32,), 128, 20, 10, ("bias", "noise", "lrelu", "res", "stats"),
             (kname(128, 1, 1, True),), k=1, pad=0, knobs=(("tc_pingpong", 2),)),
        Case("pingpong_up", "bf16", 2, (64,), 32, 7, 9, UP, (kname(128, 1, 1, True),), knobs=(("tc_pingpong", 2),)),
        Case("pingpong_excludes_tanh", "bf16", 2, (64,), 128, 18, 14, ("bias", "tanh"), (kname(128, 1, 1),),
             knobs=(("tc_pingpong", 2),)),
        Case("pingpong_excludes_torgb", "bf16", 2, (64,), 128, 18, 14, TORGB_NOSKIP + ("rgb_skip",), (kname(128, 1, 1),),
             knobs=(("tc_pingpong", 2),)),
        # N tiles: 96 = 3 x 32, 192 = 3 x 64, 256 / 512 = 2 / 4 x 128 outside the wide item, 384 = 3 x 128 across phases
        Case("n96_bf16", "bf16", 2, (64,), 96, 12, 20, FULL + sf, (kname(32, 2, 1),)),
        Case("n192_tf32", "tf32", 1, (64,), 192, 17, 21, FULL, (kname(64, 2, 0),)),
        Case("n256_f16", "f16", 2, (64,), 256, 19, 13, FULL + _split_feats("f16"), (kname(128, 1, 2),)),
        Case("n512_tf32", "tf32", 1, (64,), 512, 9, 16, ("bias", "lrelu", "res", "stats"), (kname(128, 1, 0),)),
        Case("up_n96_tf32", "tf32", 1, (32,), 96, 5, 6, UP, (kname(128, 1, 0),)),
        # stride 2 (parity views), dilation, per-sample weights
        Case("s2_bf16", "bf16", 2, (32,), 64, 17, 21, FULL, (kname(64, 1, 1),), stride=2),
        Case("s2_n256_bf16", "bf16", 1, (64,), 256, 33, 29, ("bias", "slope_vec", "res", "stats"), (kname(128, 1, 1),), stride=2),
        Case("s2_1x1_f16", "f16", 2, (64,), 32, 17, 21, FULL, (kname(32, 1, 2),), k=1, pad=0, stride=2),
        Case("dil4_bf16", "bf16", 1, (64,), 128, 24, 16, FULL + sf, (kname(128, 1, 1),), pad=4, dil=4),
        Case("dil2_tf32", "tf32", 2, (32,), 64, 12, 20, FULL, (kname(64, 2, 0),), pad=2, dil=2),
        Case("per_sample_w_bf16", "bf16", 2, (64,), 64, 17, 21, FULL + sf, (kname(64, 2, 1),), wB=2),
        Case("per_sample_w_torgb_f16", "f16", 2, (32,), 32, 16, 12, TORGB, (kname(32, 2, 2),), wB=2),
    ]
    return t


TABLE = _table()
CASES = {c.name: c for c in TABLE}


# ---- inputs and the float64 reference ---------------------------------------------------------------------------------
def blur_kernel():
    k = torch.tensor([1.0, 3.0, 3.0, 1.0])
    k = k[None, :] * k[:, None]
    return k / k.sum() * 4


def make_inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    B, Ho, Wo = c.B, c.Ho, c.Wo
    oh, ow = (2 * c.H, 2 * c.W) if "up" in c.feats else (Ho, Wo)
    cin = sum(c.cin)
    f = set(c.feats)
    inp = {"xs": [torch.randn((B, ch, c.H, c.W), generator=g) for ch in c.cin],
           "w": torch.randn((c.wB, c.cout, cin, c.k, c.k), generator=g) / math.sqrt(cin * c.k * c.k)}
    if "bias" in f:
        inp["bias"] = torch.randn(c.cout, generator=g) * 0.5
    if "noise" in f:
        inp["noise"] = torch.randn((B, 1, oh, ow), generator=g)
        inp["noise_w"] = torch.tensor([0.3])
    if "slope_vec" in f:
        inp["slope_vec"] = torch.rand(c.cout, generator=g) * 0.5 - 0.1      # distinct per channel, some negative
    if "res" in f:
        inp["res"] = torch.randn((B, c.cout, Ho, Wo), generator=g)
    if "affine" in f:
        inp["affine"] = torch.stack([1 + 0.5 * torch.randn((B, c.cin[0]), generator=g), 0.5 * torch.randn((B, c.cin[0]), generator=g)], -1)
    if "scale" in f:
        inp["scale"] = torch.rand((B, 1, c.H, c.W), generator=g) * 1.5
    if "rgb" in f:
        inp["rgb_w"] = torch.randn((c.wB, 3, c.cout), generator=g) * 0.2
        inp["rgb_bias"] = torch.randn(3, generator=g) * 0.1
        if "rgb_skip" in f:
            inp["skip"] = torch.randn((B, 3, Ho // 2, Wo // 2), generator=g)
    if "up" in f:
        inp["blur"] = blur_kernel()
    return inp


def upfirdn64(x, k, up=1, pad=(0, 0)):
    """upfirdn2d (zero-stuff by `up`, zero-pad both sides of both axes, correlate with the flipped kernel) in float64"""
    B, C, H, W = x.shape
    if up > 1:
        u = x.new_zeros((B, C, H * up, W * up))
        u[:, :, ::up, ::up] = x
        x = u
    x = F.pad(x, [pad[0], pad[1], pad[0], pad[1]])
    kf = torch.flip(k.double(), [0, 1])[None, None].repeat(C, 1, 1, 1)
    return F.conv2d(x, kf, groups=C)


def _conv64(c, x, w):
    """x [B, Cin, H, W], w [wB, Cout, Cin, k, k] (float64): the conv of the case, per-sample weights when wB == B"""
    def one(xb, wb):
        if "up" in c.feats:
            return upfirdn64(F.conv_transpose2d(xb, wb.transpose(0, 1), stride=2), blur_kernel().double(), pad=(1, 1))
        return F.conv2d(xb, wb, stride=c.stride, padding=c.pad, dilation=c.dil)
    if w.shape[0] == 1:
        return one(x, w[0])
    return torch.cat([one(x[b:b + 1], w[b]) for b in range(x.shape[0])])


def reference(c, inp):
    """float64 result of the case's descriptor and the sum of absolute terms of every element:
    -> dict(out [B, Cout, Ho', Wo'], terms, and with ToRGB rgb [B, 3, Ho, Wo], rgb_terms)"""
    d = {k: (v.double() if torch.is_tensor(v) else v) for k, v in inp.items()}
    xs = [x.double() for x in d["xs"]]
    if "affine" in d:
        xs[0] = xs[0] * d["affine"][:, :, 0, None, None] + d["affine"][:, :, 1, None, None]   # zero padding added after
    if "scale" in d:
        xs[-1] = xs[-1] * d["scale"]
    x = torch.cat(xs, 1)
    v = _conv64(c, x, d["w"])
    t = _conv64(c, x.abs(), d["w"].abs())
    if "bias" in d:
        v = v + d["bias"].view(1, -1, 1, 1)
        t = t + d["bias"].abs().view(1, -1, 1, 1)
    if "noise" in d:
        v = v + d["noise_w"] * d["noise"]
        t = t + (d["noise_w"] * d["noise"]).abs()
    f = set(c.feats)
    if "lrelu" in f or "slope_vec" in f:
        s = d["slope_vec"].view(1, -1, 1, 1) if "slope_vec" in d else torch.tensor(0.2, dtype=torch.float64)
        gain = 1.25
        v = torch.where(v > 0, v, v * s) * gain
        t = t * torch.clamp(s.abs(), min=1.0) * gain
    elif "tanh" in f:
        v = torch.tanh(torch.relu(v))
    alpha, beta = (0.6, 0.8) if "res" in f else ((0.5, 0.0) if "alpha" in f else (1.0, 0.0))
    if "res" in f:
        v = v * alpha + beta * d["res"]
        t = t * alpha + beta * d["res"].abs()
    else:
        v, t = v * alpha, t * alpha
    r = {"out": v, "terms": t}
    if "rgb" in f:
        w_rgb = d["rgb_w"].expand(c.B, 3, c.cout)
        rgb = torch.einsum("bchw,bkc->bkhw", v, w_rgb) + d["rgb_bias"].view(1, 3, 1, 1)
        rt = torch.einsum("bchw,bkc->bkhw", t, w_rgb.abs()) + d["rgb_bias"].abs().view(1, 3, 1, 1)
        if "skip" in d:
            rgb = rgb + upfirdn64(d["skip"], blur_kernel(), up=2, pad=(2, 1))
            rt = rt + upfirdn64(d["skip"].abs(), blur_kernel(), up=2, pad=(2, 1))
        r["rgb"], r["rgb_terms"] = rgb, rt
    return r


def c_mode(c):
    K = sum(c.cin) * (9 if "up" in c.feats else c.k * c.k)
    return C_OP[c.mode] + math.sqrt(K) * 2.0 ** -24


def err_over_bar(c, y, ref, terms):
    bar = c_mode(c) * terms + EPI * ref.abs() + 1e-30
    return ((y.double() - ref).abs() / bar).max().item()


# ---- running a case on the GPU -----------------------------------------------------------------------------------------
@contextlib.contextmanager
def knobs(op="bf16", **opts):
    """precision, operand split and vt_set_option keys for the duration of the block; every key must be one the library knows
    (vt_set_option returns -1 for an unknown key and changes nothing), and every setting is restored on exit"""
    from vtoonify_b200 import _lib, ops
    lib = _lib.load()
    prec, fmt, nstack = OPS[op]
    saved_ops = {k: ops.get_option(k) for k in ("rs_fmt", "bf16x3_nstack")}
    old_prec = ops.set_precision(prec)
    old = {}
    try:
        ops.set_option("rs_fmt", fmt)
        ops.set_option("bf16x3_nstack", nstack)
        for k, v in opts.items():
            prev = lib.vt_set_option(k.encode(), int(v))
            assert prev != -1, f"vt_set_option: the library has no option {k!r}"
            old.setdefault(k, prev)
        yield lib
    finally:
        for k, v in old.items():
            lib.vt_set_option(k.encode(), v)
        for k, v in saved_ops.items():
            ops.set_option(k, v)
        ops.set_precision(old_prec)


def guarded(shape):
    """(buffer, view): a NaN-filled tensor of `shape` inside a buffer with GUARD floats of GUARD_VALUE on both sides"""
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), float("nan"), device="cuda")
    buf[:GUARD] = GUARD_VALUE
    buf[GUARD + n:] = GUARD_VALUE
    return buf, buf[GUARD:GUARD + n].view(shape)


def check_guarded(buf, view, what):
    assert not torch.isnan(view).any(), f"{what}: {int(torch.isnan(view).sum())} output elements were not written"
    assert bool((buf[:GUARD] == GUARD_VALUE).all()) and bool((buf[-GUARD:] == GUARD_VALUE).all()), f"{what}: write outside the output"


_real_empty = torch.empty


def _nan_empty(*args, **kwargs):
    t = _real_empty(*args, **kwargs)
    if t.is_floating_point():
        t.fill_(float("nan"))
    return t


@contextlib.contextmanager
def nan_allocations():
    """every torch.empty inside the block starts NaN-filled: buffers the library allocates (the ToRGB image, the statistics
    workspace) show an element no kernel wrote"""
    torch.empty = _nan_empty
    try:
        yield
    finally:
        torch.empty = _real_empty


_UP2_TAPS = [(dy, dx, (dy + 1) * 3 + (dx + 1)) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]


class Gpu:
    """the case's inputs on the device in the library's layouts"""

    def __init__(self, c, inp):
        from vtoonify_b200 import ops
        self.c, self.inp = c, inp
        cin = sum(c.cin)
        self.xs = [ops.to_nhwc(x.cuda(), round_tf32=False) for x in inp["xs"]]
        w = torch.cat([ops.prep_weights(inp["w"][i].cuda(), cin_pad=cin, round_tf32=False) for i in range(c.wB)]).contiguous()
        self.w9 = w
        nhwc = lambda t: None if t is None else ops.to_nhwc(t.cuda(), round_tf32=False)
        self.res = nhwc(inp.get("res"))
        cu = lambda k: None if inp.get(k) is None else inp[k].cuda().contiguous()
        self.dev = {k: cu(k) for k in ("bias", "noise", "noise_w", "slope_vec", "affine", "scale", "rgb_w", "rgb_bias", "skip", "blur")}

    def run(self, op, trace=False, **opts):
        """-> dict(out NHWC, stats, rgb, kernels) with the output in a guarded buffer (checked here); kernels: the conv_tc
        kernel names of the launch when `trace` (under torch.profiler), else None"""
        from torch.profiler import ProfilerActivity, profile
        from vtoonify_b200 import ops
        c, dv = self.c, self.dev
        f = set(c.feats)
        with knobs(op, **{**dict(c.knobs), **opts}):
            w = self.w9
            if "up" in f:
                w = ops.fold_upconv_weights(w, dv["blur"])
            kw = dict(bias=dv["bias"], noise=dv["noise"], noise_w=dv["noise_w"])
            if "lrelu" in f or "slope_vec" in f:
                kw.update(act=ACT_LRELU, slope=0.2, gain=1.25, slope_vec=dv["slope_vec"])
            elif "tanh" in f:
                kw.update(act=ACT_RELU_TANH)
            if "res" in f:
                kw.update(res=self.res, alpha=0.6, beta=0.8)
            elif "alpha" in f:
                kw.update(alpha=0.5)
            if "affine" in f:
                kw["src_affine"] = [dv["affine"]] + [None] * (len(self.xs) - 1)
            if "scale" in f:
                kw["src_scale"] = [None] * (len(self.xs) - 1) + [dv["scale"].view(c.B, c.H, c.W)]
            if "rgb" in f:
                kw["rgb"] = {"w": dv["rgb_w"], "bias": dv["rgb_bias"], "skip": dv["skip"], "kernel": _blur_dev() if "skip" in dv and dv["skip"] is not None else None}
            if "up" in f:
                Hf, Wf = 2 * c.H, 2 * c.W
                buf, out = guarded((c.B, Hf, Wf, c.cout))
                kw.update(out=out, out_view=(0, Hf * Wf * c.cout, 2 * Wf * c.cout, 2 * c.cout),
                          phase_offs=[(ry * Wf + rx) * c.cout for ry in (0, 1) for rx in (0, 1)])
                taps, Ho, Wo = _UP2_TAPS, c.H, c.W
            else:
                buf, out = guarded((c.B, c.Ho, c.Wo, c.cout))
                kw["out"] = out
                taps, Ho, Wo = ops.conv_taps(c.k, c.pad, c.dil), c.Ho, c.Wo
            call = lambda: ops.conv2d_nhwc(self.xs, w, taps, c.stride, Ho, Wo, want_stats="stats" in f, **kw)
            call()                      # weight split and module load outside the trace
            pad = torch.zeros(1, device="cuda")
            names = None
            # a launch whose trace shows no conv_tc kernel is traced again (a plan without one shows none every time)
            for _ in range(3 if trace else 0):
                buf.fill_(float("nan"))
                buf[:GUARD] = GUARD_VALUE
                buf[-GUARD:] = GUARD_VALUE
                torch.cuda.synchronize()
                with nan_allocations(), profile(activities=[ProfilerActivity.CUDA]) as prof:
                    pad.add_(1)
                    r = call()
                    pad.add_(1)
                    torch.cuda.synchronize()
                names = tuple(sorted({m.group(0) for e in prof.events() for m in [KERNEL_RE.search(e.name)] if m}))
                if names:
                    break
            if not trace:
                buf.fill_(float("nan"))
                buf[:GUARD] = GUARD_VALUE
                buf[-GUARD:] = GUARD_VALUE
                with nan_allocations():
                    r = call()
                torch.cuda.synchronize()
        check_guarded(buf, out, c.name)
        res = {"out": out.clone(), "stats": None, "rgb": None, "kernels": names}
        if "stats" in f:
            res["stats"] = r[1]
            assert not torch.isnan(r[1]).any(), f"{c.name}: NaN statistics (a partial-sum chunk was not written)"
        if "rgb" in f:
            res["rgb"] = r[1]
            assert not torch.isnan(r[1]).any(), f"{c.name}: ToRGB pixels not written"
        return res


_BLUR = {}


def _blur_dev():
    if "k" not in _BLUR:
        _BLUR["k"] = blur_kernel().cuda()
    return _BLUR["k"]


def to_nchw64(y):
    return y.permute(0, 3, 1, 2).double().cpu()


def check_against_reference(c, got, ref, tag=""):
    """the float64 bar on the output, the image and the statistics; returns the worst err / bar"""
    worst = err_over_bar(c, to_nchw64(got["out"]), ref["out"], ref["terms"])
    if got["rgb"] is not None:
        worst = max(worst, err_over_bar(c, got["rgb"].double().cpu(), ref["rgb"], ref["rgb_terms"]))
    print(f"{c.name}{tag} [{c.mode}] {' '.join(got['kernels'] or ())}: worst err / bar {worst:.3f}")
    assert worst <= 1.0, f"{c.name}{tag}: error {worst:.2f} x the float64 bar"
    if got["stats"] is not None:
        # mean and rstd of the stored output, in float64, against the epilogue's statistics
        y = to_nchw64(got["out"])
        mean, var = y.mean(dim=(2, 3)), y.var(dim=(2, 3), unbiased=False)
        st = got["stats"].double().cpu()
        amax = y.abs().amax(dim=(2, 3))
        assert ((st[:, :, 0] - mean).abs() <= 2e-6 * torch.clamp(amax, min=1.0)).all(), f"{c.name}{tag}: mean"
        rstd = 1.0 / torch.sqrt(var + 1e-5)
        assert ((st[:, :, 1] - rstd).abs() <= 1e-5 * rstd).all(), f"{c.name}{tag}: rstd"
    return worst


# ---- host-side checks (no GPU) -----------------------------------------------------------------------------------------
def test_table_reaches_every_instantiation():
    """the cases' expected kernels are exactly the kTcKernels instantiations (each case asserts its own on the GPU)"""
    table = ktc_kernels()
    assert len(table) == len(set(table)) == 22, table
    reached = {n for c in TABLE for n in c.expect}
    print("kTcKernels:", ", ".join(sorted(table)))
    assert reached == set(table), f"not reached: {sorted(set(table) - reached)}; unknown: {sorted(reached - set(table))}"
    # the exclusions: no tanh or ToRGB case expects the wide or the ping-pong kernel
    for c in TABLE:
        if "tanh" in c.feats or "rgb" in c.feats:
            assert all("<256," not in n and "pingpong" not in n for n in c.expect), c.name


def _direct_reference(c, inp):
    """the same operation restated tap by tap (einsum over shifted input windows) and with the oracle's upfirdn2d"""
    from oracle import vt_oracle as O
    d = {k: (v.double() if torch.is_tensor(v) else v) for k, v in inp.items()}
    xs = [x.double() for x in d["xs"]]
    if "affine" in d:
        xs[0] = xs[0] * d["affine"][:, :, 0, None, None] + d["affine"][:, :, 1, None, None]
    if "scale" in d:
        xs[-1] = xs[-1] * d["scale"]
    x = torch.cat(xs, 1)
    B = x.shape[0]
    w = d["w"].expand(B, *d["w"].shape[1:])
    if "up" in c.feats:
        # transposed conv as scatter: t[2i + ky, 2j + kx] += x[i, j] * w[ky, kx]
        t = x.new_zeros((B, c.cout, 2 * c.H + 1, 2 * c.W + 1))
        for ky in range(3):
            for kx in range(3):
                t[:, :, ky:ky + 2 * c.H:2, kx:kx + 2 * c.W:2] += torch.einsum("bihw,boi->bohw", x, w[:, :, :, ky, kx])
        v = O.upfirdn2d(t, blur_kernel().double(), pad=(1, 1))
    else:
        p = c.pad
        xp = F.pad(x, [p, p, p, p])
        v = x.new_zeros((B, c.cout, c.Ho, c.Wo))
        for ky in range(c.k):
            for kx in range(c.k):
                win = xp[:, :, ky * c.dil: ky * c.dil + c.stride * (c.Ho - 1) + 1: c.stride,
                         kx * c.dil: kx * c.dil + c.stride * (c.Wo - 1) + 1: c.stride]
                v = v + torch.einsum("bihw,boi->bohw", win, w[:, :, :, ky, kx])
    if "bias" in d:
        v = v + d["bias"].view(1, -1, 1, 1)
    if "noise" in d:
        v = v + d["noise_w"] * d["noise"]
    f = set(c.feats)
    if "lrelu" in f or "slope_vec" in f:
        if "slope_vec" in d:
            v = torch.where(v > 0, v, v * d["slope_vec"].view(1, -1, 1, 1)) * 1.25
        else:
            v = F.leaky_relu(v, 0.2) * 1.25
    elif "tanh" in f:
        v = torch.tanh(F.relu(v))
    if "res" in f:
        v = v * 0.6 + 0.8 * d["res"]
    elif "alpha" in f:
        v = v * 0.5
    out = {"out": v}
    if "rgb" in f:
        rgb = F.conv2d(torch.cat([v[b:b + 1] for b in range(B)]), d["rgb_w"][0][:, :, None, None]) if c.wB == 1 else \
            torch.cat([F.conv2d(v[b:b + 1], d["rgb_w"][b][:, :, None, None]) for b in range(B)])
        rgb = rgb + d["rgb_bias"].view(1, 3, 1, 1)
        if "skip" in d:
            rgb = rgb + O.upfirdn2d(d["skip"], blur_kernel().double(), up=2, pad=(2, 1))
        out["rgb"] = rgb
    return out


HOST_CASES = [
    Case("h_concat_affine_scale", "bf16", 2, (8, 4), 6, 7, 5, FULL + SPLIT_SRC, ()),
    Case("h_stride2_dil2", "tf32", 2, (4,), 5, 9, 8, ("bias", "lrelu"), (), stride=2, pad=2, dil=2),
    Case("h_dil4_wb2", "bf16", 2, (4,), 3, 11, 10, ("bias", "noise", "slope_vec", "res"), (), pad=4, dil=4, wB=2),
    Case("h_torgb", "bf16", 2, (4,), 4, 6, 8, TORGB, ()),
    Case("h_torgb_noskip_1x1_wb2", "f16", 2, (4,), 4, 5, 7, TORGB_NOSKIP, (), k=1, pad=0, wB=2),
    Case("h_up", "bf16", 2, (3,), 4, 4, 5, UP, ()),
    Case("h_up_wb2", "bf16", 2, (3,), 2, 3, 3, UP, (), wB=2),
]


@pytest.mark.parametrize("c", HOST_CASES, ids=[c.name for c in HOST_CASES])
def test_reference_agrees_with_direct_restatement(c):
    inp = make_inputs(c, seed=len(c.name))
    ref, direct = reference(c, inp), _direct_reference(c, inp)
    for k in direct:
        assert ref[k].shape == direct[k].shape, k
        assert (ref[k] - direct[k]).abs().max().item() <= 1e-12 * max(1.0, direct[k].abs().max().item()), k
    # the terms bound the value, and the bar of the float64 result is met trivially
    assert bool((ref["out"].abs() <= ref["terms"] * (1 + 1e-12)).all())
    if "rgb" in ref:
        assert bool((ref["rgb"].abs() <= ref["rgb_terms"] * (1 + 1e-12)).all())
    assert err_over_bar(c, ref["out"].float(), ref["out"], ref["terms"]) <= 1.0


# ---- the kernels each case runs, traced in a child process -------------------------------------------------------------------
def split_case():
    """a 3x3 256 -> 256 layer whose 40 pixel tiles per 80 x 64 image leave a partial last round of wide items"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 1
    while 40 * B <= sms or (40 * B) % sms == 0:
        B += 1
    return Case("split", "bf16", B, (64,), 256, 80, 64, ("bias", "stats"), ())


def trace_kernels():
    """{launch: sorted conv_tc kernel names} for every case of the table and the wide remainder split (tc_wide 1 and 0)"""
    out = {}
    for c in TABLE:
        out[c.name] = Gpu(c, make_inputs(c, seed=sum(map(ord, c.name)))).run(c.op, trace=True)["kernels"]
    c = split_case()
    g = Gpu(c, make_inputs(c, seed=23))
    out["split"] = g.run("bf16", trace=True)["kernels"]
    out["split tc_wide=0"] = g.run("bf16", trace=True, tc_wide=0)["kernels"]
    return out


@pytest.fixture(scope="module")
def kernels_run():
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--trace-kernels"]
    r = subprocess.run(args, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"kernel trace failed:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    line = [l for l in r.stdout.splitlines() if l.startswith("KERNELS ")][-1]
    return {k: tuple(v) for k, v in json.loads(line[len("KERNELS "):]).items()}


# ---- GPU: every case of the table ---------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_case_vs_float64(name, kernels_run):
    c = CASES[name]
    inp = make_inputs(c, seed=sum(map(ord, name)))
    got = Gpu(c, inp).run(c.op)
    got["kernels"] = kernels_run[name]
    check_against_reference(c, got, reference(c, inp))
    assert got["kernels"] == tuple(sorted(c.expect)), f"{name}: the planner ran {got['kernels']}, the table expects {c.expect}"


# ---- GPU: knob sweep -----------------------------------------------------------------------------------------------------
def _tg_budgets(c):
    """tc_tgroup values: automatic, one tap per box, a KB budget of 3 taps per box and, where two such stages fit shared
    memory, one of all 9 (the MMA N of the case's N tile)"""
    n = c.cout * (4 if "up" in c.feats else 1)
    bnm = 128 if n % 128 == 0 else (64 if n % 64 == 0 else 32)
    if c.op == "nstack":
        bnm *= 2
    v = [0, 1, 3 * bnm * 128 // 1024]
    if bnm <= 64:
        v.append(9 * bnm * 128 // 1024)
    return v


SWEEP_CASES = ["n128_bf16_full", "n64m2_bf16_full", "n32m2_f16_full", "n32m4_bf16_full_1x1", "n64m2_tf32_full", "s2_bf16",
               "dil4_bf16", "nstack_m2_full", "n64m2_bf16_torgb", "wide_full", "up_bf16"]
SWEEP = {
    "tc_tgroup": _tg_budgets,
    "tc_s2_halo": lambda c: [0, 1] if c.stride == 2 else None,
    "tc_mode": lambda c: [0, 1, 3] if "up" not in c.feats else [1, 3],     # the four phases need halo staging
    "tc_m_major": lambda c: [0, 1],
    "tc_stage_policy": lambda c: [0, 1],
    "tc_halo_pct": lambda c: [50, 60, 100],
    "tc_mt": lambda c: [1, 2, 4],
    "tc_wide": lambda c: [0, 2],
    "tc_pingpong": lambda c: [0, 2],
    "tc_transpose": lambda c: [0, 2],
}
# knobs that leave the statistics chunks (one per 16 output pixels of a tile and consumer warp) where they are; the others can
# change the M tiles per work item or the view, and with them the chunk layout and the order of the finalize's sums
STATS_SAME = {"tc_m_major", "tc_halo_pct", "tc_stage_policy", "tc_pingpong", "tc_wide"}


@gpu
@pytest.mark.parametrize("knob", list(SWEEP))
@pytest.mark.parametrize("name", SWEEP_CASES)
def test_knob_sweep(name, knob):
    c = CASES[name]
    values = SWEEP[knob](c)
    if values is None:
        pytest.skip(f"{knob} does not apply to {name}")
    inp = make_inputs(c, seed=sum(map(ord, name)))
    ref = reference(c, inp)
    g = Gpu(c, inp)
    base = g.run(c.op)
    for v in values:
        got = g.run(c.op, **{knob: v})
        check_against_reference(c, got, ref, tag=f" {knob}={v}")
        assert torch.equal(got["out"], base["out"]), f"{name} {knob}={v}: output differs from the default plan"
        if got["rgb"] is not None:
            assert torch.equal(got["rgb"], base["rgb"]), f"{name} {knob}={v}: image differs from the default plan"
        if got["stats"] is not None and knob in STATS_SAME:
            assert torch.equal(got["stats"], base["stats"]), f"{name} {knob}={v}: statistics differ from the default plan"


# ---- GPU: coverage and guards of strided views, phases, the wide remainder split and the image-only launch ---------------
@gpu
@pytest.mark.parametrize("op", ["tf32", "bf16"])
def test_channel_slice_out_view(op):
    """the output as a channel slice of a wider NHWC tensor (out_view strides): the other channels stay untouched"""
    from vtoonify_b200 import ops
    c = Case("slice", op, 2, (64,), 64, 19, 13, ("bias", "lrelu"), ())
    inp = make_inputs(c, seed=3)
    g = Gpu(c, inp)
    ref = reference(c, inp)
    C_tot, c0 = 160, 64
    buf, out = guarded((c.B, c.Ho, c.Wo, C_tot))
    with knobs(op):
        ops.conv2d_nhwc(g.xs, g.w9, ops.conv_taps(3, 1), 1, c.Ho, c.Wo, out=out,
                        out_view=(c0, c.Ho * c.Wo * C_tot, c.Wo * C_tot, C_tot), bias=g.dev["bias"], act=ACT_LRELU,
                        slope=0.2, gain=1.25)
        torch.cuda.synchronize()
    check_guarded(buf, out[..., c0:c0 + c.cout], "channel slice")
    assert torch.isnan(out[..., :c0]).all() and torch.isnan(out[..., c0 + c.cout:]).all(), "write outside the channel slice"
    got = {"out": out[..., c0:c0 + c.cout], "stats": None, "rgb": None, "kernels": ()}
    check_against_reference(c, got, ref)


@gpu
def test_polyphase_transposed_conv_views():
    """conv_transpose2d(stride 2) as four launches into the phase views of one (2H+1) x (2W+1) output: every element written
    exactly by its phase"""
    from vtoonify_b200 import ops
    g = torch.Generator().manual_seed(19)
    B, Cin, Cout, H, W = 2, 64, 32, 7, 9
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / math.sqrt(Cin * 9)
    ref = F.conv_transpose2d(x.double(), w.double().transpose(0, 1), stride=2)
    terms = F.conv_transpose2d(x.double().abs(), w.double().abs().transpose(0, 1), stride=2)
    xn = ops.to_nhwc(x.cuda(), round_tf32=False)
    wp = ops.prep_weights(w.cuda(), cin_pad=Cin, round_tf32=False)
    Hf, Wf = 2 * H + 1, 2 * W + 1
    buf, out = guarded((B, Hf, Wf, Cout))
    with knobs("bf16"):
        for py in (0, 1):
            for px in (0, 1):
                taps = [(-(ky - py) // 2, -(kx - px) // 2, ky * 3 + kx) for ky in range(py, 3, 2) for kx in range(px, 3, 2)]
                ops.conv2d_nhwc([xn], wp, taps, 1, H + 1 - py, W + 1 - px, out=out,
                                out_view=((py * Wf + px) * Cout, Hf * Wf * Cout, 2 * Wf * Cout, 2 * Cout))
        torch.cuda.synchronize()
    check_guarded(buf, out, "polyphase")
    y = to_nchw64(out)
    bar = (C_OP["bf16"] + math.sqrt(Cin * 4) * 2.0 ** -24) * terms + 1e-30
    assert ((y - ref).abs() / bar).max().item() <= 1.0


@gpu
def test_wide_remainder_split_coverage(kernels_run):
    """a wide layer whose items leave a partial last round: the whole rounds run wide, the rest as a second launch of 128-wide
    items from pixel tile m_first on; together they write every element once (guards intact), as tc_wide 0 does bit for bit"""
    c = split_case()
    g = Gpu(c, make_inputs(c, seed=23))
    got = g.run("bf16")
    assert kernels_run["split"] == (kname(128, 1, 1), kname(256, 1, 1)), kernels_run["split"]
    narrow = g.run("bf16", tc_wide=0)
    assert kernels_run["split tc_wide=0"] == (kname(128, 1, 1),)
    assert torch.equal(got["out"], narrow["out"]) and torch.equal(got["stats"], narrow["stats"])


@gpu
@pytest.mark.parametrize("cout,skip", [(32, True), (64, True), (32, False)])
def test_image_only_torgb_launch(cout, skip):
    """rgb["only"] through the row-strip entry with the conv_tc route (rs_kernel 0): the kernel gets out = NULL and writes
    the image alone; every pixel of it is written and equals the launch that also stores the activation"""
    from vtoonify_b200 import ops
    feats = ("bias", "noise", "lrelu", "rgb") + (("rgb_skip",) if skip else ())
    c = Case("rgb_only", "bf16", 2, (32,), cout, 20, 36, feats, ())
    inp = make_inputs(c, seed=29 + cout)
    g = Gpu(c, inp)
    ref = reference(c, inp)
    old = {k: ops.get_option(k) for k in ("rs_min_width", "rs_conv")}
    rgb = {"w": g.dev["rgb_w"], "bias": g.dev["rgb_bias"], "skip": g.dev["skip"], "kernel": _blur_dev() if skip else None}
    kw = dict(bias=g.dev["bias"], noise=g.dev["noise"], noise_w=g.dev["noise_w"], act=ACT_LRELU, slope=0.2, gain=1.25)
    try:
        ops.set_option("rs_min_width", 1)
        ops.set_option("rs_conv", True)
        with knobs("bf16", rs_kernel=0):
            full, full_rgb = ops.conv2d_nhwc(g.xs, g.w9, ops.conv_taps(3, 1), 1, 20, 36, rgb=rgb, **kw)
            with nan_allocations():
                none, only = ops.conv2d_nhwc(g.xs, g.w9, ops.conv_taps(3, 1), 1, 20, 36, rgb=dict(rgb, only=True), **kw)
                torch.cuda.synchronize()
    finally:
        for k, v in old.items():
            ops.set_option(k, v)
    assert none is None
    assert not torch.isnan(only).any(), f"{int(torch.isnan(only).sum())} image elements not written"
    assert torch.equal(only, full_rgb)
    check_against_reference(c, {"out": full, "rgb": only, "stats": None, "kernels": ()}, ref)


# ---- GPU: descriptors the library refuses ---------------------------------------------------------------------------------
class _TcOnly:
    """the library with every convolution sent to the tensor-core entry point: a descriptor conv_tc does not support reaches
    conv_tc_run, which must refuse it with its own message (instead of the FFMA kernel's)"""

    def __init__(self, lib):
        self._lib = lib
        self.last = None

    def __getattr__(self, k):
        return getattr(self._lib, k)

    def vt_conv2d_tc_supported(self, d):
        return 1

    def vt_conv2d_tc_tf32(self, d, stream):
        self.last = d
        return self._lib.vt_conv2d_tc_tf32(d, stream)

    vt_conv2d_direct_f32 = vt_conv2d_tc_tf32


@contextlib.contextmanager
def tc_only():
    from vtoonify_b200 import _lib
    load = _lib.load
    proxy = _TcOnly(load())
    _lib.load = lambda: proxy
    try:
        yield proxy
    finally:
        _lib.load = load


@gpu
def test_refusals():
    from vtoonify_b200 import _lib, ops
    g = torch.Generator().manual_seed(31)
    B, H, W = 1, 8, 8
    x = ops.to_nhwc(torch.randn((B, 64, H, W), generator=g).cuda(), round_tf32=False)
    w256 = ops.prep_weights((torch.randn((256, 64, 3, 3), generator=g) / 24).cuda(), cin_pad=64, round_tf32=False)
    w64 = ops.prep_weights((torch.randn((64, 64, 3, 3), generator=g) / 24).cuda(), cin_pad=64, round_tf32=False)
    taps = ops.conv_taps(3, 1)

    def refused(match, fn):
        with pytest.raises(_lib.VtError, match=match):
            fn()

    with knobs("bf16"), tc_only():
        rgb = {"w": torch.zeros((1, 3, 256), device="cuda"), "bias": torch.zeros(3, device="cuda"), "skip": None}
        refused(r"conv_tc: fused ToRGB needs Cout a power of two <= 128",
                lambda: ops.conv2d_nhwc([x], w256, taps, 1, H, W, rgb=rgb))
        buf = torch.zeros(64 + 1, device="cuda")
        refused(r"conv_tc: slope_vec not 16-byte aligned",
                lambda: ops.conv2d_nhwc([x], w64, taps, 1, H, W, act=ACT_LRELU, slope_vec=buf[1:]))
        sc = torch.ones((B, H, W), device="cuda")
        refused(r"conv_tc: src_scale / src_affine need the bf16x3 mode and stride 1",
                lambda: ops.conv2d_nhwc([x], w64, taps, 2, H // 2, W // 2, src_scale=[sc]))
    with knobs("tf32"), tc_only():
        refused(r"conv_tc: src_scale / src_affine need the bf16x3 mode and stride 1",
                lambda: ops.conv2d_nhwc([x], w64, taps, 1, H, W, src_scale=[sc]))
    # output statistics of a four-phase launch: refused by conv2d_nhwc, and by the library's plan for the descriptor
    wf = ops.fold_upconv_weights(w64, _blur_dev())
    with knobs("bf16"):
        with pytest.raises(_lib.VtError, match="want_stats needs a dense single-phase output"):
            ops.conv2d_nhwc([x], wf, _UP2_TAPS, 1, H, W, out=torch.empty((B, 2 * H, 2 * W, 64), device="cuda"),
                            out_view=(0, 4 * H * W * 64, 4 * W * 64, 128), phase_offs=[0, 64, 2 * W * 64, 2 * W * 64 + 64],
                            want_stats=True)
        with tc_only() as lib:
            out = torch.empty((B, 2 * H, 2 * W, 64), device="cuda")
            ops.conv2d_nhwc([x], wf, _UP2_TAPS, 1, H, W, out=out, out_view=(0, 4 * H * W * 64, 4 * W * 64, 128),
                            phase_offs=[0, 64, 2 * W * 64, 2 * W * 64 + 64])
            torch.cuda.synchronize()
            assert lib.last is not None
            assert lib.vt_conv2d_tc_stats_chunks(lib.last) == -1
            assert b"conv_tc: output statistics need one phase and no fused ToRGB" in lib.vt_last_error()


if __name__ == "__main__" and sys.argv[1:] == ["--trace-kernels"]:
    # the child process of the kernels_run fixture: a process whose only profiler sessions are these
    sys.path.insert(0, ROOT)
    print("KERNELS " + json.dumps(trace_kernels()))
