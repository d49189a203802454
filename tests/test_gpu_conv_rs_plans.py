"""conv_rs (csrc/conv_rs.cu, the row-strip entry point vt_conv2d_rs) against a float64 reference, instantiation by instantiation.

Every case of TABLE names the kernel the launch must run: conv_rs_kernel<CIN, COUT>, or conv_tc_kernel<...> for a descriptor
vt_conv_rs_takes declines.  The names come from torch.profiler traces taken in one child process (as in
test_gpu_conv_tc_plans.py), and test_table_reaches_every_instantiation reads kRsKernels from the source to check that the table
reaches all four instantiations.  The reference, the error bar and the guarded, NaN-filled output buffers are those of
test_gpu_conv_tc_plans.py: an element's bar is C_OP["bf16"] (+ the fp32 accumulation term) times the float64 sum of the
absolute values of every term that went into it.  The N-stacked split conv_rs_kernel runs at Cout = 32 keeps all four hi/lo
products, so the bf16 bar is no looser there than it is at Cout = 64.

Every case also checks that two launches give the same bits and that sample b of a B-sample launch equals a 1-sample launch of
that sample bit for bit: a pixel's accumulation order and the ToRGB shuffle order must not depend on which CTA or consumer
warpgroup owns its tile.  The edges: tiles ragged in x and y, images smaller than one 8 x 16 tile and a single row, one tile
per sample with more than two samples per CTA (per-sample weights reloaded on every work item), the fused ToRGB image (with
and without the up-sampled skip, and the image-only launch), and the output as a channel slice of a wider NHWC buffer.

The production shapes (the last two VToonify-D layers and LPIPS conv1_2) run with the default routing options and are checked
against float64 in row bands, each computed on the CPU from the rows it reads.
"""
import contextlib
import dataclasses
import json
import math
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.test_gpu_conv_tc_plans import (ACT_LRELU, Case, Gpu, _blur_dev, _direct_reference, blur_kernel,  # noqa: E402
                                          check_against_reference, check_guarded, err_over_bar, guarded, kname, knobs,
                                          make_inputs, nan_allocations, reference, upfirdn64, GUARD, GUARD_VALUE)

torch.set_grad_enabled(False)
gpu = pytest.mark.gpu

CONV_RS_SRC = os.path.join(ROOT, "vtoonify_b200", "csrc", "conv_rs.cu")
KERNEL_RE = re.compile(r"conv_(?:rs|tc|tc_pingpong)_kernel<[\d, ]+>")
PER_SAMPLE = 0          # Case.B / Case.wB placeholder: B = 2 x the SM count + 7 (resolve), wB = B


def rs_kname(cin, cout):
    return f"conv_rs_kernel<{cin}, {cout}>"


def krs_kernels():
    """kernel names of the kRsKernels entries of csrc/conv_rs.cu"""
    src = open(CONV_RS_SRC).read()
    table = re.search(r"const RsKernel kRsKernels\[\] = \{(.*?)\};", src, re.S).group(1)
    return [rs_kname(int(a), int(b)) for a, b in re.findall(r"VT_RS\((\d+), (\d+)\)", table)]


# ---- the case table ---------------------------------------------------------------------------------------------------
# Features beyond test_gpu_conv_tc_plans.py's bias / noise / lrelu / rgb / rgb_skip / stats:
#   nw0     a noise_w of 0 passed without noise      only    the image-only ToRGB launch (rgb["only"]: no activation stored)
#   slice0  output channels [0, Cout) of a 2 Cout-channel NHWC buffer, sliceC: channels [Cout, 2 Cout)
EPI = ("bias", "noise", "lrelu")
CHANNELS = ((32, 32), (32, 64), (64, 32), (64, 64))


def _table():
    t = []
    for ci, co in CHANNELS:
        n, rs = f"{ci}to{co}", (rs_kname(ci, co),)
        # conv_tc at 38 x 20 (not handed over transposed): N tile Cout, two M tiles per item; a Cout = 32 launch that takes the
        # row-strip route in ops gets the N-stacked weights (MMA N 64), the statistics and fp16-split launches the plain split
        tc_bf16, tc_f16 = kname(co, 2, 1), kname(co, 2, 2)
        tc_rs_weights = kname(64, 2, 3) if co == 32 else tc_bf16
        t += [
            Case(f"ragged_{n}", "bf16", 2, (ci,), co, 37, 13, EPI, rs),
            Case(f"none_nw0_{n}", "bf16", 2, (ci,), co, 21, 30, ("nw0",), rs),
            Case(f"tiny_{n}", "bf16", 2, (ci,), co, 5, 3, EPI, rs),
            Case(f"one_row_{n}", "bf16", 3, (ci,), co, 1, 40, EPI, rs),
            # one 8 x 16 tile per sample, more than two samples per CTA: weights reloaded on every item
            Case(f"per_sample_{n}", "bf16", PER_SAMPLE, (ci,), co, 16, 8, EPI, rs, wB=PER_SAMPLE),
            Case(f"per_sample_w1_{n}", "bf16", PER_SAMPLE, (ci,), co, 16, 8, EPI, rs),
            Case(f"torgb_skip_{n}", "bf16", 2, (ci,), co, 38, 20, EPI + ("rgb", "rgb_skip"), rs, wB=2),
            Case(f"torgb_noskip_{n}", "bf16", 2, (ci,), co, 37, 13, EPI + ("rgb",), rs, wB=2),
            Case(f"torgb_only_{n}", "bf16", 2, (ci,), co, 38, 20, EPI + ("rgb", "rgb_skip", "only"), rs, wB=2),
            Case(f"slice0_noise_{n}", "bf16", 2, (ci,), co, 37, 13, EPI + ("slice0",), rs),
            Case(f"sliceC_{n}", "bf16", 2, (ci,), co, 37, 13, ("bias", "lrelu", "sliceC"), rs),
            # fallbacks: vt_conv_rs_takes declines the noise of a view whose offset is not a whole pixel, statistics and fp16
            Case(f"sliceC_noise_{n}", "bf16", 2, (ci,), co, 38, 20, EPI + ("sliceC",), (tc_rs_weights,)),
            Case(f"stats_{n}", "bf16", 2, (ci,), co, 38, 20, EPI + ("stats",), (tc_bf16,)),
            Case(f"f16_{n}", "f16", 2, (ci,), co, 38, 20, EPI, (tc_f16,)),
        ]
    return t


TABLE = _table()
CASES = {c.name: c for c in TABLE}

# the full-resolution layers at their real sizes: the last two VToonify-D layers (the 32 -> 32 one stores only the image) and
# LPIPS conv1_2 of the G step; default routing options (rs_min_width 256)
PROD = [
    Case("prod_32to32_2304x4096_rgb_only", "bf16", 2, (32,), 32, 2304, 4096, ("bias", "lrelu", "rgb", "rgb_skip", "only"),
         (rs_kname(32, 32),), wB=2),
    Case("prod_64to64_1152x2048_torgb", "bf16", 2, (64,), 64, 1152, 2048, EPI + ("rgb", "rgb_skip"), (rs_kname(64, 64),), wB=2),
    Case("prod_64to64_512x512_lpips", "bf16", 2, (64,), 64, 512, 512, ("bias", "lrelu"), (rs_kname(64, 64),)),
]
PRODS = {c.name: c for c in PROD}


def resolve(c):
    """the case with the PER_SAMPLE placeholders replaced (needs the device)"""
    if c.B != PER_SAMPLE:
        return c
    B = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 7
    return dataclasses.replace(c, B=B, wB=B if c.wB == PER_SAMPLE else c.wB)


def case_inputs(c):
    inp = make_inputs(c, seed=sum(map(ord, c.name)))
    if "nw0" in c.feats:
        inp["noise_w"] = torch.zeros(1)
    return inp


# ---- band reference: output rows [r0, r1) from the rows they read --------------------------------------------------------
def band_reference(c, small, rows, r0, r1):
    """reference() of output rows [r0, r1) of case c, computed from input rows r0 - 1 .. r1 (zero rows only beyond the image's
    own borders), noise rows r0 .. r1 - 1 and, for the image, the skip rows those output rows read.  small: the CPU weights,
    bias, noise_w and ToRGB operands; rows(key, a, b): rows [a, b) of "x", "noise" or "skip" as CPU NCHW tensors."""
    H, W = c.H, c.W
    x = torch.nn.functional.pad(rows("x", max(r0 - 1, 0), min(r1 + 1, H)).double(), [1, 1, int(r0 == 0), int(r1 == H)])
    bc = dataclasses.replace(c, H=r1 - r0 + 2, W=W + 2, pad=0, feats=tuple(f for f in c.feats if f != "rgb_skip"))
    inp = dict(small, xs=[x])
    if "noise" in c.feats:
        inp["noise"] = rows("noise", r0, r1)
    r = reference(bc, inp)
    if "rgb_skip" in c.feats:
        # upfirdn2d(up 2, pad (2, 1)): skip row i is padded up-sampled row 2 i + 2, and output row y reads padded rows y .. y + 3
        s0, s1 = max((r0 - 1) // 2, 0), min(r1 // 2 + 1, H // 2)
        sk = rows("skip", s0, s1).double()
        u = sk.new_zeros((c.B, 3, r1 - r0 + 3, W + 3))
        u[:, :, 2 * s0 + 2 - r0:2 * s1 + 2 - r0:2, 2:W + 2:2] = sk
        r["rgb"] = r["rgb"] + upfirdn64(u, blur_kernel())
        r["rgb_terms"] = r["rgb_terms"] + upfirdn64(u.abs(), blur_kernel())
    return r


def bands(H):
    """the first rows, a band across a 16-row tile seam mid-image and the last rows"""
    seam = H // 2 // 16 * 16
    return [(0, 12), (seam - 5, seam + 6), (H - 13, H)]


# ---- host-side checks (no GPU) -----------------------------------------------------------------------------------------
def test_table_reaches_every_instantiation():
    table = krs_kernels()
    assert len(table) == len(set(table)) == 4, table
    print("kRsKernels:", ", ".join(table))
    reached = {n for c in TABLE + PROD for n in c.expect if n.startswith("conv_rs")}
    assert reached == set(table), f"not reached: {sorted(set(table) - reached)}; unknown: {sorted(reached - set(table))}"
    # every instantiation also has each declined descriptor
    for ci, co in CHANNELS:
        for kind in ("sliceC_noise", "stats", "f16"):
            assert CASES[f"{kind}_{ci}to{co}"].expect[0].startswith("conv_tc_kernel<")


HOST_CASES = [
    Case("h_band_torgb_wb2", "bf16", 2, (4,), 4, 38, 20, EPI + ("rgb", "rgb_skip"), (), wB=2),
    Case("h_band_odd", "bf16", 2, (4,), 3, 37, 13, ("bias", "noise", "lrelu", "rgb"), ()),
    Case("h_band_small", "bf16", 1, (4,), 3, 6, 10, ("rgb", "rgb_skip"), ()),
]


@pytest.mark.parametrize("c", HOST_CASES, ids=[c.name for c in HOST_CASES])
def test_band_reference_equals_full_reference(c):
    inp = case_inputs(c)
    full = reference(c, inp)
    small = {k: inp[k] for k in ("w", "bias", "noise_w", "rgb_w", "rgb_bias") if k in inp}
    rows = lambda k, a, b: (inp["xs"][0] if k == "x" else inp[k])[:, :, a:b]
    H = c.H
    spans = [(0, H), (0, 1), (0, 5), (1, 2), (max(H // 2 - 3, 0), min(H // 2 + 4, H)), (H - 5, H), (H - 1, H)]
    for r0, r1 in spans + (bands(H) if H >= 32 else []):
        band = band_reference(c, small, rows, r0, r1)
        for k, v in band.items():
            want = full[k][:, :, r0:r1]
            assert v.shape == want.shape, (k, r0, r1)
            assert (v - want).abs().max().item() <= 1e-12 * max(1.0, want.abs().max().item()), (k, r0, r1)


RESTATE_CASES = [
    Case("h_rs_ragged", "bf16", 2, (4,), 5, 7, 5, EPI, ()),
    Case("h_rs_nw0", "bf16", 2, (4,), 3, 5, 3, ("nw0",), ()),
    Case("h_rs_one_row_wb3", "bf16", 3, (4,), 3, 1, 6, EPI, (), wB=3),
    Case("h_rs_torgb_wb2", "bf16", 2, (4,), 4, 6, 8, EPI + ("rgb", "rgb_skip"), (), wB=2),
]


@pytest.mark.parametrize("c", RESTATE_CASES, ids=[c.name for c in RESTATE_CASES])
def test_reference_agrees_with_direct_restatement(c):
    inp = case_inputs(c)
    ref, direct = reference(c, inp), _direct_reference(c, inp)
    for k in direct:
        assert ref[k].shape == direct[k].shape, k
        assert (ref[k] - direct[k]).abs().max().item() <= 1e-12 * max(1.0, direct[k].abs().max().item()), k
    assert bool((ref["out"].abs() <= ref["terms"] * (1 + 1e-12)).all())


# ---- running a case on the GPU -----------------------------------------------------------------------------------------
@contextlib.contextmanager
def rs_route(min_width=1):
    """ops options for the block: rs_conv on and rs_min_width = min_width (None: left at its default); restored on exit"""
    from vtoonify_b200 import ops
    old = {k: ops.get_option(k) for k in ("rs_conv", "rs_min_width")}
    try:
        ops.set_option("rs_conv", True)
        if min_width is not None:
            ops.set_option("rs_min_width", min_width)
        yield
    finally:
        for k, v in old.items():
            ops.set_option(k, v)


@contextlib.contextmanager
def guarded_allocations():
    """every float32 CUDA torch.empty inside the block (the ToRGB image, the statistics workspace) comes NaN-filled inside
    GUARD_VALUE guards (guarded()); the others NaN-filled (nan_allocations).  Yields the list of (buffer, view) made."""
    made = []
    with nan_allocations():
        nan_empty = torch.empty

        def empty(*shape, **kw):
            size = shape[0] if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)) else shape
            dev = kw.get("device")
            if (set(kw) <= {"device", "dtype"} and kw.get("dtype", torch.float32) == torch.float32 and dev is not None
                    and torch.device(dev).type == "cuda" and all(isinstance(s, int) for s in size)):
                made.append(guarded(tuple(size)))
                return made[-1][1]
            return nan_empty(*shape, **kw)
        torch.empty = empty
        try:
            yield made
        finally:
            torch.empty = nan_empty


def _reset(buf):
    buf.fill_(float("nan"))
    buf[:GUARD] = GUARD_VALUE
    buf[-GUARD:] = GUARD_VALUE


class RsGpu(Gpu):
    """a case on the device (Gpu) run through ops.conv2d_nhwc with the row-strip route enabled"""
    min_width = 1

    def run(self, trace=False, only=None):
        """-> dict(out NHWC (the channel slice for the slice cases, None for the image-only launch), rgb, stats, kernels),
        every output written into NaN-filled buffers with guards (checked here); kernels: the conv_rs / conv_tc kernel names
        of the launch when `trace`"""
        from torch.profiler import ProfilerActivity, profile
        from vtoonify_b200 import ops
        c, dv = self.c, self.dev
        f = set(c.feats)
        only = "only" in f if only is None else only
        kw = dict(bias=dv["bias"], noise=dv["noise"], noise_w=dv["noise_w"], want_stats="stats" in f)
        if "lrelu" in f:
            kw.update(act=ACT_LRELU, slope=0.2, gain=1.25)
        if "rgb" in f:
            kw["rgb"] = {"w": dv["rgb_w"], "bias": dv["rgb_bias"], "skip": dv["skip"],
                         "kernel": _blur_dev() if dv["skip"] is not None else None, "only": only}
        c_tot, c0 = (2 * c.cout, 0 if "slice0" in f else c.cout) if ("slice0" in f or "sliceC" in f) else (c.cout, 0)
        buf = full = None
        if not only:
            buf, full = guarded((c.B, c.Ho, c.Wo, c_tot))
            kw["out"] = full
            if c_tot != c.cout:
                kw["out_view"] = (c0, c.Ho * c.Wo * c_tot, c.Wo * c_tot, c_tot)
        call = lambda: ops.conv2d_nhwc(self.xs, self.w9, ops.conv_taps(3, 1), 1, c.Ho, c.Wo, **kw)
        names = None
        with knobs(c.op), rs_route(self.min_width):
            call()                      # weight split and module load outside the trace
            torch.cuda.synchronize()
            pad = torch.zeros(1, device="cuda")
            # a launch whose trace shows no conv kernel is traced again: a trace can come back without any of its kernels (not
            # even the marker adds around the launch); eight such traces in a row, or three with kernels but no conv kernel,
            # leave names empty and fail the case's route check
            lost = 0
            for attempt in range(8 if trace else 1):
                if attempt - lost >= 3:
                    break
                if buf is not None:
                    _reset(buf)
                torch.cuda.synchronize()
                with guarded_allocations() as made, (profile(activities=[ProfilerActivity.CUDA]) if trace else
                                                     contextlib.nullcontext()) as prof:
                    if trace:
                        pad.add_(1)
                    r = call()
                    if trace:
                        pad.add_(1)
                    torch.cuda.synchronize()
                if trace:
                    events = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                    names = tuple(sorted({m.group(0) for n in events for m in [KERNEL_RE.search(n)] if m}))
                    if names:
                        break
                    lost += not events
        res = {"out": None, "rgb": None, "stats": None, "kernels": names}
        if only:
            assert r[0] is None, f"{c.name}: the image-only launch returned an activation"
        else:
            out = full[..., c0:c0 + c.cout]
            check_guarded(buf, out, c.name)
            if c_tot != c.cout:
                rest = torch.cat([full[..., :c0], full[..., c0 + c.cout:]], -1)
                assert torch.isnan(rest).all(), f"{c.name}: write outside the channel slice"
            res["out"] = out.clone()
        for b, v in made:
            assert bool((b[:GUARD] == GUARD_VALUE).all()) and bool((b[-GUARD:] == GUARD_VALUE).all()), \
                f"{c.name}: write outside a buffer the library allocated"
        key = "rgb" if "rgb" in f else ("stats" if "stats" in f else None)
        if key:
            assert not torch.isnan(r[1]).any(), f"{c.name}: {int(torch.isnan(r[1]).sum())} {key} elements not written"
            res[key] = r[1].clone()
        return res


def sample_inputs(inp, b, per_sample_w):
    """sample b of the case's inputs (its weights when they are per sample)"""
    s = {}
    for k, v in inp.items():
        if k == "xs":
            s[k] = [x[b:b + 1] for x in v]
        elif k in ("noise", "skip") or (per_sample_w and k in ("w", "rgb_w")):
            s[k] = v[b:b + 1]
        else:
            s[k] = v
    return s


def invariance_samples(B):
    if B <= 4:
        return list(range(B))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sorted({0, 1, sms - 1, sms, 2 * sms, B - 1})


# ---- production shapes ------------------------------------------------------------------------------------------------------
class ProdGpu(RsGpu):
    """a production-size case generated on the device (default routing options); rows() copies rows back for band_reference"""
    min_width = None

    def __init__(self, c):
        from vtoonify_b200 import ops
        self.c = c
        g = torch.Generator(device="cuda").manual_seed(sum(map(ord, c.name)))
        rnd = lambda *s: torch.randn(s, generator=g, device="cuda")
        cin = c.cin[0]
        x = rnd(c.B, c.H, c.W, cin)
        w = rnd(c.wB, c.cout, cin, 3, 3) / math.sqrt(cin * 9)
        self.xs = [x]
        self.w9 = torch.cat([ops.prep_weights(w[i], cin_pad=cin, round_tf32=False) for i in range(c.wB)]).contiguous()
        f = set(c.feats)
        dv = dict.fromkeys(("bias", "noise", "noise_w", "rgb_w", "rgb_bias", "skip"))
        dv["bias"] = rnd(c.cout) * 0.5
        if "noise" in f:
            dv["noise"], dv["noise_w"] = rnd(c.B, 1, c.H, c.W), torch.full((1,), 0.3, device="cuda")
        if "rgb" in f:
            dv["rgb_w"], dv["rgb_bias"] = rnd(c.wB, 3, c.cout) * 0.2, rnd(3) * 0.1
        if "rgb_skip" in f:
            dv["skip"] = rnd(c.B, 3, c.H // 2, c.W // 2)
        self.dev = dv
        self.small = {"w": w.double().cpu(), **{k: dv[k].double().cpu() for k in ("bias", "noise_w", "rgb_w", "rgb_bias")
                                                 if dv[k] is not None}}

    def rows(self, key, a, b):
        if key == "x":
            return self.xs[0][:, a:b].permute(0, 3, 1, 2).double().cpu()
        return self.dev[key][:, :, a:b].double().cpu()


# ---- the kernels each case runs, traced in a child process -------------------------------------------------------------------
def trace_kernels():
    out = {}
    for c in TABLE:
        c = resolve(c)
        try:
            out[c.name] = RsGpu(c, case_inputs(c)).run(trace=True)["kernels"]
        except Exception as e:   # reported by the case's own test
            out[c.name] = [f"error: {e}"]
    for c in PROD:
        try:
            out[c.name] = ProdGpu(c).run(trace=True)["kernels"]
        except Exception as e:
            out[c.name] = [f"error: {e}"]
        torch.cuda.empty_cache()
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
    c = resolve(CASES[name])
    inp = case_inputs(c)
    g = RsGpu(c, inp)
    got = g.run()
    again = g.run()
    for k in ("out", "rgb", "stats"):
        if got[k] is not None:
            assert torch.equal(got[k], again[k]), f"{name}: two launches differ ({k})"
    got["kernels"] = kernels_run[name]
    if "only" in c.feats:
        full = g.run(only=False)
        assert torch.equal(got["rgb"], full["rgb"]), f"{name}: the image-only image differs from the full launch's"
        got["out"] = full["out"]
    check_against_reference(c, got, reference(c, inp))
    assert got["kernels"] == tuple(sorted(c.expect)), f"{name}: ran {got['kernels']}, the table expects {c.expect}"
    # batch invariance: a sample's bits do not depend on the rest of the batch or on which CTA / warpgroup owns its tiles
    for b in invariance_samples(c.B):
        cb = dataclasses.replace(c, B=1, wB=1)
        one = RsGpu(cb, sample_inputs(inp, b, c.wB > 1)).run()
        for k in ("out", "rgb", "stats"):
            if got[k] is not None and one[k] is not None:
                assert torch.equal(got[k][b:b + 1], one[k]), f"{name}: sample {b} differs from its 1-sample launch ({k})"


@gpu
@pytest.mark.parametrize("name", list(PRODS))
def test_production_shape_bands_vs_float64(name, kernels_run):
    c = PRODS[name]
    g = ProdGpu(c)
    got = g.run()
    kernels = kernels_run[name]
    assert kernels == tuple(sorted(c.expect)), f"{name}: ran {kernels}, expected {c.expect}"
    worst = 0.0
    for r0, r1 in bands(c.H):
        ref = band_reference(c, g.small, g.rows, r0, r1)
        if got["out"] is not None:
            y = got["out"][:, r0:r1].permute(0, 3, 1, 2).double().cpu()
            worst = max(worst, err_over_bar(c, y, ref["out"], ref["terms"]))
        if got["rgb"] is not None:
            worst = max(worst, err_over_bar(c, got["rgb"][:, :, r0:r1].double().cpu(), ref["rgb"], ref["rgb_terms"]))
    print(f"{name} [bf16] {' '.join(kernels)}: worst err / bar {worst:.3f} over rows {bands(c.H)}")
    assert worst <= 1.0, f"{name}: error {worst:.2f} x the float64 bar"
    del g, got
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("cout", [32, 64])
def test_image_only_hint_off_the_row_strip_route(cout):
    """with rs_conv off, conv2d_nhwc sends the launch to conv_tc, which ignores rgb["only"]: the activation is still returned,
    and it and the image are bit-identical to the launch without the hint"""
    from vtoonify_b200 import ops
    c = Case("only_off_rs", "bf16", 2, (32,), cout, 20, 36, EPI + ("rgb", "rgb_skip"), (), wB=2)
    inp = case_inputs(c)
    g = RsGpu(c, inp)
    dv, xs, w9 = g.dev, g.xs, g.w9
    rgb = {"w": dv["rgb_w"], "bias": dv["rgb_bias"], "skip": dv["skip"], "kernel": _blur_dev()}
    kw = dict(bias=dv["bias"], noise=dv["noise"], noise_w=dv["noise_w"], act=ACT_LRELU, slope=0.2, gain=1.25)
    with knobs("bf16"), rs_route():
        ops.set_option("rs_conv", False)
        out, img = ops.conv2d_nhwc(xs, w9, ops.conv_taps(3, 1), 1, c.Ho, c.Wo, rgb=dict(rgb, only=True), **kw)
        full, full_img = ops.conv2d_nhwc(xs, w9, ops.conv_taps(3, 1), 1, c.Ho, c.Wo, rgb=rgb, **kw)
        torch.cuda.synchronize()
    assert out is not None and torch.equal(out, full) and torch.equal(img, full_img)
    check_against_reference(c, {"out": out, "rgb": img, "stats": None, "kernels": ()}, reference(c, inp))


# ---- GPU: ToRGB operands ops.conv2d_nhwc refuses ----------------------------------------------------------------------------
@gpu
def test_torgb_operand_refusals():
    """the fused ToRGB operands are read by raw pointer ("w" as a dense [wB][3][Cout] with the conv weight's wB): a tensor of
    another shape or layout is refused instead of being read as one"""
    from vtoonify_b200 import _lib, ops
    B, H, W, C = 2, 8, 16, 32
    x = torch.randn((B, H, W, C), device="cuda")
    w = ops.prep_weights(torch.randn((C, C, 3, 3), device="cuda") / 17, cin_pad=C, round_tf32=False)
    good = {"w": torch.zeros((1, 3, C), device="cuda"), "bias": torch.zeros(3, device="cuda"),
            "skip": torch.zeros((B, 3, H // 2, W // 2), device="cuda"), "kernel": _blur_dev()}

    def conv(**rgb):
        return ops.conv2d_nhwc([x], w, ops.conv_taps(3, 1), 1, H, W, rgb=dict(good, **rgb))

    def refused(match, **rgb):
        with pytest.raises(_lib.VtError, match=match):
            conv(**rgb)

    with knobs("bf16"), rs_route():
        conv()
        conv(w=torch.zeros((1, 1, 3, C), device="cuda"))
        conv(skip=None, kernel=None)
        refused(r"rgb\['w'\]", w=torch.zeros((B, 3, C), device="cuda"))               # per-sample ToRGB weights, wB = 1
        refused(r"rgb\['w'\]", w=torch.zeros((1, C, 3), device="cuda").transpose(1, 2))  # not contiguous
        refused(r"rgb\['w'\]", w=torch.zeros((1, 3, 2 * C), device="cuda")[:, :, :C])
        refused(r"rgb\['w'\]", w=torch.zeros((3 * C,), device="cuda"))
        refused(r"rgb\['bias'\]", bias=torch.zeros(4, device="cuda"))
        refused(r"rgb\['bias'\]", bias=torch.zeros(6, device="cuda")[::2])
        refused(r"rgb\['skip'\]", skip=torch.zeros((B, 3, H // 2 + 1, W // 2), device="cuda"))
        refused(r"rgb\['skip'\]", skip=torch.zeros((1, 3, H // 2, W // 2), device="cuda"))
        refused(r"rgb\['kernel'\]", kernel=torch.ones((3, 3), device="cuda"))
        refused(r"rgb\['kernel'\]", kernel=None)
        torch.cuda.synchronize()


if __name__ == "__main__" and sys.argv[1:] == ["--trace-kernels"]:
    # the child process of the kernels_run fixture: a process whose only profiler sessions are these
    print("KERNELS " + json.dumps(trace_kernels()))
