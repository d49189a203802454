"""The weight-gradient kernel (csrc/conv_wgrad.cu) called directly through the C ABI, on a designed list of cases around its tile,
plan and padding edges, each checked element by element against the float64 reduction with the bars of tests/wgrad_bounds.py
(hard, statistical, exact zeros); plus cross-sample isolation, batch permutation, ignored pad channels and guard regions
around the output and workspace buffers."""
import ctypes
import math

import pytest
import torch

from tests import wgrad_bounds as WB

pytestmark = pytest.mark.gpu

# the output and workspace are placed inside larger buffers of this NaN pattern: guard regions must keep it, and an element the
# kernel never writes stays NaN and fails the finiteness check
GUARD = 4096
CANARY = 0x7FA5A5A5


def k(kh, kw, pad=0, dil=1):
    """the (dy, dx) taps of a kh x kw cross-correlation (per-axis padding and dilation)"""
    py, px = (pad, pad) if isinstance(pad, int) else pad
    dy, dx = (dil, dil) if isinstance(dil, int) else dil
    return [(ky * dy - py, kx * dx - px) for ky in range(kh) for kx in range(kw)]


def case(name, B, M, N, ah, aw, taps, stride=1, ps=0, sh=None, sw=None, data="randn"):
    return dict(name=name, B=B, M=M, N=N, ah=ah, aw=aw, taps=taps, stride=stride, ps=ps,
                sh=ah if sh is None else sh, sw=aw if sw is None else sw, data=data)


CASES = [
    # M and N around the tile edges (nw 32 / 64 / 128, the M tail, several N tiles with a partial last one); A-grid widths
    # around the box_w thresholds 8 / 16 / 32
    case("m1_n3_aw1", 1, 1, 3, 7, 1, k(3, 3, 1)),
    case("m3_n22_aw7", 2, 3, 22, 9, 7, k(3, 3, 1)),
    case("m33_n33_aw9", 3, 33, 33, 15, 9, k(3, 3, 1)),
    case("m63_n64_aw8_5x5", 2, 63, 64, 17, 8, k(5, 5, 2)),
    case("m64_n65_aw16", 1, 64, 65, 13, 16, k(3, 3, 1)),
    case("m65_n96_aw17_1x3", 2, 65, 96, 11, 17, k(1, 3, (0, 1))),
    case("m129_n129_aw15_3x1", 1, 129, 129, 9, 15, k(3, 1, (1, 0))),
    case("m200_n160_aw31", 1, 200, 160, 7, 31, k(3, 3, 1)),
    case("m33_n257_aw33", 1, 33, 257, 9, 33, k(3, 3, 1)),
    case("m65_n320_aw32_d2", 2, 65, 320, 15, 32, k(3, 3, 2, 2)),
    case("m64_n512_aw100", 1, 64, 512, 5, 100, k(1, 1)),
    # taps: dilation 4 on a 4 x 4 map (eight of nine taps wholly in the padding), 36 taps, asymmetric per-axis offsets,
    # taps wholly outside S on every side
    case("d4_on_4x4", 2, 64, 512, 4, 4, k(3, 3, 4, 4)),
    case("taps36", 1, 22, 48, 13, 17, k(6, 6, (2, 3))),
    case("asym_3x5_dil12", 2, 32, 32, 11, 9, k(3, 5, (0, 2), (1, 2))),
    case("taps_outside", 2, 32, 64, 7, 8, [(0, 0), (100, 0), (-50, -50), (0, 9), (-8, 0), (0, -9)]),
    # stride 2: S of odd and even height and width, negative offsets (parity views 1 with vx = -1), 1x1
    case("s2_odd_p0", 2, 64, 32, 8, 7, k(3, 3), stride=2, sh=17, sw=15),
    case("s2_even_p1", 2, 48, 64, 8, 8, k(3, 3, 1), stride=2, sh=16, sw=16),
    case("s2_1x1", 2, 32, 64, 8, 7, k(1, 1), stride=2, sh=16, sw=13),
    case("s2_5x5_p2", 1, 33, 22, 9, 11, k(5, 5, 2), stride=2, sh=18, sw=22),
    case("s2_even_h_odd_w", 3, 64, 129, 7, 9, k(3, 3, 1), stride=2, sh=14, sw=17),
    # plans: many splits, the ksteps / 16 cap (2 and many), per-sample with and without splits, the largest K of the suite
    case("split15", 2, 64, 64, 64, 64, k(3, 3, 1)),
    case("split2_capped", 1, 64, 64, 32, 32, [(0, 0)]),
    case("split6_capped", 3, 200, 22, 33, 32, [(0, 1)]),
    case("ps_split8", 2, 64, 64, 64, 64, k(3, 3, 1), ps=1),
    case("ps_nosplit", 4, 32, 64, 13, 18, k(3, 3, 1), ps=1),
    case("ps_b8_split2", 8, 32, 64, 32, 32, k(3, 3, 1), ps=1),
    case("largest_k", 2, 64, 64, 128, 128, k(3, 3, 1)),
    # data a max-relative tolerance cannot see
    case("channel_scales", 2, 40, 72, 12, 20, k(3, 3, 1), data="scales"),
    case("positive_s", 2, 64, 64, 32, 32, k(3, 3, 1), data="positive"),
    case("positive_s_split", 1, 32, 32, 64, 64, k(3, 3, 1), data="positive"),
    case("one_loud_sample", 4, 32, 32, 16, 16, k(3, 3, 1), data="loud"),
    case("ps_one_loud_sample", 4, 32, 32, 16, 16, k(3, 3, 1), ps=1, data="loud"),
]


def plan_of(c):
    return WB.plan(c["B"], c["M"], c["N"], c["ah"], c["aw"], len(c["taps"]), c["ps"])


def largest_k_case():
    return max(CASES, key=lambda c: plan_of(c)["ksteps"])


def assert_plan_coverage(cases, ws_floats=None):
    """the case list reaches every choice of plan(): nw 32 / 64 / 128, box_w 8 / 16 / 32, splits 1 / 2 / many, the K-step cap,
    per-sample with and without splits, more than one N tile with a partial last tile, an M over 64 that is not a multiple of 64,
    and stride 2.  ``ws_floats(case)``: the library's workspace size, which must agree with the restated split count."""
    plans = [(c, plan_of(c)) for c in cases]
    assert {p["nw"] for _, p in plans} == {32, 64, 128}
    assert {p["box_w"] for _, p in plans} == {8, 16, 32}
    splits = {p["splits"] for _, p in plans}
    assert 1 in splits and 2 in splits and max(splits) > 2
    assert any(p["capped"] and p["splits"] == 2 for _, p in plans) and any(p["capped"] and p["splits"] > 2 for _, p in plans)
    assert any(c["ps"] and p["splits"] > 1 for c, p in plans) and any(c["ps"] and p["splits"] == 1 for c, p in plans)
    assert any(p["n_tiles"] > 1 and c["N"] % (2 * p["nw"]) for c, p in plans)
    assert any(c["M"] > 64 and c["M"] % 64 for c, p in plans)
    assert any(c["stride"] == 2 for c in cases)
    assert {1, 3, 33, 63, 64, 65, 129, 200} <= {c["M"] for c in cases}
    assert {3, 22, 33, 64, 65, 96, 129, 160, 257, 320, 512} <= {c["N"] for c in cases}
    assert {1, 7, 8, 9, 15, 16, 17, 31, 32, 33, 100} <= {c["aw"] for c in cases}
    assert any(len(c["taps"]) == 36 for c in cases)
    if ws_floats is not None:
        for c, p in plans:
            slice_ = (c["B"] if c["ps"] else 1) * c["M"] * c["N"] * len(c["taps"])
            assert ws_floats(c) == (p["splits"] * slice_ if p["splits"] > 1 else 0), c["name"]


def desc(c, a_cstride=None, s_cstride=None):
    """the descriptor of a case (device pointers filled in by the caller)"""
    from vtoonify_b200 import _lib
    d = _lib.ConvWgradDesc()
    d.struct_size = ctypes.sizeof(_lib.ConvWgradDesc)
    d.B, d.per_sample, d.stride = c["B"], c["ps"], c["stride"]
    d.a_h, d.a_w, d.M, d.a_cstride = c["ah"], c["aw"], c["M"], a_cstride or (c["M"] + 31) // 32 * 32
    d.s_h, d.s_w, d.N, d.s_cstride = c["sh"], c["sw"], c["N"], s_cstride or (c["N"] + 31) // 32 * 32
    d.taps = len(c["taps"])
    for t, (dy, dx) in enumerate(c["taps"]):
        d.tap_dy[t], d.tap_dx[t] = dy, dx
    return d


def host_ws_floats(c):
    from vtoonify_b200 import _lib
    return _lib.load().vt_conv2d_wgrad_ws_floats(ctypes.byref(desc(c)))


# ---------------------------------------------------------------------------------------------------------------------------
def case_data(c, seed):
    """A [B, M, ah, aw] (a grad_output: zero mean) and S [B, N, sh, sw] in float32"""
    g = torch.Generator().manual_seed(seed)
    B = c["B"]
    a = torch.randn((B, c["M"], c["ah"], c["aw"]), generator=g)
    s = torch.randn((B, c["N"], c["sh"], c["sw"]), generator=g)
    if c["data"] == "scales":
        a *= 10.0 ** (8 * torch.rand((1, c["M"], 1, 1), generator=g) - 4)
        s *= 10.0 ** (8 * torch.rand((1, c["N"], 1, 1), generator=g) - 4)
    elif c["data"] == "positive":
        s = 4.0 + 0.25 * s.clamp(-3, 3)                     # post-activation inputs: all positive, mean 16x the spread
    elif c["data"] == "loud":
        a[1] *= 1e3
    return a, s


def nhwc(x, cpad, fill=0.0):
    """[B, C, H, W] -> [B, H, W, cpad] on the GPU with channels C..cpad set to ``fill``"""
    B, C, H, W = x.shape
    out = torch.full((B, H, W, cpad), fill, dtype=torch.float32)
    out[..., :C] = x.permute(0, 2, 3, 1)
    return out.cuda()


def _canary(n):
    return torch.full((n,), CANARY, dtype=torch.int32, device="cuda").view(torch.float32)


def run_wgrad(c, a_dev, s_dev):
    """the C ABI with the output (and the workspace, when the call splits) inside NaN-patterned buffers; asserts the guards are
    intact and returns the output as [nb * M, N, T]"""
    from vtoonify_b200 import _lib, ops
    lib = _lib.load()
    d = desc(c, a_dev.shape[3], s_dev.shape[3])
    d.a, d.s = a_dev.data_ptr(), s_dev.data_ptr()
    n_out = (c["B"] if c["ps"] else 1) * c["M"] * c["N"] * len(c["taps"])
    n_ws = lib.vt_conv2d_wgrad_ws_floats(ctypes.byref(d))
    assert n_ws >= 0
    out_buf = _canary(n_out + 2 * GUARD)
    ws_buf = _canary(n_ws + 2 * GUARD) if n_ws else None
    d.out = out_buf.data_ptr() + 4 * GUARD
    if n_ws:
        d.ws, d.ws_floats = ws_buf.data_ptr() + 4 * GUARD, n_ws
    _lib.check(lib.vt_conv2d_wgrad(ctypes.byref(d), ops._stream()))
    torch.cuda.synchronize()
    for name, buf in (("out", out_buf), ("ws", ws_buf)):
        if buf is None:
            continue
        bits = buf.view(torch.int32)
        assert (bits[:GUARD] == CANARY).all() and (bits[-GUARD:] == CANARY).all(), f"{c['name']}: write outside {name}"
    return out_buf[GUARD:GUARD + n_out].reshape(-1, c["N"], len(c["taps"])).cpu()


def _check_case(c, seed=1):
    a, s = case_data(c, seed)
    y = run_wgrad(c, nhwc(a, (c["M"] + 31) // 32 * 32), nhwc(s, (c["N"] + 31) // 32 * 32))
    y64, E, R = WB.bounds(lambda u, v: WB.wgrad(u, v, c["taps"], c["stride"], c["ps"]), a, s)
    p = plan_of(c)
    WB.check(y, y64, E, R, f"wgrad {c['name']} (nw {p['nw']}, box_w {p['box_w']}, splits {p['splits']}, K steps {p['ksteps']})")
    return y


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_wgrad_kernel(c):
    _check_case(c)


def test_case_list_reaches_every_plan():
    """also a CPU test (tests/test_wgrad_bounds.py)"""
    assert_plan_coverage(CASES, host_ws_floats)


def test_python_entry_point_matches_abi():
    """ops.conv_wgrad_nhwc (torch.empty output and workspace) gives the bits of the guarded C-ABI call, split and unsplit"""
    from vtoonify_b200 import ops
    for c in (case("split", 2, 48, 40, 24, 24, k(3, 3, 1)), case("nosplit", 2, 96, 160, 9, 12, k(3, 3, 1))):
        a, s = case_data(c, 3)
        a_dev, s_dev = nhwc(a, (c["M"] + 31) // 32 * 32), nhwc(s, (c["N"] + 31) // 32 * 32)
        y = ops.conv_wgrad_nhwc(a_dev, s_dev, c["M"], c["N"], c["taps"], c["stride"], bool(c["ps"])).cpu()
        assert torch.equal(y, run_wgrad(c, a_dev, s_dev)), c["name"]


ISO = case("iso", 4, 64, 64, 32, 32, k(3, 3, 1), ps=1)          # 36 items, 2 splits per slice


def test_per_sample_isolation():
    """per sample, zeroing one sample's A makes its slice exactly 0 and leaves every other slice bit-identical"""
    assert plan_of(ISO)["splits"] > 1
    a, s = case_data(ISO, 4)
    M, N = ISO["M"], ISO["N"]
    y0 = run_wgrad(ISO, nhwc(a, M), nhwc(s, N))
    a[2] = 0
    y1 = run_wgrad(ISO, nhwc(a, M), nhwc(s, N))
    assert torch.equal(y1[2 * M:3 * M], torch.zeros_like(y1[2 * M:3 * M]))
    keep = torch.ones(4 * M, dtype=torch.bool)
    keep[2 * M:3 * M] = False
    assert torch.equal(y1[keep], y0[keep])


def test_per_sample_permutation():
    """permuting the batch in the per-sample form permutes the output slices bit for bit"""
    a, s = case_data(ISO, 5)
    M, N = ISO["M"], ISO["N"]
    perm = [2, 0, 3, 1]
    y = run_wgrad(ISO, nhwc(a, M), nhwc(s, N)).reshape(4, M, N, -1)
    yp = run_wgrad(ISO, nhwc(a[perm], M), nhwc(s[perm], N)).reshape(4, M, N, -1)
    assert torch.equal(yp, y[perm])


@pytest.mark.parametrize("c", [case("pad_split", 2, 33, 40, 24, 24, k(3, 3, 1)),
                               case("pad_ps", 3, 70, 20, 9, 17, k(3, 3, 1), ps=1),
                               case("pad_s2", 2, 40, 33, 8, 8, k(3, 3, 1), stride=2, sh=16, sw=16)],
                         ids=lambda c: c["name"])
def test_pad_channels_ignored(c):
    """A and S with channel strides wider than M and N and NaN in the pad channels give the zero-padded call's bits"""
    a, s = case_data(c, 6)
    ca, cs = (c["M"] + 31) // 32 * 32, (c["N"] + 31) // 32 * 32
    y = run_wgrad(c, nhwc(a, ca), nhwc(s, cs))
    y_nan = run_wgrad(c, nhwc(a, ca + 64, math.nan), nhwc(s, cs + 32, math.nan))
    assert torch.equal(y, y_nan)
