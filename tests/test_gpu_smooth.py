"""Parsing-map smoothing end to end on the GPU: the warp drop-in against the reference's fixture, smooth_parsing_maps against the float64
restatement (tests/oracle_smooth.py) in fp32, bf16x3 and tf32, the cached flows against RAFT.forward bit for bit, CPU- and
device-resident inputs, the launches of an interior frame and one run at the smoothing size."""
import pytest
import torch

from tests import oracle_smooth as O
from tests.golden.make_golden_raft import images, raft_args
from tests.golden.make_golden_smooth import parsing_maps, parsing_seed
from tests.test_smooth_host import case
from vtoonify_b200 import ops, set_precision
from vtoonify_b200 import smooth_parsing as S
from vtoonify_b200._lib import launch_count
from vtoonify_b200.raft import RAFT
from vtoonify_b200.weights import det_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
BARS = {"fp32": 2e-5, "bf16x3": 5e-3, "tf32": 4e-2}     # measured worst on an H100: 4.6e-6, 1.05e-3, 9.5e-3 (DESIGN.md section 12)
_REF64 = {}


@pytest.fixture(scope="module")
def model_sd():
    torch.manual_seed(0)
    m = RAFT(raft_args()).eval()
    sd = det_state_dict(m, seed=0)
    m.load_state_dict(sd, strict=True)
    m.requires_grad_(False)
    return m.to(DEV), {k: v.to(DEV) for k, v in sd.items()}


@pytest.fixture(autouse=True)
def _restore_precision():
    yield
    set_precision(ops.DEFAULT_PRECISION)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_warp_dropin_matches_fixture(golden):
    d = golden("smooth_warp")
    x, flo = torch.from_numpy(d["x"]).to(DEV), torch.from_numpy(d["flo"]).to(DEV)
    out, mask = S.warp(x, flo)
    assert mask.shape == x.shape
    assert torch.equal(mask.cpu(), torch.from_numpy(d["mask"]).expand(mask.shape))
    err = float((out.cpu() - torch.from_numpy(d["out"])).abs().max())
    print(f"warp against the reference fixture: max |err| {err:.2e}")
    assert err <= 2e-6, err                       # measured 0 (the same arithmetic as the CPU reference)


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "tf32"])
@pytest.mark.parametrize("name", ["w2", "w5"])
def test_smoothing_against_float64(golden, model_sd, name, prec):
    m, sd = model_sd
    Is, Ps, window, ch, ref32 = case(golden, name)
    set_precision(prec)
    with torch.no_grad():
        out = S.smooth_parsing_maps(Is, Ps, m, window=window, iters=20)
        if name not in _REF64:
            sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
            _REF64[name] = O.smooth(sd64, Is.to(DEV).double(), Ps.to(DEV).double(), window, 20)
        ref = _REF64[name]
    assert out.device == Ps.device and out.shape == ref.shape
    err = _rel(out, ref.cpu())
    err32 = _rel(out[:, ch], ref32)
    print(f"smoothing {name} {prec}: relative L2 {err:.3e} against float64, {err32:.3e} against the reference's float32 fixture")
    assert err <= BARS[prec], err


@pytest.mark.parametrize("name", ["w2", "w5"])
def test_cached_flows_bit_identical_to_forward(golden, model_sd, name):
    """each frame's fnet features and each centre's cnet state computed once give the flows RAFT.forward gives on the same pairs"""
    m, _ = model_sd
    Is, Ps, window, _, _ = case(golden, name)
    set_precision("bf16x3")
    got = {}
    with torch.no_grad():
        S._smooth(Is, Ps, m, window, 20, flow_sink=lambda i, up: got.__setitem__(i, up.clone()))
        Is_ = torch.cat((Is[0:window], Is, Is[-window:]), 0).to(DEV)
        for ii in range(Is.shape[0]):
            i = ii + window
            nb = torch.cat((Is_[i - window:i], Is_[i + 1:i + window + 1]), 0)
            image1 = Is_[i].repeat(2 * window, 1, 1, 1)
            _, up = m((image1 + 1) * 255.0 / 2, (nb + 1) * 255.0 / 2, iters=20, test_mode=True)
            assert torch.equal(got[ii], up), (ii, float((got[ii] - up).abs().max()))


def test_cpu_and_device_inputs_identical(golden, model_sd):
    m, _ = model_sd
    Is, Ps, window, _, _ = case(golden, "w2")
    set_precision("bf16x3")
    with torch.no_grad():
        a = S.smooth_parsing_maps(Is, Ps, m, window=window, iters=4)
        b = S.smooth_parsing_maps(Is.to(DEV), Ps.to(DEV), m, window=window, iters=4)
    assert a.device.type == "cpu" and b.device.type == "cuda"
    assert torch.equal(a, b.cpu())


def test_window_zero_is_the_downsampled_maps(golden, model_sd):
    m, _ = model_sd
    Is, Ps, _, _, _ = case(golden, "w2")
    n0 = launch_count()
    with torch.no_grad():
        out = S.smooth_parsing_maps(Is, Ps, m, window=0)
    assert launch_count() - n0 == 2 * Is.shape[0]                 # a fusion (the identity) and a down-sampling per frame
    torch.testing.assert_close(out, O.down(Ps.double()).float(), rtol=1e-6, atol=1e-6)


def test_interior_frame_launches(model_sd):
    """an interior frame: one fnet encode (the frame entering the window), one cnet encode, the 2 * window pair iterations, the
    fusion and the down-sampling"""
    m, _ = model_sd
    set_precision("bf16x3")
    window, iters, H, W = 2, 3, 128, 128
    frames = torch.cat([images(1, H, W, 40 + k)[0] for k in range(9)]) / 127.5 - 1.0
    Ps = parsing_maps(parsing_seed(9, 5)[:, :4], H, W)
    totals = []
    with torch.no_grad():
        for N in (6, 7, 8):
            n0 = launch_count()
            S.smooth_parsing_maps(frames[:N], Ps[:N], m, window=window, iters=iters)
            totals.append(launch_count() - n0)
        x = ((frames[:1] + 1) * 255.0 / 2).to(DEV)
        n0 = launch_count()
        f = m._features(m._input_s2d(x))
        n_fnet = launch_count() - n0
        n0 = launch_count()
        net, inp = m._context(m._input_s2d(x))
        n_cnet = launch_count() - n0
        B = 2 * window
        n0 = launch_count()
        m._iterate(f.expand(B, -1, -1, -1).contiguous(), f.expand(B, -1, -1, -1).contiguous(), net.expand(B, -1, -1, -1).contiguous(),
                   inp.expand(B, -1, -1, -1).contiguous(), iters)
        n_iter = launch_count() - n0
    per = n_fnet + n_cnet + n_iter + 2
    print(f"smoothing launches: N=6,7,8 -> {totals}; fnet {n_fnet}, cnet {n_cnet}, iterations {n_iter}, per interior frame {per}")
    assert totals[1] - totals[0] == per and totals[2] - totals[1] == per


def test_smoothing_size_against_device_restatement(model_sd):
    """7 frames at 800x800, window 5, 20 iterations, bf16x3, against the restatement in fp32 on cuDNN with TF32 off"""
    m, sd = model_sd
    set_precision("bf16x3")
    N, H = 7, 800
    Is = torch.cat([images(1, H, H, 60 + k)[k % 2] for k in range(N)]) / 127.5 - 1.0
    Ps = parsing_maps(parsing_seed(N, 9), H, H)
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        out = S.smooth_parsing_maps(Is, Ps, m, window=5, iters=20)
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        tf = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        try:
            ref = O.smooth(sd, Is.to(DEV), Ps.to(DEV), 5, 20)
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf
    assert out.shape == (N, 19, H // 2, H // 2) and torch.isfinite(out).all()
    err = _rel(out, ref.cpu())
    print(f"smoothing 7x800x800 window 5 bf16x3 vs fp32 restatement: relative L2 {err:.3e}; peak {peak:.2f} GB")
    assert err <= 2.5e-3, err                    # measured 6.3e-4
