"""Parsing-map smoothing on the host: the plain-torch restatement (tests/oracle_smooth.py) against the reference's float32 fixtures, the
slot -> frame map, the temporal weights and every argument error of vtoonify_b200.smooth_parsing (CPU only)."""
import pytest
import torch

from tests import oracle_smooth as O
from tests.golden.make_golden_raft import raft_args
from tests.golden.make_golden_smooth import parsing_maps, script_inputs
from vtoonify_b200 import smooth_parsing as S
from vtoonify_b200.raft import RAFT
from vtoonify_b200.weights import det_state_dict


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _model():
    torch.manual_seed(0)
    m = RAFT(raft_args()).eval()
    sd = det_state_dict(m, seed=0)
    m.load_state_dict(sd, strict=True)
    return m, sd


def case(golden, name):
    """the script's Is and Ps of a fixture, and the fixture's window and stored parse channels"""
    d = golden(f"smooth_{name}")
    Is = script_inputs(d["frames"])
    Ps = parsing_maps(torch.from_numpy(d["seed"]), Is.shape[2], Is.shape[3])
    return Is, Ps, int(d["window"]), [int(c) for c in d["channels"]], torch.from_numpy(d["parse"])


def test_restated_warp_matches_fixture(golden):
    d = golden("smooth_warp")
    out, mask = O.warp(torch.from_numpy(d["x"]), torch.from_numpy(d["flo"]))
    ref_mask = torch.from_numpy(d["mask"]).expand_as(mask)
    assert torch.equal(mask, ref_mask)
    assert 0.2 < float(mask.mean()) < 0.9                 # both outcomes are well represented
    assert torch.equal(out, torch.from_numpy(d["out"]))    # the same CPU grid_sample on the same grid


@pytest.mark.parametrize("name", ["w2", "w5"])
def test_restated_smoothing_matches_fixture(golden, name):
    """the reference's own float32 level: its RAFT and the restated RAFT differ in the last bits"""
    Is, Ps, window, ch, ref = case(golden, name)
    _, sd = _model()
    with torch.no_grad():
        out = O.smooth(sd, Is, Ps, window, 20)
    assert out.shape == (Is.shape[0], Ps.shape[1], Is.shape[2] // 2, Is.shape[3] // 2)
    err = _rel(out[:, ch], ref)
    print(f"restated smoothing {name}: relative L2 {err:.3e} against the reference")
    assert err <= 2e-5, err


@pytest.mark.parametrize("window", [0, 1, 2, 5])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_slot_frames_match_reference_indexing(window, k):
    N = {1: max(window, 1), 2: window + 1, 3: max(3 * window, 1)}[k]
    Is = torch.arange(N)
    Is_ = torch.cat((Is[0:window], Is, Is[-window:]), dim=0)      # the script's line 129
    slots = S.slot_frames(N, window)
    assert len(slots) == N
    for ii in range(N):
        i = ii + window
        assert slots[ii] == Is_[i - window:i + window + 1].tolist()


@pytest.mark.parametrize("window", [0, 1, 2, 5, 31])
def test_temporal_weights_bit_identical(window):
    wt = torch.exp(-(torch.arange(2 * window + 1).float() - window) ** 2 / (2 * ((window + 0.5) ** 2))).reshape(2 * window + 1, 1, 1, 1)
    mine = S.temporal_weights(window)
    assert mine.dtype == torch.float32 and torch.equal(mine, wt.reshape(-1))
    assert torch.equal(torch.tensor(mine.tolist(), dtype=torch.float32), wt.reshape(-1))     # the host floats handed to the kernel


def _inputs(N=6, C=4, H=128, W=136):
    return torch.zeros((N, 3, H, W)), torch.zeros((N, C, H, W))


def test_argument_errors():
    m, _ = _model()
    m.requires_grad_(False)
    Is, Ps = _inputs()
    with pytest.raises(ValueError, match="fewer than the window"):
        S.smooth_parsing_maps(Is[:2], Ps[:2], m, window=3)
    with pytest.raises(ValueError, match="window"):
        S.smooth_parsing_maps(Is, Ps, m, window=-1)
    with pytest.raises(ValueError, match="window"):
        S.smooth_parsing_maps(Is, Ps, m, window=S.MAX_WINDOW + 1)
    with pytest.raises(ValueError, match="multiples of 8"):
        S.smooth_parsing_maps(*_inputs(H=132), m, window=2)
    with pytest.raises(ValueError, match="multiples of 8"):
        S.smooth_parsing_maps(*_inputs(W=120), m, window=2)
    with pytest.raises(ValueError, match="must be"):
        S.smooth_parsing_maps(Is, Ps[:5], m, window=2)
    with pytest.raises(ValueError, match="must be"):
        S.smooth_parsing_maps(Is, Ps[..., :128], m, window=2)
    with pytest.raises(ValueError, match="must be"):
        S.smooth_parsing_maps(Ps, Ps, m, window=2)
    with pytest.raises(ValueError, match="float32"):
        S.smooth_parsing_maps(Is.double(), Ps, m, window=2)
    with pytest.raises(ValueError, match="iters"):
        S.smooth_parsing_maps(Is, Ps, m, window=2, iters=0)


@torch.enable_grad()
def test_unsupported_model_and_grad():
    m, _ = _model()
    Is, Ps = _inputs()
    with pytest.raises(NotImplementedError, match="requires grad"):          # parameters that require grad, in grad mode
        S.smooth_parsing_maps(Is, Ps, m, window=2)
    m.requires_grad_(False)
    with pytest.raises(NotImplementedError, match="require grad"):
        S.smooth_parsing_maps(Is.clone().requires_grad_(True), Ps, m, window=2)
    with pytest.raises(NotImplementedError, match="train mode"):
        S.smooth_parsing_maps(Is, Ps, m.train(), window=2)
    with pytest.raises(NotImplementedError, match="vtoonify_b200.raft.RAFT"):
        S.smooth_parsing_maps(Is, Ps, torch.nn.Identity(), window=2)
    with pytest.raises(NotImplementedError, match="require grad"):
        S.warp(torch.zeros(1, 3, 8, 8, requires_grad=True), torch.zeros(1, 2, 8, 8))
    with pytest.raises(ValueError, match="warp"):
        S.warp(torch.zeros(1, 3, 8, 8), torch.zeros(1, 2, 8, 9))


def test_no_cuda_device_is_an_error():
    """CPU inputs and a CPU model: there is no CPU fallback"""
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    m, _ = _model()
    m.requires_grad_(False)
    with pytest.raises(ValueError, match="CUDA"):
        S.smooth_parsing_maps(*_inputs(), m, window=2)

