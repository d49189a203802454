"""Pins the float64 restatement tests/oracle_raft.py to the unmodified reference RAFT (float32 fixtures, CPU)."""
import numpy as np
import pytest
import torch

from tests import oracle_raft as O
from tests.golden.make_golden_raft import CASES, KEEP, UP_ROWS, raft_args
from vtoonify_b200.raft import RAFT
from vtoonify_b200.weights import det_state_dict


@pytest.fixture(scope="module")
def sd64():
    sd = det_state_dict(RAFT(raft_args()), seed=0)
    return {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference(golden, sd64, name):
    """float64 restatement against the reference's float32 run: relative L2 at float32 level (measured 3.6e-7 .. 3.7e-6; the 20-iteration
    case carries the most float32 rounding of the reference itself).  The fixtures keep part of the larger outputs (make_golden_raft)."""
    c, g = CASES[name], golden(f"raft_{name}")
    fi = torch.from_numpy(g["flow_init"]).double() if "flow_init" in g else None
    out = O.raft_forward(sd64, torch.from_numpy(g["image1"]).double(), torch.from_numpy(g["image2"]).double(), c["iters"], fi,
                         c["test_mode"])
    if c["test_mode"]:
        up = out[1][:, :, :UP_ROWS] if name == "b2" else out[1]
        assert _rel(out[0], g["flow_low"]) < 2e-5
        assert _rel(up, g["flow_up"]) < 2e-5
    else:
        assert len(out) == c["iters"] == int(g["n_pred"])
        assert _rel(torch.stack([out[k] for k in KEEP]), g["flow_up"]) < 2e-5
    assert float(np.abs(g["flow_up"]).mean()) > 1.0           # the fixtures hold real motion


def test_oracle_lookup_matches_corrblock(golden):
    """channel l*81 + 9i + j samples x-offset i - 4 and y-offset j - 4 (a swap would fail on this non-symmetric volume); the reference
    goes through grid_sample's normalised coordinates, hence the float32-level bar"""
    g = golden("raft_lookup")
    pyr = O.pyramid(torch.from_numpy(g["fmap1"]).double(), torch.from_numpy(g["fmap2"]).double())
    out = O.lookup(pyr, torch.from_numpy(g["coords"]).double())
    ref = torch.from_numpy(g["corr"]).double()
    assert float((out - ref).abs().max()) < 2e-5 * float(ref.abs().max())
    swapped = O.lookup(pyr, torch.from_numpy(g["coords"]).double().flip(1))
    assert float((swapped - ref).abs().max()) > 0.1 * float(ref.abs().max())
