"""CPU: the float64 restatement of the on-demand correlation (AlternateCorrBlock) against the CorrBlock restatement and the reference's
CorrBlock fixture, and the ``raft_corr`` option's default and validation."""
import pytest
import torch

from tests import oracle_raft as O
from tests import oracle_raft_ondemand as OD
from vtoonify_b200 import ops


def _maps(B, C, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, h, w, generator=g, dtype=torch.float64), torch.randn(B, C, h, w, generator=g, dtype=torch.float64)


def _coords(B, h, w, seed, spread=3.0):
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    return torch.stack([xs, ys])[None].repeat(B, 1, 1, 1) + spread * torch.randn(B, 2, h, w, generator=g, dtype=torch.float64)


EDGE = [[-1.0, -0.5, 20.5, 21.0, 1e4, -3e6, -4.0, -9.5, -13.0, 0.0],
        [-0.25, -1.0, 0.0, 16.0, 5.0, 2.0, -7.75, 30.0, -4.0, -41.0]]


def _both(f1, f2, coords):
    a = OD.ondemand(f1, OD.fmap_pyramid(f2), coords)
    b = O.lookup(O.pyramid(f1, f2), coords)
    return a, b


# C is a square: oracle_raft.pyramid divides by a float32 sqrt(C), as CorrBlock does
@pytest.mark.parametrize("B,C,h,w,spread", [(1, 16, 17, 21, 3.0), (2, 9, 13, 11, 6.0), (3, 4, 9, 15, 0.0), (1, 64, 16, 16, 25.0)])
def test_ondemand_equals_corrblock_float64(B, C, h, w, spread):
    """odd and even level sizes; centres (spread 0), fractional, far-reaching flows; border, just and far outside, negative"""
    f1, f2 = _maps(B, C, h, w, h * w)
    coords = _coords(B, h, w, B + h, spread)
    coords[0, :, 0, :len(EDGE[0])] = torch.tensor(EDGE, dtype=torch.float64)[:, :w]
    a, b = _both(f1, f2, coords)
    assert a.shape == b.shape == (B, 324, h, w)
    scale = float(b.abs().max())
    assert (a - b).abs().max().item() <= 1e-12 * scale
    # the far-outside coordinates give exact zeros at every level
    assert not a[0, :, 0, 4].any() and not a[0, :, 0, 5].any()


def test_ondemand_matches_reference_fixture(golden):
    """the reference's CorrBlock output (float32, [1, 16, 17, 21]: level sizes 17x21, 8x10, 4x5, 2x2)"""
    g = golden("raft_lookup")
    f1, f2 = torch.from_numpy(g["fmap1"]).double(), torch.from_numpy(g["fmap2"]).double()
    ref = torch.from_numpy(g["corr"]).double()
    out = OD.ondemand(f1, OD.fmap_pyramid(f2), torch.from_numpy(g["coords"]).double())
    assert (out - ref).abs().max().item() <= 2e-5 * float(ref.abs().max())


def test_option_default_and_validation():
    assert ops.get_option("raft_corr") == "volume"
    try:
        ops.set_option("raft_corr", "on_demand")
        assert ops.get_option("raft_corr") == "on_demand"
        for bad in ("alternate", "Volume", None, True, 1):
            with pytest.raises(ValueError, match="raft_corr"):
                ops.set_option("raft_corr", bad)
        assert ops.get_option("raft_corr") == "on_demand"
    finally:
        ops.set_option("raft_corr", "volume")


def test_alternate_corr_still_refused_and_points_to_the_option():
    from tests.golden.make_golden_raft import raft_args
    from vtoonify_b200.raft import RAFT
    with pytest.raises(NotImplementedError, match="alternate_corr.*raft_corr"):
        RAFT(raft_args(["--alternate_corr"]))
