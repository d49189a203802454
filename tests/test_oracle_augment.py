"""CPU: the float64 restatement of random_apply_affine (tests/oracle_augment.py) against the unmodified reference's float64 output
(tests/golden/augment_*.npz), and its upfirdn2d against the reference's op_cpu semantics on the passes the augmentation uses."""
import os

import numpy as np
import pytest
import torch

from tests import oracle_augment as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ("a", "odd", "id", "zoom")


def load(case):
    z = np.load(os.path.join(GOLDEN, f"augment_{case}.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference(case):
    f = load(case)
    out = O.apply(f["img"].double(), f["G"])
    ref = f["out64"]
    assert out.shape == ref.shape == f["img"].shape
    err = (out - ref).abs().max().item()
    print(f"{case}: oracle vs reference float64 max |err| {err:.3e}")
    assert err <= 1e-12 * max(1.0, ref.abs().max().item())


def test_upfirdn2d_is_a_true_convolution():
    """up 2 with pad (6, 5) and kernel k: y[n] = sum_i x[i] k[n + 5 - 2i]; down 2 with pad (-1, -1) and the flipped kernel:
    y[n] = sum_t k[t] x[2n + 1 + t]"""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 1, 3, 9, dtype=torch.float64, generator=g)
    k = torch.randn(12, dtype=torch.float64, generator=g)
    up = O.upfirdn2d(x, k.view(1, 12), up=(2, 1), pad=(6, 5, 0, 0))
    want = torch.zeros(1, 1, 3, 18, dtype=torch.float64)
    for n in range(18):
        for i in range(9):
            if 0 <= n + 5 - 2 * i < 12:
                want[..., n] += x[..., i] * k[n + 5 - 2 * i]
    assert torch.allclose(up, want, rtol=0, atol=1e-14)
    a = torch.randn(1, 1, 2, 30, dtype=torch.float64, generator=g)
    down = O.upfirdn2d(a, torch.flip(k, (0,)).view(1, 12), down=(2, 1), pad=(-1, -1, 0, 0))
    want = torch.stack([(k * a[..., 2 * n + 1:2 * n + 13]).sum(-1) for n in range(9)], -1)
    assert down.shape == want.shape and torch.allclose(down, want, rtol=0, atol=1e-14)
