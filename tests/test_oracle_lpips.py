"""CPU: the float64 LPIPS restatement (tests/oracle_lpips.py) against the reference's own PNetLin (tests/golden/lpips_*.npz), and the
reference's state-dict keys against the library's PNetLin."""
import json
import os

import numpy as np
import pytest
import torch

from tests import oracle_lpips as O
from vtoonify_b200.weights import det_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def ref_keys():
    with open(os.path.join(GOLDEN, "state_dict_keys_lpips.json")) as f:
        return json.load(f)


def oracle_sd():
    """the float64 weights the fixtures were made with: det_state_dict (seed 0) over the PNetLin keys and shapes"""
    from vtoonify_b200.lpips import PNetLin
    return {k: v.double() for k, v in det_state_dict(PNetLin(pnet_rand=True), seed=0).items()}


@pytest.mark.parametrize("case", sorted(O.CASES))
def test_oracle_matches_reference(case):
    shape, seed, g_pred, g_target = O.CASES[case]
    z = np.load(os.path.join(GOLDEN, f"lpips_{case}.npz"))
    pred, target = O.inputs(shape, seed)
    assert np.array_equal(pred.numpy(), z["pred"]) and np.array_equal(target.numpy(), z["target"])
    sd = oracle_sd()
    pred.requires_grad_(g_pred)
    target.requires_grad_(g_target)
    with torch.enable_grad():            # other test modules may leave grad mode off
        loss = O.perceptual_loss(sd, pred, target)
        (loss.flatten() * O.loss_weights(shape[0], seed)).sum().backward()
    assert loss.shape == (shape[0], 1, 1, 1)
    np.testing.assert_allclose(loss.detach().numpy(), z["loss"], rtol=1e-12, atol=0)
    for name, t, want in (("pred_grad", pred, g_pred), ("target_grad", target, g_target)):
        if want:
            np.testing.assert_allclose(t.grad.numpy(), z[name], rtol=1e-9, atol=1e-15)
        else:
            assert name not in z.files


def test_oracle_normalize_is_the_affine_map():
    sd = oracle_sd()
    pred, target = O.inputs((1, 3, 20, 18), 5)
    p01, t01 = (pred + 1) / 2, (target + 1) / 2
    a = O.perceptual_loss(sd, p01, t01, normalize=True)
    b = O.perceptual_loss(sd, pred, target)
    torch.testing.assert_close(a, b, rtol=1e-12, atol=0)


def test_state_dict_keys_match_reference():
    from vtoonify_b200.lpips import PNetLin
    keys = ref_keys()
    assert len(keys) == 33
    assert list(PNetLin(pnet_rand=True).state_dict().keys()) == keys
