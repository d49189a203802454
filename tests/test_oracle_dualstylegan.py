"""CPU: pin the DualStyleGAN.forward restatement (tests/oracle_dualstylegan.py) against outputs of the unmodified reference
(tests/golden/dualstylegan64.npz), and the module's state_dict against the reference's keys and shapes."""
import json

import pytest
import torch

from tests.oracle_dualstylegan import KEYS, CASES, case_inputs, case_outputs, dualstylegan_forward, state_dict

torch.set_grad_enabled(False)


def assert_close(a, b, atol, what):
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item()
    assert err <= atol, f"{what}: max abs err {err:.3e} > {atol:.1e}"


def test_state_dict_keys_match_reference():
    from vtoonify_b200.dualstylegan import DualStyleGAN
    keys = json.load(open(KEYS))
    ours = {k: list(v.shape) for k, v in DualStyleGAN(64, 512, 8).state_dict().items()}
    assert ours == keys


@pytest.mark.parametrize("name", list(CASES))
def test_dualstylegan_oracle_golden(golden, name):
    g = golden("dualstylegan64")
    sd = state_dict()
    kw, inputs = CASES[name]
    styles, ex = case_inputs(g, inputs)
    noises = [sd[f"generator.noises.noise_{i}"] for i in range(9)]
    y = dualstylegan_forward(sd, styles, ex, noises, **kw)
    if name == "feat":
        y = (y[0][:, ::32], y[1])
    for got, ref in zip(y if isinstance(y, tuple) else (y,), case_outputs(g, name)):
        assert_close(got, ref, 5e-5, f"DualStyleGAN(64) {name}")
