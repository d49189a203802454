"""CPU: pin the float64 restatement of ConditionalDiscriminator.forward and its gradients (tests/oracle_discriminator.py) to the
unmodified reference's discriminator step (tests/golden/discriminator_*.npz)."""
import pytest
import torch

from tests.oracle_discriminator import CASES, CHANNEL_MULTIPLIER, SIZE, WSTEP, case_inputs, forward, loss_fn


def T(a):
    return torch.from_numpy(a)


def rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def oracle_step(case, sd):
    """float64 forward + softplus(-out).mean() backward of the restatement -> (out, x.grad, {name: grad})"""
    p = {k: v.double().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    x, d, s = case_inputs(case)
    x = x.double().requires_grad_()
    with torch.enable_grad():
        out = forward(p, x, d.double(), s)
        loss_fn(out).backward()
    return out.detach(), x.grad, {k: v.grad for k, v in p.items() if v.grad is not None}


@pytest.mark.parametrize("case", list(CASES))
def test_discriminator_oracle_golden(golden, case):
    from vtoonify_b200.vtoonify import ConditionalDiscriminator
    from vtoonify_b200.weights import det_state_dict
    g = golden(f"discriminator_{case}")
    sd = det_state_dict(ConditionalDiscriminator(SIZE, channel_multiplier=CHANNEL_MULTIPLIER, **CASES[case]), seed=0)
    out, gx, grads = oracle_step(case, sd)
    checks = [("out", out, T(g["out"])), ("x.grad", gx[:, :, ::4, ::4], T(g["x_grad_sub"]))]
    for k, gr in grads.items():
        if gr.dim() == 1:
            checks.append((k, gr, T(g["g:" + k])))
        else:
            checks.append((k, gr.flatten()[::WSTEP], T(g["gs:" + k])))
            assert abs(gr.norm().item() - float(g["gn:" + k])) <= 1e-10 * float(g["gn:" + k]), k
    assert len(grads) == sum(1 for n in g.files if n.startswith(("g:", "gs:")))
    for name, got, ref in checks:
        assert got.shape == ref.shape, name
        assert rel(got, ref) <= 1e-10, f"{case} {name}: relative L2 {rel(got, ref):.2e}"
