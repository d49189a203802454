"""CPU: pin the float64 restatement of the return_feat path and its gradients (tests/oracle_vtoonify_feat.py) to the unmodified
reference's encoder-pretraining step (tests/golden/feat_grad_*.npz)."""
import pytest
import torch

from tests.oracle_vtoonify_feat import CASES, WSTEP, case_inputs, loss_and_grads, targets


def T(a):
    return torch.from_numpy(a)


def rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("case", list(CASES))
def test_feat_grad_oracle_golden(golden, case):
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict
    g = golden(f"feat_grad_{case}")
    backbone, d_s = CASES[case]
    sd = det_state_dict(VToonify(backbone=backbone), seed=0)
    x, style = case_inputs()
    t_f, t_s = targets((2, 512, 8, 6), (2, 3, 8, 6))
    r = loss_and_grads(sd, x, style, d_s, backbone, t_f, t_s)
    # both sides are float64 with the same operation order up to library kernels: agreement at ~1e-12
    assert abs(r["loss"].item() - float(g["loss"])) <= 1e-12 * float(g["loss"])
    checks = [("feat", r["feat"][:, ::8], T(g["feat_sub"])), ("skip", r["skip"], T(g["skip"])),
              ("x.grad", r["x_grad"][:, :, ::4, ::4], T(g["x_grad_sub"]))]
    for k, gr in r["grads"].items():
        if gr.dim() == 1:
            checks.append((k, gr, T(g["g:" + k])))
        else:
            checks.append((k, gr.flatten()[::WSTEP], T(g["gs:" + k])))
            assert abs(gr.norm().item() - float(g["gn:" + k])) <= 1e-10 * float(g["gn:" + k]), k
    assert len(r["grads"]) == sum(1 for n in g.files if n.startswith(("g:", "gs:")))
    for name, got, ref in checks:
        assert got.shape == ref.shape, name
        assert rel(got, ref) <= 1e-10, f"{case} {name}: relative L2 {rel(got, ref):.2e}"
