"""Generates tests/golden/feat_grad_{d05,d0,t}.npz: the encoder-pretraining step of the UNMODIFIED reference VToonify
(train_vtoonify_d.py:140-148: forward(return_feat=True), mse_loss on feat and skip, backward) on CPU through its op_cpu path, with
the deterministic weights of vtoonify_b200/weights.py (seed 0) and the seeded inputs and targets of tests/oracle_vtoonify_feat.py.
The reference runs this path in float64 (every module is plain torch), so the fixtures are float64.  Stored per case: the loss,
feat[:, ::8], skip, x.grad[:, :, ::4, ::4], every encoder bias gradient, and for each encoder weight gradient every WSTEP-th element
of the flattened tensor plus the whole tensor's L2 norm.  Run in the build container, like make_golden.py, whose reference set-up
it reuses:

    python tests/golden/make_golden_feat_grad.py
"""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import RefVToonify, save  # noqa: E402
from tests.oracle_vtoonify_feat import CASES, WSTEP, case_inputs, targets  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402


def golden_feat_grad():
    for case, (backbone, d_s) in CASES.items():
        m = RefVToonify(backbone=backbone)
        m.load_state_dict(det_state_dict(m, seed=0), strict=True)
        m = m.double()
        x, style = case_inputs()
        x = x.double().requires_grad_()
        feat, skip = m(x, style.double(), d_s=d_s, return_feat=True)
        t_f, t_s = targets(feat.shape, skip.shape)
        loss = F.mse_loss(feat, t_f.double()) + F.mse_loss(skip, t_s.double())
        loss.backward()
        out = {"loss": loss.detach(), "feat_sub": feat.detach()[:, ::8], "skip": skip.detach(),
               "x_grad_sub": x.grad[:, :, ::4, ::4]}
        for name, p in m.named_parameters():
            if not name.startswith("encoder."):
                continue
            if p.dim() == 1:
                out["g:" + name] = p.grad
            else:
                out["gs:" + name] = p.grad.flatten()[::WSTEP]
                out["gn:" + name] = p.grad.norm()
        print(f"feat_grad_{case}: loss {loss.item():.6f}, |x.grad| {x.grad.norm():.3e}")
        save(f"feat_grad_{case}", **out)


if __name__ == "__main__":
    torch.set_grad_enabled(True)        # make_golden switches it off at import
    golden_feat_grad()
