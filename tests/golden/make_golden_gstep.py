"""Generates tests/golden/gstep_{d05,d0,t}_{sq,ns}.npz: the G step of the UNMODIFIED reference VToonify (train_vtoonify_d.py:299-338:
forward with return_mask, a loss on the image and every mask, backward into x, the encoder and the fusion modules) on CPU through its
op_cpu path in float64, with the deterministic weights of vtoonify_b200/weights.py (seed 0) and the seeded inputs, target and mask
weights of tests/oracle_vtoonify_gstep.py.  The reference's own mask loss relu(mean(m_E) - gd_s) can be flat, so every mean(m_E) gets
its own weight instead.  Stored per case: the loss, img[:, :, ::4, ::4], every mask, x.grad[:, :, ::4, ::4], every trained bias
gradient, and for each trained weight gradient every WSTEP-th element of the flattened tensor plus the whole tensor's L2 norm.  Run in
the build container, like make_golden.py, whose reference set-up it reuses:

    python tests/golden/make_golden_gstep.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import RefVToonify, save  # noqa: E402
from tests.oracle_vtoonify_gstep import CASES, GEOMS, WSTEP, image_target, inputs, loss_of, trained  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402


def golden_gstep():
    for case, (backbone, d_s) in CASES.items():
        for geom in GEOMS:
            m = RefVToonify(backbone=backbone)
            m.load_state_dict(det_state_dict(m, seed=0), strict=True)
            m = m.double()
            for n, p in m.named_parameters():
                p.requires_grad_(trained(n))
            x, style = inputs(geom)
            x = x.double().requires_grad_()
            torch.set_default_dtype(torch.float64)      # Fusion builds its d_s label with torch.zeros (model/vtoonify.py:122)
            try:
                r = m(x, style.double(), d_s=d_s, return_mask=True)
            finally:
                torch.set_default_dtype(torch.float32)
            img, masks = r if backbone == "dualstylegan" else (r, [])
            loss = loss_of(img, masks, image_target(img.shape))
            loss.backward()
            out = {"loss": loss.detach(), "img_sub": img.detach()[:, :, ::4, ::4], "x_grad_sub": x.grad[:, :, ::4, ::4]}
            for i, mk in enumerate(masks):
                out[f"mask{i}"] = mk.detach()
            for name, p in m.named_parameters():
                if not trained(name):
                    continue
                if p.dim() == 1:
                    out["g:" + name] = p.grad
                else:
                    out["gs:" + name] = p.grad.flatten()[::WSTEP]
                    out["gn:" + name] = p.grad.norm()
            print(f"gstep_{case}_{geom}: loss {loss.item():.6f}, |x.grad| {x.grad.norm():.3e}")
            save(f"gstep_{case}_{geom}", **out)


if __name__ == "__main__":
    torch.set_grad_enabled(True)        # make_golden switches it off at import
    golden_gstep()
