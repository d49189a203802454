"""Generates tests/golden/lpips_{sq,odd,both}.npz and state_dict_keys_lpips.json: the UNMODIFIED reference PNetLin
(model/stylegan/lpips/networks_basic.py, VGG16 net-lin, pnet_rand=True so torchvision downloads nothing) in float64 on the CPU, with
the deterministic weights of vtoonify_b200/weights.py (seed 0) and the seeded inputs of tests/oracle_lpips.py.  The LPIPS modules import
skimage and IPython at the top without calling them on this path, so those imports are stubbed.  Stored per case: pred, target, the
loss [B, 1, 1, 1] and the gradients of sum_b weight_b * loss_b.  Run where the reference checkout is:

    python tests/golden/make_golden_lpips.py
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")

for name in ("skimage", "skimage.color", "skimage.transform", "skimage.metrics", "IPython"):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules["skimage"].color = sys.modules["skimage.color"]
sys.modules["skimage"].transform = sys.modules["skimage.transform"]
sys.modules["skimage.metrics"].structural_similarity = None
sys.modules["IPython"].embed = None

from model.stylegan.lpips.networks_basic import PNetLin  # noqa: E402

from tests.oracle_lpips import CASES, inputs, loss_weights  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402


def main():
    net = PNetLin(pnet_rand=True, pnet_tune=False, pnet_type="vgg", use_dropout=True, spatial=False, version="0.1", lpips=True)
    net.load_state_dict(det_state_dict(net, seed=0), strict=True)
    net = net.eval().double()
    keys = list(net.state_dict().keys())
    with open(os.path.join(HERE, "state_dict_keys_lpips.json"), "w") as f:
        json.dump(keys, f, indent=0)
    print(f"state_dict_keys_lpips.json: {len(keys)} keys")
    for name, (shape, seed, g_pred, g_target) in CASES.items():
        pred, target = inputs(shape, seed)
        pred.requires_grad_(g_pred)
        target.requires_grad_(g_target)
        loss = net(target, pred)                     # PerceptualLoss.forward(pred, target) = DistModel.forward(target, pred)
        (loss.flatten() * loss_weights(shape[0], seed)).sum().backward()
        out = {"pred": pred.detach(), "target": target.detach(), "loss": loss.detach()}
        if g_pred:
            out["pred_grad"] = pred.grad
        if g_target:
            out["target_grad"] = target.grad
        out = {k: v.numpy() for k, v in out.items()}
        path = os.path.join(HERE, f"lpips_{name}.npz")
        np.savez_compressed(path, **out)
        print(f"lpips_{name}.npz  {os.path.getsize(path) / 1024:.0f} KiB  loss {loss.flatten().tolist()}")


if __name__ == "__main__":
    main()
