"""Writes tests/golden/raft_*.npz and state_dict_keys_raft.json from the unmodified reference RAFT (model/raft/core/raft.py) on the
CPU in float32, with det_state_dict weights (non-trivial BatchNorm running statistics).

    python tests/golden/make_golden_raft.py /path/to/reference

Inputs are seeded smooth integer-valued images in 0..255 (stored as uint8); image2 is image1 shifted and slightly rotated, so the
flows are not zero.  Cases (to keep each file small, only part of the larger outputs is stored):
       ``b2``  [2, 3, 128, 160], 3 iterations, test mode: flow_low, and the first UP_ROWS rows of flow_up (the top border and every
               sub-pixel row of 8 flow-field rows, both samples);
       ``init`` [1, 3, 144, 128] with flow_init, 12 iterations, non-test mode: the predictions KEEP of the list;
       ``it20`` [1, 3, 136, 128], 20 iterations, test mode (the smoothing script's setting): flow_low and flow_up.
``raft_lookup.npz``: the reference CorrBlock on random feature maps [1, 16, 17, 21] (level sizes 17x21, 8x10, 4x5, 2x2; odd sides,
no symmetry) at coordinates on pixel centres, fractional, on the border and outside.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from vtoonify_b200.weights import det_state_dict  # noqa: E402


def raft_args(argv=()):
    p = argparse.ArgumentParser()
    p.add_argument("--model")
    p.add_argument("--small", action="store_true")
    p.add_argument("--mixed_precision", action="store_true")
    p.add_argument("--alternate_corr", action="store_true")
    return p.parse_args(["--model", "raft.pth", *argv])


def images(B, H, W, seed):
    """smooth random RGB content in 0..255 and the same content shifted by a few pixels and rotated by ~2 degrees"""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand((B, 3, H // 8 + 3, W // 8 + 3), generator=g), size=(H + 24, W + 24), mode="bicubic",
                         align_corners=False)
    base = base + 0.15 * F.interpolate(torch.rand((B, 3, H // 2 + 6, W // 2 + 6), generator=g), size=(H + 24, W + 24),
                                       mode="bilinear", align_corners=False)
    img1 = base[:, :, 12:12 + H, 12:12 + W]
    th = torch.tensor(0.035)
    theta = torch.tensor([[torch.cos(th), -torch.sin(th), 0.05], [torch.sin(th), torch.cos(th), -0.03]]).expand(B, 2, 3)
    grid = F.affine_grid(theta, (B, 3, H + 24, W + 24), align_corners=False)
    img2 = F.grid_sample(base, grid, mode="bilinear", padding_mode="border", align_corners=False)[:, :, 12:12 + H, 12:12 + W]
    lo, hi = base.min(), base.max()
    return (torch.round((img1 - lo) / (hi - lo) * 255.0).contiguous(),
            torch.round((img2 - lo) / (hi - lo) * 255.0).contiguous())


UP_ROWS = 64            # rows of flow_up stored for the b2 case
KEEP = (0, 5, 11)       # predictions stored for the init case

CASES = {
    "b2": dict(B=2, H=128, W=160, iters=3, test_mode=True, flow_init=False, seed=1),
    "init": dict(B=1, H=144, W=128, iters=12, test_mode=False, flow_init=True, seed=2),
    "it20": dict(B=1, H=136, W=128, iters=20, test_mode=True, flow_init=False, seed=3),
}


def case_inputs(c):
    """float32 images (integer values, as stored) and flow_init of a case"""
    img1, img2 = images(c["B"], c["H"], c["W"], c["seed"])
    fi = None
    if c["flow_init"]:
        g = torch.Generator().manual_seed(100 + c["seed"])
        fi = F.interpolate(2.0 * torch.randn((c["B"], 2, 3, 3), generator=g), size=(c["H"] // 8, c["W"] // 8), mode="bilinear",
                           align_corners=True).contiguous()
    return img1, img2, fi


def main(ref_root):
    sys.path.insert(0, ref_root)
    from model.raft.core.raft import RAFT
    torch.manual_seed(0)
    model = RAFT(raft_args()).eval()
    sd = det_state_dict(model, seed=0)
    model.load_state_dict(sd, strict=True)
    with open(os.path.join(HERE, "state_dict_keys_raft.json"), "w") as f:
        json.dump(list(sd.keys()), f, indent=0)
    from model.raft.core.corr import CorrBlock
    g = torch.Generator().manual_seed(7)
    f1, f2 = torch.randn((1, 16, 17, 21), generator=g), torch.randn((1, 16, 17, 21), generator=g)
    coords = torch.rand((1, 2, 17, 21), generator=g) * torch.tensor([23.0, 19.0]).view(1, 2, 1, 1) - 1.0
    coords[0, :, :4] = torch.floor(coords[0, :, :4])                       # pixel centres
    coords[0, :, 8, :3] = torch.tensor([[-5.5, 0.0, 20.0], [3.0, -4.25, 16.0]])   # outside / on the border
    with torch.no_grad():
        look = CorrBlock(f1, f2, num_levels=4, radius=4)(coords)
    np.savez_compressed(os.path.join(HERE, "raft_lookup.npz"), fmap1=f1.numpy(), fmap2=f2.numpy(), coords=coords.numpy(), corr=look.numpy())
    for name, c in CASES.items():
        img1, img2, fi = case_inputs(c)
        with torch.no_grad():
            out = model(img1, img2, iters=c["iters"], flow_init=fi, test_mode=c["test_mode"])
        arrs = dict(image1=img1.to(torch.uint8).numpy(), image2=img2.to(torch.uint8).numpy())
        if fi is not None:
            arrs["flow_init"] = fi.numpy()
        if name == "b2":
            arrs["flow_low"], arrs["flow_up"] = out[0].numpy(), out[1][:, :, :UP_ROWS].contiguous().numpy()
        elif c["test_mode"]:
            arrs["flow_low"], arrs["flow_up"] = out[0].numpy(), out[1].numpy()
        else:
            arrs["flow_up"] = torch.stack([out[k] for k in KEEP], 0).numpy()
            arrs["n_pred"] = np.array(len(out))
        np.savez_compressed(os.path.join(HERE, f"raft_{name}.npz"), **arrs)
        fu = arrs["flow_up"]
        print(name, {k: v.shape for k, v in arrs.items()}, "mean |flow_up|", float(np.abs(fu).mean()), "nan", bool(np.isnan(fu).any()))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
