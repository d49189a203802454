"""Generates tests/golden/dualstylegan64.npz and state_dict_keys_dualstylegan64.json: outputs of the UNMODIFIED reference
DualStyleGAN(64, 512, 8).forward (model/dualstylegan.py:84-194) on CPU through its op_cpu path, with the deterministic weights
of vtoonify_b200/weights.py (seed 5) and the stored noise buffers.  Size 64 has 10 latents: ModRes blocks at 4², 8², 16² and
32² (layers 0-6) and the structure transform T_s (EqualLinear) on layers 7-9.  Run in the build container, like
make_golden.py, whose reference set-up it reuses:

    python tests/golden/make_golden_dualstylegan.py
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, gen, ref_dual, save  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402

W_RES = [0.6] * 7 + [1.0] * 3          # interp_weights: d_s on the ModRes layers, 1 on the colour layers
W_FIX_COLOR = [0.6] * 7 + [0.0] * 3    # the fix_color form: colour layers keep the intrinsic code


def golden_dualstylegan():
    m = ref_dual.DualStyleGAN(64, 512, 8).eval()
    keys = {k: list(v.shape) for k, v in m.state_dict().items()}
    with open(os.path.join(HERE, "state_dict_keys_dualstylegan64.json"), "w") as f:
        json.dump(keys, f, indent=0)
    m.load_state_dict(det_state_dict(m, seed=5), strict=True)
    g = gen(64)
    B, L = 2, m.n_latent
    latent = torch.randn((B, L, 512), generator=g)
    exstyles = torch.randn((B, L, 512), generator=g)
    zplus = torch.randn((B, L, 512), generator=g)
    w1, w2 = torch.randn((B, 512), generator=g), torch.randn((B, 512), generator=g)
    ex2 = torch.randn((B, 512), generator=g)
    out = {"latent": latent, "exstyles": exstyles, "zplus": zplus, "w1": w1, "w2": w2, "ex2": ex2}
    kw = dict(input_is_latent=True, randomize_noise=False)
    out["res"] = m([latent], exstyles, interp_weights=W_RES, **kw)[0]
    out["fix_color"] = m([latent], exstyles, interp_weights=W_FIX_COLOR, **kw)[0]
    out["fuse4"] = m([latent], exstyles, fuse_index=4, interp_weights=W_RES, **kw)[0]
    out["nores"] = m([latent], exstyles, use_res=False, **kw)[0]
    feat, skip = m([latent], exstyles, return_feat=True, truncation=0.5, truncation_latent=0, interp_weights=W_RES, **kw)
    out["feat_sub"], out["feat_skip"] = feat[:, ::32], skip      # every 32nd channel: the whole map alone is 4 MB
    out["zplus_y"] = m([zplus], exstyles, z_plus_latent=True, randomize_noise=False, interp_weights=W_RES)[0]
    out["mix"] = m([w1, w2], ex2, inject_index=4, interp_weights=W_RES, **kw)[0]
    # both extrinsic paths really act on the output
    for name in ("fix_color", "nores"):
        print(f"dualstylegan64 {name}: max |y - res| {(out[name] - out['res']).abs().max():.3f}")
    print("dualstylegan64 rms %.3f, feat %s" % (out["res"].pow(2).mean().sqrt(), tuple(feat.shape)))
    save("dualstylegan64", **out)


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    golden_dualstylegan()
