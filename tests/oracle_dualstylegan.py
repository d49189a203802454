"""CPU restatement of DualStyleGAN.forward (model/dualstylegan.py:84-194), driven by its state_dict and built from the
oracle's StyleGAN2 / ModRes pieces.  Test infrastructure only: pinned against the unmodified reference by
tests/test_oracle_dualstylegan.py (fixture tests/golden/dualstylegan64.npz from tests/golden/make_golden_dualstylegan.py).
Also holds the fixture's case table, shared with the GPU test."""
import json
import re

import numpy as np
import torch

from oracle import vt_oracle as O
from vtoonify_b200.weights import det_state_dict


def mapping(sd, z, prefix):
    """PixelNorm + the EqualLinear(lr_mul 0.01, fused_lrelu) stack ``{prefix}1..n`` (model/stylegan/model.py:409-417)."""
    t = O.pixel_norm(z)
    i = 1
    while f"{prefix}{i}.weight" in sd:
        t = O.equal_linear(t, sd[f"{prefix}{i}.weight"], sd[f"{prefix}{i}.bias"], 0.01, True)
        i += 1
    return t


def dualstylegan_forward(sd, styles, exstyles, noises, return_feat=False, inject_index=None, truncation=1,
                         truncation_latent=None, input_is_latent=False, z_plus_latent=False, use_res=True, fuse_index=18,
                         interp_weights=(1,) * 18, res_index=6):
    """``noises``: one tensor per generator layer (randomize_noise=False passes the stored buffers).  Returns the image, or
    ``(feat, skip)`` with ``return_feat``."""
    g = "generator."
    n_levels = len([k for k in sd if re.fullmatch(r"generator\.to_rgbs\.\d+\.bias", k)])
    n_latent = 2 * (n_levels + 2) - 2
    if not input_is_latent:
        styles = [mapping(sd, s.reshape(-1, s.shape[-1]), g + "style.").reshape(s.shape) for s in styles]
    if truncation < 1:
        styles = [truncation_latent + truncation * (s - truncation_latent) for s in styles]

    def widen(s, n):
        return s.unsqueeze(1).repeat(1, n, 1) if s.ndim < 3 else s
    if len(styles) < 2:
        latent = widen(styles[0], n_latent)
    elif styles[0].ndim < 3:
        latent = torch.cat([widen(styles[0], inject_index), widen(styles[1], n_latent - inject_index)], 1)
    else:
        latent = torch.cat([styles[0][:, :inject_index], styles[1][:, inject_index:]], 1)
    if use_res:
        adastyles = widen(exstyles, n_latent)
        resstyles = mapping(sd, adastyles.reshape(-1, adastyles.shape[-1]), "style.").reshape(adastyles.shape)

    def modres(x, j):
        if use_res and fuse_index >= max(j, 1) and j <= res_index:
            return O.ada_res_block(x, resstyles[:, j], interp_weights[j], sd, f"res.{j}.", 1)
        return x

    def style(j):
        if use_res and fuse_index >= j and j > res_index:
            t = O.equal_linear(adastyles[:, j], sd[f"res.{j}.weight"], sd[f"res.{j}.bias"])
            return interp_weights[j] * t + (1 - interp_weights[j]) * latent[:, j]
        return latent[:, j]

    B = latent.shape[0]
    out = sd[g + "input.input"].repeat(B, 1, 1, 1)
    out = modres(O.styled_conv(out, latent[:, 0], sd, g + "conv1.", noises[0]), 0)
    skip = O.to_rgb(out, latent[:, 1], sd, g + "to_rgb1.")
    i = 1
    for lv in range(n_levels):
        out = modres(O.styled_conv(out, style(i), sd, f"{g}convs.{2 * lv}.", noises[i], upsample=True), i)
        out = modres(O.styled_conv(out, style(i + 1), sd, f"{g}convs.{2 * lv + 1}.", noises[i + 1]), i + 1)
        skip = O.to_rgb(out, style(i + 2), sd, f"{g}to_rgbs.{lv}.", skip)
        i += 2
        if return_feat and i > res_index:
            return out, skip
    return skip


# ---------------------------------------------------------------------------------------------- the fixture's cases
W_RES = [0.6] * 7 + [1.0] * 3
W_FIX_COLOR = [0.6] * 7 + [0.0] * 3
KEYS = "tests/golden/state_dict_keys_dualstylegan64.json"

# fixture key -> (forward keyword arguments, the inputs by fixture name); every case runs with the stored noise buffers
CASES = {
    "res": (dict(input_is_latent=True, interp_weights=W_RES), ("latent", "exstyles")),
    "fix_color": (dict(input_is_latent=True, interp_weights=W_FIX_COLOR), ("latent", "exstyles")),
    "fuse4": (dict(input_is_latent=True, fuse_index=4, interp_weights=W_RES), ("latent", "exstyles")),
    "nores": (dict(input_is_latent=True, use_res=False), ("latent", "exstyles")),
    "feat": (dict(input_is_latent=True, return_feat=True, truncation=0.5, truncation_latent=0, interp_weights=W_RES),
             ("latent", "exstyles")),
    "zplus_y": (dict(z_plus_latent=True, interp_weights=W_RES), ("zplus", "exstyles")),
    "mix": (dict(input_is_latent=True, inject_index=4, interp_weights=W_RES), ("w1", "w2", "ex2")),
}


def T(a):
    return torch.from_numpy(np.asarray(a))


def state_dict():
    """the fixture's deterministic weights, rebuilt from the reference's key list"""
    sd = det_state_dict({k: torch.empty(v) for k, v in json.load(open(KEYS)).items()}, seed=5)
    for k in sd:
        if k.endswith("blur.kernel") or k.endswith("upsample.kernel"):
            sd[k] = O.make_kernel([1, 3, 3, 1]) * 4      # FIR buffers are architecture constants
    return sd


def case_inputs(g, names):
    """-> (styles list, exstyles)"""
    *styles, ex = [T(g[n]) for n in names]
    return styles, ex


def case_outputs(g, name):
    return (T(g["feat_sub"]), T(g["feat_skip"])) if name == "feat" else (T(g[name]),)
