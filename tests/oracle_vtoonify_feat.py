"""Float64 restatement of VToonify.forward(x, style, d_s, return_feat=True) (model/vtoonify.py:210-244), differentiated with torch
autograd: the oracle of the encoder-pretraining gradients (train_vtoonify_d.py:132-148).  Built from oracle/vt_oracle.py's pieces
and driven by a state_dict.  Test infrastructure only: pinned against the unmodified reference by tests/test_oracle_feat_grad.py
(fixtures tests/golden/feat_grad_*.npz from tests/golden/make_golden_feat_grad.py).  Also holds the case table and the seeded
inputs, shared with the fixture generator and the GPU tests."""
import math

import torch
import torch.nn.functional as F

from oracle import vt_oracle as O
from vtoonify_b200.weights import det_inputs

# case -> (backbone, d_s)
CASES = {"d05": ("dualstylegan", 0.5), "d0": ("dualstylegan", 0.0), "t": ("toonify", 0.5)}
WSTEP = 997          # stride of the stored weight-gradient subsample (flattened)


def case_inputs(B=2, H=64, W=48, seed=0):
    """Seeded network input x [B, 22, H, W] and per-sample W+ styles [B, 18, 512] (fp32, CPU)."""
    x, style = det_inputs(B, H, W, seed=seed)
    g = torch.Generator().manual_seed(4321 + seed)
    return x, style + 0.25 * torch.randn(style.shape, generator=g)


def targets(feat_shape, skip_shape, seed=0):
    g = torch.Generator().manual_seed(8765 + seed)
    return torch.randn(feat_shape, generator=g), torch.randn(skip_shape, generator=g)


def encoder_keys(sd):
    return [k for k in sd if k.startswith("encoder.")]


def feat_forward(sd, x, style, d_s, backbone, in_size=256):
    """-> (feat, skip) of the return_feat path."""
    D = backbone == "dualstylegan"
    if style.ndim < 3:
        style = style.unsqueeze(1).repeat(1, 18, 1)
    if D:
        nB, nL, nD = style.shape
        t = O.pixel_norm(style.reshape(nB * nL, nD))
        for i in (1, 2):
            t = O.equal_linear(t, sd[f"generator.style.{i}.weight"], sd[f"generator.style.{i}.bias"], 0.01, True)
        resstyles = t.reshape(nB, nL, nD)

    def conv(t, key, stride=1, padding=1):
        return F.conv2d(t, sd[key + ".weight"], sd[key + ".bias"], stride=stride, padding=padding)

    n_blocks = int(math.log2(in_size)) - 4
    feat = x
    for bi in range(n_blocks):
        feat = F.leaky_relu(conv(feat, f"encoder.{bi}.0", stride=1 if bi == 0 else 2), 0.2)
        feat = F.leaky_relu(conv(feat, f"encoder.{bi}.2"), 0.2)
    dil = {1: 4, 2: 4, 3: 2, 4: 2, 5: 1, 6: 1}
    for ii in range(6):
        p = f"encoder.{n_blocks}.{ii}."
        out = F.leaky_relu(conv(feat, p + "conv"), 0.2)
        out = F.leaky_relu(conv(out, p + "conv2"), 0.2)
        feat = (out + feat) / math.sqrt(2)
        if D:
            feat = O.ada_res_block(feat, resstyles[:, ii + 1], d_s, sd, f"res.{ii + 1}.", dil[ii + 1])
    return feat, conv(feat, f"encoder.{n_blocks + 1}", padding=0)


def loss_and_grads(sd, x, style, d_s, backbone, t_f, t_s, dtype=torch.float64, x_grad=True):
    """mse(feat, t_f) + mse(skip, t_s) (train_vtoonify_d.py:143) and its gradients, all in ``dtype`` ->
    dict(loss, feat, skip, x_grad, grads={encoder key: gradient})."""
    sd = {k: v.detach().to(dtype).requires_grad_(k.startswith("encoder.")) for k, v in sd.items()}
    x = x.detach().to(dtype).requires_grad_(x_grad)
    with torch.enable_grad():           # test modules may switch grad mode off at import
        feat, skip = feat_forward(sd, x, style.to(x.device, dtype), d_s, backbone)
        loss = F.mse_loss(feat, t_f.to(x.device, dtype)) + F.mse_loss(skip, t_s.to(x.device, dtype))
        loss.backward()
    return {"loss": loss.detach(), "feat": feat.detach(), "skip": skip.detach(), "x_grad": x.grad if x_grad else None,
            "grads": {k: sd[k].grad for k in encoder_keys(sd)}}
