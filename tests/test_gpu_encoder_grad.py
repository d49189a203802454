"""GPU: gradients of VToonify.forward(return_feat=True) (encoder pretraining, train_vtoonify_d.py:132-148) against the float64
oracle (tests/oracle_vtoonify_feat.py), the autograd-mode forward against the inference forward, training semantics (Adam steps,
in-place updates, .grad accumulation, hooks, the frozen-path error) and determinism."""
import pytest
import torch
import torch.nn.functional as F

from tests.oracle_vtoonify_feat import CASES, case_inputs, loss_and_grads, targets

pytestmark = pytest.mark.gpu

# Relative L2 and max|err| / max|ref| bars per precision, about 4x the worst values measured on an H100 (printed by the test).
# The gradients of this 28-layer stack are poorly conditioned: PyTorch's own fp32 autograd (cuDNN, TF32 off) lands 2e-3 (d_s 0.5)
# to 4e-3 (d_s 0) in relative L2 from float64 on x.grad, because LeakyReLU gates whose pre-activation is within rounding of 0
# flip and the difference grows towards the input.  The fp32 case is also held to that yardstick directly.
BARS = {"fp32": (2e-2, 6e-2), "bf16x3": (6e-2, 0.3), "tf32": (0.3, 0.5)}


def make_model(backbone):
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict
    m = VToonify(backbone=backbone)
    m.load_state_dict(det_state_dict(m, seed=0), strict=True)
    m = m.cuda()
    if backbone == "dualstylegan":
        m.res.requires_grad_(False)                 # the frozen path, as train_vtoonify_d.py:425-428
    m.generator.requires_grad_(False)
    return m


@pytest.fixture(scope="module")
def models():
    return {b: make_model(b) for b in ("dualstylegan", "toonify")}


def inputs(B=2, H=64, W=48):
    x, style = case_inputs(B, H, W)
    t_f, t_s = targets((B, 512, H // 8, W // 8), (B, 3, H // 8, W // 8))
    return x.cuda(), style.cuda(), t_f.cuda(), t_s.cuda()


def lib_step(m, x, style, d_s, t_f, t_s, x_grad=True):
    m.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(x_grad)
    with torch.enable_grad():
        feat, skip = m(x, style, d_s=d_s, return_feat=True)
        loss = F.mse_loss(feat, t_f) + F.mse_loss(skip, t_s)
        loss.backward()
    grads = {n: p.grad.clone() for n, p in m.named_parameters() if n.startswith("encoder.")}
    return loss.detach(), feat.detach(), skip.detach(), x.grad, grads


def errs(got, ref):
    d = (got.double() - ref.double()).flatten()
    return (d.norm() / ref.double().norm()).item(), (d.abs().max() / ref.double().abs().max()).item()


CASE_PREC = [(c, p) for c in CASES for p in ("fp32", "bf16x3", "tf32")] + [("d05@256", "bf16x3")]


@pytest.mark.parametrize("case,prec", CASE_PREC)
def test_gradients_vs_float64_oracle(models, case, prec):
    from vtoonify_b200 import ops
    big = case.endswith("@256")
    backbone, d_s = CASES[case.split("@")[0]]
    m = models[backbone]
    x, style, t_f, t_s = inputs(2, 256, 256) if big else inputs()
    sd = {k: v.cuda() for k, v in m.state_dict().items()}
    ref = loss_and_grads(sd, x, style, d_s, backbone, t_f, t_s)
    old = ops.set_precision(prec)
    try:
        loss, feat, skip, gx, grads = lib_step(m, x, style, d_s, t_f, t_s)
    finally:
        ops.set_precision(old)
    assert set(grads) == set(ref["grads"])
    assert all(p.grad is None for p in list(m.fusion_out.parameters()) + list(m.fusion_skip.parameters()))
    worst = (0.0, 0.0)
    rows = [("feat", feat, ref["feat"]), ("skip", skip, ref["skip"]), ("x.grad", gx, ref["x_grad"])]
    rows += [(k, grads[k], ref["grads"][k]) for k in ref["grads"]]
    lines, bad = [], []
    for name, got, want in rows:
        e = errs(got, want)
        worst = (max(worst[0], e[0]), max(worst[1], e[1]))
        lines.append(f"  {name:28s} rel L2 {e[0]:.2e}  max/max {e[1]:.2e}")
        if e[0] > BARS[prec][0] or e[1] > BARS[prec][1]:
            bad.append(name)
    print(f"\n{case} {prec}: loss {loss.item():.6f} vs {ref['loss'].item():.6f}; worst rel L2 {worst[0]:.2e}, "
          f"worst max/max {worst[1]:.2e}\n" + "\n".join(lines))
    assert not bad, f"{case} {prec}: above the bars: {bad}"
    if prec == "fp32" and not big:
        torch.backends.cudnn.allow_tf32 = False
        try:
            r32 = loss_and_grads(sd, x, style, d_s, backbone, t_f, t_s, dtype=torch.float32)
        finally:
            torch.backends.cudnn.allow_tf32 = True
        e_lib, e_torch = errs(gx, ref["x_grad"])[0], errs(r32["x_grad"], ref["x_grad"])[0]
        print(f"  x.grad rel L2: library fp32 {e_lib:.2e}, PyTorch fp32 autograd {e_torch:.2e}")
        assert e_lib <= 4 * e_torch


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
@pytest.mark.parametrize("case", list(CASES))
def test_autograd_forward_matches_inference(models, case, prec):
    from vtoonify_b200 import _lib, ops
    backbone, d_s = CASES[case]
    m = models[backbone]
    x, style, _, _ = inputs()
    old = ops.set_precision(prec)
    try:
        with torch.no_grad():
            m(x, style, d_s=d_s, return_feat=True)          # style-only tensors are cached from here on
            n0 = _lib.launch_count()
            f0, s0 = m(x, style, d_s=d_s, return_feat=True)
            n_nograd = _lib.launch_count() - n0
        with torch.enable_grad():
            f1, s1 = m(x.clone().requires_grad_(), style, d_s=d_s, return_feat=True)
            assert f1.grad_fn is not None and s1.grad_fn is not None
            # grad mode with nothing that requires grad: the inference route, the same launches
            m.encoder.requires_grad_(False)
            try:
                n0 = _lib.launch_count()
                f2, s2 = m(x, style, d_s=d_s, return_feat=True)
                n_frozen = _lib.launch_count() - n0
            finally:
                m.encoder.requires_grad_(True)
    finally:
        ops.set_precision(old)
    assert f2.grad_fn is None and torch.equal(f2, f0) and torch.equal(s2, s0) and n_frozen == n_nograd
    ef = (f1.detach() - f0).abs().max().item() / f0.abs().max().item()
    es = (s1.detach() - s0).abs().max().item() / s0.abs().max().item()
    print(f"\n{case} {prec}: autograd-mode forward vs inference: feat {ef:.2e}, skip {es:.2e} (of max); {n_nograd} launches")
    if prec == "bf16x3" and CASES[case] == ("dualstylegan", 0.5):
        # the inference route takes each ModRes block's input statistics from the epilogue of the res block's last convolution, which
        # also adds the residual; the autograd route keeps that convolution's activation, adds the residual in its own pass and runs
        # the statistics pass over the sum (measured on an H100: 8.9e-6 of max|feat|, 1.3e-5 of max|skip|)
        assert ef <= 5e-5 and es <= 5e-5
    else:
        assert torch.equal(f1.detach(), f0) and torch.equal(s1.detach(), s0)      # the same operations in the same order


def test_adam_steps_track_the_oracle_and_updates_reach_the_forward(models):
    """Two Adam steps (betas (0.9, 0.99), train_vtoonify_d.py:438) on the library model and on the float64 oracle."""
    from vtoonify_b200.vtoonify import VToonify
    m = make_model("dualstylegan")
    x, style, t_f, t_s = inputs()
    d_s = 0.5
    enc = [(n, p) for n, p in m.named_parameters() if n.startswith("encoder.")]
    sd = {k: v.detach().clone().double() for k, v in m.state_dict().items()}
    leaves = {n: sd[n].requires_grad_() for n, _ in enc}
    opt_l = torch.optim.Adam([p for _, p in enc], lr=1e-4, betas=(0.9, 0.99))
    opt_o = torch.optim.Adam(list(leaves.values()), lr=1e-4, betas=(0.9, 0.99))
    losses = []
    for step in range(2):
        loss, feat, _, _, _ = lib_step(m, x, style, d_s, t_f, t_s, x_grad=False)
        opt_l.step()
        opt_o.zero_grad()
        from tests.oracle_vtoonify_feat import feat_forward
        with torch.enable_grad():
            f_o, s_o = feat_forward(sd, x.double(), style.double(), d_s, "dualstylegan")
            loss_o = F.mse_loss(f_o, t_f.double()) + F.mse_loss(s_o, t_s.double())
            loss_o.backward()
        opt_o.step()
        losses.append((loss.item(), loss_o.item()))
    # Adam's first step moves every element by lr * sign(grad): an element whose gradient is within rounding of 0 may step the other
    # way, so the updates are compared in L2 over each tensor
    init = {k: v.double() for k, v in make_model("dualstylegan").state_dict().items()}
    worst_p = worst_d = 0.0
    for n, p in enc:
        p0, d_o = sd[n].detach(), sd[n].detach() - init[n]
        worst_p = max(worst_p, ((p.detach().double() - p0).norm() / p0.norm()).item())
        worst_d = max(worst_d, ((p.detach().double() - init[n] - d_o).norm() / d_o.norm()).item())
    print(f"\nAdam x2: losses {losses}; worst relative difference of the parameters {worst_p:.2e}, of the updates {worst_d:.2e}")
    # measured on an H100 (bf16x3): 1.2e-3 and 0.17; the losses of both steps agree to 2e-4
    assert worst_p <= 5e-3 and worst_d <= 0.5
    assert all(abs(a - b) <= 1e-3 * b for a, b in losses)
    # the in-place optimizer updates reach the next forward: cached (prepped / split) weights key on _version
    with torch.no_grad():
        fresh = VToonify(backbone="dualstylegan").cuda()
        fresh.load_state_dict(m.state_dict())
        f_a, s_a = m(x, style, d_s=d_s, return_feat=True)
        f_b, s_b = fresh(x, style, d_s=d_s, return_feat=True)
    assert torch.equal(f_a, f_b) and torch.equal(s_a, s_b)


def test_short_pretraining_run_lowers_the_loss(models):
    m = make_model("dualstylegan")
    x, style, t_f, t_s = inputs()
    opt = torch.optim.Adam([p for n, p in m.named_parameters() if n.startswith("encoder.")], lr=1e-4, betas=(0.9, 0.99))
    losses = []
    for i in range(6):
        loss = lib_step(m, x, style, 0.5, t_f, t_s, x_grad=False)[0]
        opt.step()
        losses.append(round(loss.item(), 5))
    print(f"\nloss over a short run: {losses}")
    assert all(b < a for a, b in zip(losses, losses[1:]))


def test_grad_accumulates_hooks_fire_and_backward_is_deterministic(models):
    m = models["dualstylegan"]
    x, style, t_f, t_s = inputs()
    calls = []
    h = m.encoder[0][0].weight.register_hook(lambda g: calls.append(1))
    try:
        m.zero_grad(set_to_none=True)
        once = {}
        for rep in range(2):
            with torch.enable_grad():
                feat, skip = m(x, style, d_s=0.5, return_feat=True)
                (F.mse_loss(feat, t_f) + F.mse_loss(skip, t_s)).backward()
            if rep == 0:
                once = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
        assert len(calls) == 2
        for n, p in m.named_parameters():
            if n in once:
                assert torch.equal(p.grad, 2 * once[n]), n       # same bits each time: the sum is exactly twice
    finally:
        h.remove()
    a = lib_step(m, x, style, 0.5, t_f, t_s)
    b = lib_step(m, x, style, 0.5, t_f, t_s)
    assert torch.equal(a[3], b[3]) and all(torch.equal(a[4][k], b[4][k]) for k in a[4])


def test_frozen_path_requiring_grad_raises(models):
    m = models["dualstylegan"]
    x, style, _, _ = inputs()
    with torch.enable_grad():
        m.res[1].conv[0].weight.requires_grad_(True)
        try:
            with pytest.raises(NotImplementedError, match=r"res\.1\.conv\.0\.weight.*requires_grad_\(False\)"):
                m(x, style, d_s=0.5, return_feat=True)
        finally:
            m.res[1].conv[0].weight.requires_grad_(False)
        with pytest.raises(NotImplementedError, match="style"):
            m(x, style.clone().requires_grad_(), d_s=0.5, return_feat=True)
        feat, _ = m(x, style.clone().requires_grad_(), d_s=0, return_feat=True)     # d_s = 0: no frozen tensor on the path
        assert feat.grad_fn is not None
