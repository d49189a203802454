"""GPU: gradients of VToonify.forward(x, style, d_s, return_mask=True) (the G step, train_vtoonify_d.py:299-338, train_vtoonify_t.py:
242-270) against the float64 oracle (tests/oracle_vtoonify_gstep.py), the autograd-mode forward against inference, training semantics
(.grad accumulation, hooks, needs_input_grad, the frozen-path error, Adam steps) and a training-size G step with the discriminator."""
import pytest
import torch
import torch.nn.functional as F

from tests.oracle_vtoonify_gstep import CASES, image_target, inputs, loss_and_grads, loss_of, trained

pytestmark = pytest.mark.gpu

# Relative L2 bars per precision, about 4x the worst values measured on an H100 (printed by the test).  As for the encoder (DESIGN §6)
# LeakyReLU gates whose pre-activation is within rounding of 0 flip, so the gradients towards x are the least accurate; the fp32 case
# is also held to PyTorch's own fp32 autograd yardstick (cuDNN, TF32 off) directly.
# Measured (DESIGN §8): fp32 2.2e-4, bf16x3 2.2e-2, tf32 9.6e-2; the batch-2 training-size step 2.6e-2 (bf16x3).
BARS = {"fp32": 1e-3, "bf16x3": 9e-2, "tf32": 0.4}
STEP_BAR = 0.1


def make_model(backbone):
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict
    m = VToonify(backbone=backbone)
    m.load_state_dict(det_state_dict(m, seed=0), strict=True)
    m = m.cuda()
    m.generator.requires_grad_(False)
    if backbone == "dualstylegan":
        m.res.requires_grad_(False)
    return m


@pytest.fixture(scope="module")
def models():
    return {b: make_model(b) for b in ("dualstylegan", "toonify")}


def cuda_inputs(geom="sq"):
    x, style = inputs(geom)
    return x.cuda(), style.cuda()


def lib_step(m, x, style, d_s, x_grad=True):
    m.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(x_grad)
    with torch.enable_grad():
        r = m(x, style, d_s=d_s, return_mask=True)
        img, masks = r if m.backbone == "dualstylegan" else (r, [])
        loss = loss_of(img, masks, image_target(img.shape).cuda())
        loss.backward()
    grads = {n: p.grad.clone() for n, p in m.named_parameters() if trained(n) and p.grad is not None}
    return loss.detach(), img.detach(), [k.detach() for k in masks], x.grad, grads


def rel(got, ref):
    return ((got.double() - ref.double()).norm() / ref.double().norm()).item()


CASE_PREC = [(c, p) for c in CASES for p in ("fp32", "bf16x3", "tf32")] + [("d05@ns", "bf16x3"), ("t@ns", "fp32")]


@pytest.mark.parametrize("case,prec", CASE_PREC)
def test_gradients_vs_float64_oracle(models, case, prec):
    """x [2, 22, 32, 32], and for two cases the non-square [1, 22, 48, 40] (``@ns``)."""
    from vtoonify_b200 import ops
    name, _, geom = case.partition("@")
    backbone, d_s = CASES[name]
    m = models[backbone]
    x, style = cuda_inputs(geom or "sq")
    sd = {k: v.cuda() for k, v in m.state_dict().items()}
    ref = loss_and_grads(sd, x, style, d_s, backbone)
    old = ops.set_precision(prec)
    try:
        loss, img, masks, gx, grads = lib_step(m, x, style, d_s)
    finally:
        ops.set_precision(old)
    assert set(grads) == set(ref["grads"])
    assert all(p.grad is None for n, p in m.named_parameters() if not trained(n))
    rows = [("img", img, ref["img"]), ("x.grad", gx, ref["x_grad"])]
    rows += [(f"mask{i}", a, b) for i, (a, b) in enumerate(zip(masks, ref["masks"]))]
    rows += [(k, grads[k], ref["grads"][k]) for k in ref["grads"] if ref["grads"][k].norm() > 0]
    errs = [(name, rel(got, want)) for name, got, want in rows]
    worst = max(e for _, e in errs)
    print(f"\n{case} {prec}: loss {loss.item():.6f} vs {ref['loss'].item():.6f}; worst rel L2 {worst:.2e}\n" +
          "\n".join(f"  {n:36s} {e:.2e}" for n, e in sorted(errs, key=lambda t: -t[1])[:8]))
    bad = [n for n, e in errs if e > BARS[prec]]
    assert not bad, f"{case} {prec}: above the bar: {bad}"
    if prec == "fp32":
        torch.backends.cudnn.allow_tf32 = False
        try:
            r32 = loss_and_grads(sd, x, style, d_s, backbone, dtype=torch.float32)
        finally:
            torch.backends.cudnn.allow_tf32 = True
        e_lib = max(rel(grads[k], ref["grads"][k]) for k in ref["grads"] if ref["grads"][k].norm() > 0)
        e_torch = max(rel(r32["grads"][k], ref["grads"][k]) for k in ref["grads"] if ref["grads"][k].norm() > 0)
        ex_lib, ex_torch = rel(gx, ref["x_grad"]), rel(r32["x_grad"], ref["x_grad"])
        print(f"  worst parameter rel L2: library fp32 {e_lib:.2e}, PyTorch fp32 autograd {e_torch:.2e}; "
              f"x.grad: {ex_lib:.2e} vs {ex_torch:.2e}")
        assert e_lib <= 4 * e_torch and ex_lib <= 4 * ex_torch


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
@pytest.mark.parametrize("case", list(CASES))
def test_autograd_forward_matches_inference(models, case, prec):
    from vtoonify_b200 import ops
    backbone, d_s = CASES[case]
    m = models[backbone]
    x, style = cuda_inputs("ns")
    old = ops.set_precision(prec)
    try:
        with torch.no_grad():
            r0 = m(x, style, d_s=d_s, return_mask=True)
        with torch.enable_grad():
            r1 = m(x.clone().requires_grad_(), style, d_s=d_s, return_mask=True)
    finally:
        ops.set_precision(old)
    i0, k0 = r0 if backbone == "dualstylegan" else (r0, [])
    i1, k1 = r1 if backbone == "dualstylegan" else (r1, [])
    assert i1.grad_fn is not None and all(k.grad_fn is not None for k in k1)
    ei = (i1.detach() - i0).abs().max().item() / i0.abs().max().item()
    ek = max([(a.detach() - b).abs().max().item() for a, b in zip(k1, k0)] + [0.0])
    print(f"\n{case} {prec}: autograd-mode forward vs inference: image {ei:.2e} of max, masks {ek:.2e}")
    if prec == "fp32":
        assert torch.equal(i1.detach(), i0) and all(torch.equal(a.detach(), b) for a, b in zip(k1, k0))
    else:
        # bf16x3 inference multiplies f_E by m_E while the fusion convolutions stage their tiles and takes the ModRes statistics from
        # an epilogue; the autograd route writes f_E * m_E and runs the separate statistics pass
        assert ei <= 1e-4 and ek <= 1e-4


def test_accumulation_hooks_determinism_and_needs_input_grad(models):
    from vtoonify_b200 import _lib
    m = models["dualstylegan"]
    x, style = cuda_inputs()
    calls = []
    h = m.fusion_out[1].conv2.weight.register_hook(lambda g: calls.append(1))
    try:
        m.zero_grad(set_to_none=True)
        once = {}
        for rep in range(2):
            with torch.enable_grad():
                img, masks = m(x, style, d_s=0.5, return_mask=True)
                loss_of(img, masks, image_target(img.shape).cuda()).backward()
            if rep == 0:
                once = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
        assert len(calls) == 2
        for n, p in m.named_parameters():
            if n in once:
                assert torch.equal(p.grad, 2 * once[n]), n
    finally:
        h.remove()
    a = lib_step(m, x, style, 0.5)
    b = lib_step(m, x, style, 0.5)
    assert torch.equal(a[3], b[3]) and all(torch.equal(a[4][k], b[4][k]) for k in a[4])
    # x frozen: encoder.0.0 computes no input gradient (fewer launches, x.grad stays None), the parameter gradients are unchanged
    counts = []
    for xg in (True, False):
        n0 = _lib.launch_count()
        r = lib_step(m, x, style, 0.5, x_grad=xg)
        counts.append(_lib.launch_count() - n0)
    assert r[3] is None and counts[1] < counts[0]
    assert all(torch.equal(r[4][k], a[4][k]) for k in a[4])


def test_frozen_path_requiring_grad_raises(models):
    m = models["dualstylegan"]
    x, style = cuda_inputs()
    with torch.enable_grad():
        for name, t in (("generator.generator.convs.6.conv.weight", m.generator.generator.convs[6].conv.weight),
                        ("res.1.conv.0.weight", m.res[1].conv[0].weight)):
            t.requires_grad_(True)
            try:
                with pytest.raises(NotImplementedError, match=name.replace(".", r"\.")):
                    m(x, style, d_s=0.5)
            finally:
                t.requires_grad_(False)
        with pytest.raises(NotImplementedError, match="style"):
            m(x, style.clone().requires_grad_(), d_s=0.5)
    with torch.no_grad():
        assert m(x, style, d_s=0.5).grad_fn is None


def test_adam_steps_track_the_oracle_and_updates_reach_the_forward():
    """Two Adam steps (betas (0.9, 0.99), train_vtoonify_d.py:438) on the library model and on the float64 oracle."""
    from vtoonify_b200.vtoonify import VToonify
    from tests.oracle_vtoonify_gstep import O
    m = make_model("dualstylegan")
    x, style = cuda_inputs()
    d_s = 0.5
    tr = [(n, p) for n, p in m.named_parameters() if trained(n)]
    sd = {k: v.detach().clone().double() for k, v in m.state_dict().items()}
    leaves = {n: sd[n].requires_grad_() for n, _ in tr}
    opt_l = torch.optim.Adam([p for _, p in tr], lr=1e-4, betas=(0.9, 0.99))
    opt_o = torch.optim.Adam(list(leaves.values()), lr=1e-4, betas=(0.9, 0.99))
    target = image_target((2, 3, 128, 128)).cuda()
    losses = []
    for step in range(2):
        loss = lib_step(m, x, style, d_s, x_grad=False)[0]
        opt_l.step()
        opt_o.zero_grad()
        torch.set_default_dtype(torch.float64)
        try:
            with torch.enable_grad():
                img, masks = O.vtoonify_forward(sd, x.double(), style.double(), d_s, "dualstylegan", return_mask=True)
                loss_o = loss_of(img, masks, target)
                loss_o.backward()
        finally:
            torch.set_default_dtype(torch.float32)
        opt_o.step()
        losses.append((loss.item(), loss_o.item()))
    init = {k: v.double() for k, v in make_model("dualstylegan").state_dict().items()}
    worst_p = worst_d = 0.0
    for n, p in tr:
        p0, d_o = sd[n].detach(), sd[n].detach() - init[n]
        if d_o.norm() == 0:
            continue
        worst_p = max(worst_p, ((p.detach().double() - p0).norm() / p0.norm()).item())
        worst_d = max(worst_d, ((p.detach().double() - init[n] - d_o).norm() / d_o.norm()).item())
    print(f"\nAdam x2: losses {losses}; worst relative difference of the parameters {worst_p:.2e}, of the updates {worst_d:.2e}")
    # Measured on an H100 (bf16x3): parameters 8.8e-4, losses 1.8e-5 and 4.5e-4 apart; bars about 4x.  Adam moves every element by
    # about lr whatever its gradient's size (it normalises by sqrt(v)), so an element whose gradient is within rounding of 0 may step
    # the other way, and the second step's gradients are then taken at slightly different parameters.  The updates' difference (0.33)
    # counts such elements rather than the gradients' precision, so it is only required to stay below 1: updates correlated with the
    # oracle's (DESIGN §8).
    assert worst_p <= 5e-3 and worst_d < 1.0
    assert all(abs(a - b) <= 2e-3 * b for a, b in losses)
    with torch.no_grad():
        fresh = VToonify(backbone="dualstylegan").cuda()
        fresh.load_state_dict(m.state_dict())
        ia, ma = m(x, style, d_s=d_s, return_mask=True)
        ib, mb = fresh(x, style, d_s=d_s, return_mask=True)
    assert torch.equal(ia, ib) and all(torch.equal(a, b) for a, b in zip(ma, mb))


def _g_step(m, D, x, style, d_s, degree, style_ind):
    """The G step's structure (train_vtoonify_d.py:299-338): the model at 256^2 and on the 224^2 crop of the 896^2 frame (down(down(.)))
    as a second call, the conditional discriminator's adversarial loss on the first output, an image loss and the mask terms."""
    with torch.enable_grad():
        img, masks = m(x, style, d_s=d_s, return_mask=True)
        crop = x[:, :, 16:240, 16:240].contiguous()
        img2, masks2 = m(crop, style, d_s=d_s, return_mask=True)
        adv = F.softplus(-D(F.adaptive_avg_pool2d(img, 256), degree, style_ind)).mean()
        loss = adv + loss_of(img2, masks2, image_target(img2.shape).to(img2)) + sum(w * k.mean() for w, k in zip((0.2, 0.4), masks))
        loss.backward()
    return loss.detach()


def test_training_size_g_step_runs_and_matches_the_oracle_at_batch_2():
    from vtoonify_b200 import ops
    from vtoonify_b200.vtoonify import ConditionalDiscriminator
    from vtoonify_b200.weights import det_inputs, det_state_dict
    m = make_model("dualstylegan")
    D = ConditionalDiscriminator(256, use_condition=True, style_num=4)
    D.load_state_dict(det_state_dict(D, seed=3))
    D = D.cuda().requires_grad_(False)
    x8, style8 = det_inputs(8, 256, 256, seed=2)
    x8, style8 = x8.cuda(), style8.cuda()
    deg, ind = torch.full((8, 1), 0.5, device="cuda"), torch.arange(8, device="cuda") % 4
    m.zero_grad(set_to_none=True)
    torch.cuda.reset_peak_memory_stats()
    loss = _g_step(m, D, x8, style8, 0.5, deg, ind)
    torch.cuda.synchronize()
    print(f"\nG step at batch 8 (256^2 + 224^2 calls): loss {loss.item():.5f}, peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    assert torch.isfinite(loss)
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for n, p in m.named_parameters() if trained(n))
    # batch 2 against the float64 restatement on the device (the discriminator as its float64 oracle)
    from tests import oracle_discriminator as OD
    from tests.oracle_vtoonify_gstep import O
    x2, s2 = x8[:2], style8[:2]
    m.zero_grad(set_to_none=True)
    _g_step(m, D, x2, s2, 0.5, deg[:2], ind[:2])
    got = {n: p.grad.clone() for n, p in m.named_parameters() if trained(n)}
    sd = {k: v.detach().double().requires_grad_(trained(k)) for k, v in m.state_dict().items()}
    dsd = {k: v.detach().double() for k, v in D.state_dict().items()}
    torch.set_default_dtype(torch.float64)
    try:
        with torch.enable_grad():
            xd = x2.double()
            img, masks = O.vtoonify_forward(sd, xd, s2.double(), 0.5, return_mask=True)
            img2, masks2 = O.vtoonify_forward(sd, xd[:, :, 16:240, 16:240].contiguous(), s2.double(), 0.5, return_mask=True)
            adv = F.softplus(-OD.forward(dsd, F.adaptive_avg_pool2d(img, 256), deg[:2].double(), ind[:2])).mean()
            loss_o = adv + loss_of(img2, masks2, image_target(img2.shape).to(img2)) + sum(w * k.mean() for w, k in zip((0.2, 0.4), masks))
            loss_o.backward()
    finally:
        torch.set_default_dtype(torch.float32)
    errs = {n: rel(got[n], sd[n].grad) for n in got if sd[n].grad.norm() > 0}
    worst = max(errs.values())
    print(f"batch 2 vs float64 ({ops.get_precision()}): worst rel L2 {worst:.2e} ({max(errs, key=errs.get)})")
    assert worst <= STEP_BAR


def test_level_b_restatement_gradients_match_the_oracle(models):
    """tools/gstep_bench.py's level (b) arm, the reference module's statements on vtoonify_b200.op, computes the G step's gradients."""
    from tests.oracle_vtoonify_gstep import library_ops, restated_forward
    from vtoonify_b200 import ops
    m = models["dualstylegan"]
    x, style = cuda_inputs()
    sd = {k: v.cuda() for k, v in m.state_dict().items()}
    ref = loss_and_grads(sd, x, style, 0.5, "dualstylegan", x_grad=False)
    sd32 = {k: v.detach().clone().requires_grad_(trained(k)) for k, v in sd.items()}
    old = ops.set_precision("bf16x3")
    try:
        with torch.enable_grad():
            img, masks = restated_forward(sd32, x, style, 0.5, "dualstylegan", ops=library_ops())
            loss_of(img, masks, image_target(img.shape).cuda()).backward()
    finally:
        ops.set_precision(old)
    errs = {k: rel(sd32[k].grad, ref["grads"][k]) for k in ref["grads"] if ref["grads"][k].norm() > 0}
    print(f"\nlevel (b) bf16x3: worst rel L2 {max(errs.values()):.2e} ({max(errs, key=errs.get)})")
    # its nn.Conv2d layers (encoder, fusion) run on cuDNN with TF32, PyTorch's default for convolutions: the TF32 bar
    assert max(errs.values()) <= BARS["tf32"]
