"""GPU: vtoonify_b200.lpips.PerceptualLoss (VGG16 net-lin) against the reference's own PNetLin (tests/golden/lpips_*.npz) and the
float64 restatement (tests/oracle_lpips.py) in fp32, bf16x3 and tf32: the loss per sample and the relative L2 of each input gradient.
Also: a row-strip-wide case, normalize=True, gradients to pred / target / both / neither, no records outside autograd, the frozen-
parameter and CPU-tensor errors, bit-identical reruns, a training-size batch against the fp32 cuDNN restatement, and a composed G step
(VToonify.forward, adaptive_avg_pool2d, this loss) into the encoder and fusion parameters against float64."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import oracle_lpips as O

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# Bars per precision, about 4x the worst values measured on an H100 (printed by the tests; DESIGN §9): relative error of the loss per
# sample, and relative L2 of an input gradient.
# Measured worst (fixtures, wide case, training size): loss 1.3e-7 / 1.9e-6 / 1.4e-4, gradient 6.0e-5 / 8.9e-3 / 6.2e-2.
LOSS_BARS = {"fp32": 5e-7, "bf16x3": 8e-6, "tf32": 6e-4}
GRAD_BARS = {"fp32": 2.5e-4, "bf16x3": 3e-2, "tf32": 0.25}
PRECS = ("fp32", "bf16x3", "tf32")


def make_loss(seed=0):
    from vtoonify_b200.lpips import PNetLin, PerceptualLoss
    from vtoonify_b200.weights import det_state_dict
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "vgg.pth")
        torch.save({k: v for k, v in det_state_dict(PNetLin(pnet_rand=True), seed=seed).items() if k.startswith("lin")}, path)
        p = PerceptualLoss(model="net-lin", net="vgg", use_gpu=True, gpu_ids=[0], model_path=path, pnet_rand=True)
    p.model.net.load_state_dict(det_state_dict(p.model.net, seed=seed), strict=True)
    p.model.net.requires_grad_(False)
    return p


@pytest.fixture(scope="module")
def percept():
    return make_loss()


def oracle_sd(p):
    return {k: v.detach().double().cpu() for k, v in p.model.net.state_dict().items()}


def rel(got, ref):
    return ((got.double().cpu() - ref.double().cpu()).norm() / ref.double().cpu().norm()).item()


def lib_run(p, pred, target, want_pred, want_target, weights, prec, normalize=False):
    from vtoonify_b200 import ops
    old = ops.set_precision(prec)
    try:
        pr = pred.detach().float().cuda().requires_grad_(want_pred)
        tg = target.detach().float().cuda().requires_grad_(want_target)
        with torch.enable_grad():
            loss = p(pr, tg, normalize=normalize)
            if want_pred or want_target:
                (loss.flatten() * weights.float().cuda()).sum().backward()
        torch.cuda.synchronize()
    finally:
        ops.set_precision(old)
    return loss.detach(), pr.grad, tg.grad


def oracle_run(sd, pred, target, want_pred, want_target, weights, normalize=False):
    pr = pred.detach().double().cpu().clone().requires_grad_(want_pred)
    tg = target.detach().double().cpu().clone().requires_grad_(want_target)
    with torch.enable_grad():
        loss = O.perceptual_loss(sd, pr, tg, normalize=normalize)
        if want_pred or want_target:
            (loss.flatten() * weights.double()).sum().backward()
    return loss.detach(), pr.grad, tg.grad


def check(name, prec, loss, gp, gt, ref_loss, ref_gp, ref_gt):
    el = ((loss.double().cpu().flatten() - ref_loss.double().flatten()).abs() / ref_loss.double().flatten().abs()).max().item()
    eg = {n: rel(a, b) for n, a, b in (("pred.grad", gp, ref_gp), ("target.grad", gt, ref_gt)) if b is not None}
    print(f"\n{name} {prec}: loss rel {el:.2e}; " + ", ".join(f"{n} rel L2 {e:.2e}" for n, e in eg.items()))
    assert loss.shape == ref_loss.shape
    assert el <= LOSS_BARS[prec], f"{name} {prec}: loss rel err {el:.2e}"
    for n, e in eg.items():
        assert e <= GRAD_BARS[prec], f"{name} {prec}: {n} rel L2 {e:.2e}"
    assert (gp is None) == (ref_gp is None) and (gt is None) == (ref_gt is None)


@pytest.mark.parametrize("case", sorted(O.CASES))
@pytest.mark.parametrize("prec", PRECS)
def test_against_reference_fixtures(percept, case, prec):
    shape, seed, g_pred, g_target = O.CASES[case]
    z = np.load(os.path.join(GOLDEN, f"lpips_{case}.npz"))
    pred, target = torch.from_numpy(z["pred"]), torch.from_numpy(z["target"])
    loss, gp, gt = lib_run(percept, pred, target, g_pred, g_target, O.loss_weights(shape[0], seed), prec)
    check(f"golden {case}", prec, loss, gp, gt, torch.from_numpy(z["loss"]),
          torch.from_numpy(z["pred_grad"]) if g_pred else None, torch.from_numpy(z["target_grad"]) if g_target else None)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("want", [(True, False), (False, True), (True, True)])
def test_against_oracle_wide_and_normalized(percept, prec, want):
    """[1, 3, 24, 264]: wide enough for conv1_2's forward to take the row-strip route in bf16x3; inputs in [0, 1] with normalize."""
    pred, target = O.inputs((1, 3, 24, 264), 9)
    pred, target = (pred + 1) / 2, (target + 1) / 2
    wts = O.loss_weights(1, 9)
    sd = oracle_sd(percept)
    ref = oracle_run(sd, pred, target, *want, wts, normalize=True)
    got = lib_run(percept, pred, target, *want, wts, prec, normalize=True)
    check(f"wide normalize want={want}", prec, *got, *ref)


def test_no_gradient_wanted_keeps_nothing(percept):
    pred, target = O.inputs((2, 3, 32, 32), 4)
    pred, target = pred.float().cuda(), target.float().cuda()
    ref = percept(pred, target)
    torch.cuda.synchronize()
    for mode in ("no_grad", "grad_no_inputs"):
        m0 = torch.cuda.memory_allocated()
        if mode == "no_grad":
            with torch.no_grad():
                out = percept(pred.clone().requires_grad_(), target)
        else:
            with torch.enable_grad():
                out = percept(pred, target)
        torch.cuda.synchronize()
        assert out.grad_fn is None and not out.requires_grad
        assert torch.equal(out, ref)
        assert torch.cuda.memory_allocated() - m0 <= 512, mode
        del out


def test_records_are_released_after_backward(percept):
    pred, target = O.inputs((2, 3, 32, 32), 4)
    pred, target = pred.float().cuda().requires_grad_(), target.float().cuda()
    with torch.enable_grad():
        percept(pred, target).sum().backward()            # builds the cached transposed weights
    pred.grad = None
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    with torch.enable_grad():
        loss = percept(pred, target)
        assert torch.cuda.memory_allocated() > m0 + 4 * 2 * 32 * 32 * 64 * 4
        loss.sum().backward()
    del loss
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() - m0 <= pred.numel() * 4 + 512


def test_reruns_are_bit_identical(percept):
    pred, target = O.inputs((2, 3, 40, 48), 6)
    wts = O.loss_weights(2, 6)
    a = lib_run(percept, pred, target, True, True, wts, "bf16x3")
    b = lib_run(percept, pred, target, True, True, wts, "bf16x3")
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_trainable_parameter_raises(percept):
    pred, target = O.inputs((1, 3, 16, 16), 7)
    w = percept.model.net.lin2.model[1].weight
    w.requires_grad_(True)
    try:
        with torch.enable_grad(), pytest.raises(NotImplementedError, match="lin2.model.1.weight"):
            percept(pred.float().cuda().requires_grad_(), target.float().cuda())
    finally:
        w.requires_grad_(False)
    c = getattr(percept.model.net.net.slice3, "12").weight
    c.requires_grad_(True)
    try:
        with torch.enable_grad(), pytest.raises(NotImplementedError, match="net.slice3.12.weight"):
            percept(pred.float().cuda(), target.float().cuda())
    finally:
        c.requires_grad_(False)


def test_cpu_tensors_raise(percept):
    from vtoonify_b200._lib import VtError
    pred, target = O.inputs((1, 3, 16, 16), 7)
    with pytest.raises(VtError):
        percept(pred.float(), target.float())
    with torch.enable_grad(), pytest.raises(VtError):
        percept(pred.float().requires_grad_(), target.float())


def test_training_size_against_cudnn_fp32(percept):
    """batch 8 at 512², gradient to pred (the training scripts' call), against the restatement on cuDNN in fp32 (TF32 off)."""
    pred, target = O.inputs((8, 3, 512, 512), 12)
    wts = O.loss_weights(8, 12)
    sd = {k: v.float().cuda() for k, v in percept.model.net.state_dict().items()}
    torch.backends.cudnn.allow_tf32 = False
    try:
        ref = oracle_run_device(sd, pred, target, wts)
    finally:
        torch.backends.cudnn.allow_tf32 = True
    got = lib_run(percept, pred, target, True, False, wts, "bf16x3")
    el = ((got[0].double() - ref[0].double()).abs() / ref[0].double().abs()).max().item()
    eg = rel(got[1], ref[1])
    print(f"\ntraining size bf16x3 vs cuDNN fp32: loss rel {el:.2e}, pred.grad rel L2 {eg:.2e}")
    assert el <= LOSS_BARS["bf16x3"] and eg <= GRAD_BARS["bf16x3"]


def oracle_run_device(sd, pred, target, wts):
    pr = pred.float().cuda().requires_grad_()
    with torch.enable_grad():
        loss = O.perceptual_loss(sd, pr, target.float().cuda())
        (loss.flatten() * wts.float().cuda()).sum().backward()
    return loss.detach(), pr.grad


@pytest.mark.parametrize("prec", PRECS)
def test_composed_g_step_against_float64(percept, prec):
    """VToonify-D forward (x [2, 22, 32, 32] -> image 128²), adaptive_avg_pool2d to 64², this loss, back into the encoder and fusion
    parameters and x, against oracle.vt_oracle's VToonify plus the LPIPS restatement in float64."""
    from tests.oracle_vtoonify_gstep import O as VO, inputs, trained
    from tests.test_gpu_vtoonify_grad import make_model
    from vtoonify_b200 import ops
    m = make_model("dualstylegan")
    x, style = inputs("sq")
    real = torch.rand((2, 3, 128, 128), generator=torch.Generator().manual_seed(31), dtype=torch.float64) * 2 - 1
    # float64 oracle
    sd = {k: v.detach().double().cpu().requires_grad_(trained(k)) for k, v in m.state_dict().items()}
    x64 = x.double().requires_grad_()
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        with torch.enable_grad():
            img, _ = VO.vtoonify_forward(sd, x64, style.double(), 0.5, "dualstylegan", return_mask=True)
            ref_loss = O.perceptual_loss(oracle_sd(percept), F.adaptive_avg_pool2d(img, 64), F.adaptive_avg_pool2d(real, 64)).sum()
            ref_loss.backward()
    finally:
        torch.set_default_dtype(old)
    # library
    old = ops.set_precision(prec)
    try:
        xg = x.cuda().requires_grad_()
        with torch.enable_grad():
            img, _ = m(xg, style.cuda(), d_s=0.5, return_mask=True)
            loss = percept(F.adaptive_avg_pool2d(img, 64), F.adaptive_avg_pool2d(real.float().cuda(), 64)).sum()
            loss.backward()
    finally:
        ops.set_precision(old)
    rows = [("x.grad", xg.grad, x64.grad)] + [(n, p.grad, sd[n].grad) for n, p in m.named_parameters()
                                               if trained(n) and sd[n].grad is not None and sd[n].grad.norm() > 0]
    errs = {n: rel(a, b) for n, a, b in rows}
    el = abs(loss.item() - ref_loss.item()) / abs(ref_loss.item())
    worst = max(errs.values())
    print(f"\ncomposed G step {prec}: loss rel {el:.2e}; worst grad rel L2 {worst:.2e} ({max(errs, key=errs.get)})")
    assert el <= COMPOSED_LOSS_BARS[prec] and worst <= COMPOSED_BARS[prec]


# The composed step also carries VToonify's own gradient error (tests/test_gpu_vtoonify_grad.py).  Measured worst: loss 2.5e-7 /
# 1.0e-5 / 9.6e-5, gradient 9.6e-4 / 1.2e-2 / 0.105.
COMPOSED_LOSS_BARS = {"fp32": 1e-6, "bf16x3": 4e-5, "tf32": 4e-4}
COMPOSED_BARS = {"fp32": 4e-3, "bf16x3": 5e-2, "tf32": 0.4}
