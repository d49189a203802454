"""RAFT drop-in on the GPU: the whole forward in fp32, bf16x3 and tf32 against the float64 restatement (tests/oracle_raft.py), reruns,
flow_init, the non-test prediction list and one run at the smoothing size.

Bars are about 4x the worst relative L2 measured on an H100 (DESIGN.md section 11).  RAFT iterates: a rounding difference that moves a
bilinear tap across a pixel boundary of the correlation pyramid changes that tap's neighbours, and the GRU carries it on, so the error
grows with the iterations; the 20-iteration case has the widest bar for that reason, not a looser arithmetic."""
import numpy as np
import pytest
import torch

from tests import oracle_raft as O
from tests.golden.make_golden_raft import CASES, case_inputs, images, raft_args
from vtoonify_b200 import ops, set_precision
from vtoonify_b200._lib import launch_count
from vtoonify_b200.raft import RAFT
from vtoonify_b200.weights import det_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
BARS = {"fp32": 3e-5, "bf16x3": 5e-4, "tf32": 3e-2}      # measured worst: 7.7e-6, 1.24e-4, 7.4e-3 (the it20 case)


@pytest.fixture(scope="module")
def model_sd():
    m = RAFT(raft_args()).eval()
    sd = det_state_dict(m, seed=0)
    m.load_state_dict(sd, strict=True)
    m.requires_grad_(False)
    return m.to(DEV), {k: v.to(DEV) for k, v in sd.items()}


@pytest.fixture(autouse=True)
def _restore_precision():
    yield
    set_precision(ops.DEFAULT_PRECISION)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _oracle64(sd, c):
    i1, i2, fi = case_inputs(c)
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    with torch.no_grad():
        return O.raft_forward(sd64, i1.to(DEV).double(), i2.to(DEV).double(), c["iters"], None if fi is None else fi.to(DEV).double(),
                              c["test_mode"], every_mask=False)


def _run(m, c):
    i1, i2, fi = case_inputs(c)
    with torch.no_grad():
        return m(i1.to(DEV), i2.to(DEV), iters=c["iters"], flow_init=None if fi is None else fi.to(DEV), test_mode=c["test_mode"])


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "tf32"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_forward_against_float64(model_sd, name, prec):
    m, sd = model_sd
    c = CASES[name]
    set_precision(prec)
    out = _run(m, c)
    ref = _oracle64(sd, c)
    if c["test_mode"]:
        err = max(_rel(out[0], ref[0]), _rel(out[1], ref[1]))
    else:
        assert isinstance(out, list) and len(out) == c["iters"]
        err = max(_rel(o, r) for o, r in zip(out, ref))
    print(f"RAFT {name} {prec}: worst relative L2 {err:.3e}")
    assert err <= BARS[prec], err


def test_rerun_bit_identical(model_sd):
    m, _ = model_sd
    c = CASES["b2"]
    set_precision("bf16x3")
    a, b = _run(m, c), _run(m, c)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_non_test_list_and_flow_init(model_sd):
    """the list's last entry is the test-mode flow_up; flow_init shifts the starting coordinates (zero flow_init == none)"""
    m, _ = model_sd
    set_precision("bf16x3")
    i1, i2 = images(1, 128, 144, 9)
    i1, i2 = i1.to(DEV), i2.to(DEV)
    with torch.no_grad():
        lst = m(i1, i2, iters=4)
        low, up = m(i1, i2, iters=4, test_mode=True)
        low0, up0 = m(i1, i2, iters=4, test_mode=True, flow_init=torch.zeros(1, 2, 16, 18, device=DEV))
        low1, _ = m(i1, i2, iters=1, test_mode=True, flow_init=torch.full((1, 2, 16, 18), 3.0, device=DEV))
    assert len(lst) == 4 and torch.equal(lst[-1], up) and lst[-1].shape == (1, 2, 128, 144)
    assert torch.equal(up0, up) and torch.equal(low0, low)
    assert float((low1 - 3.0).abs().mean()) < float(low1.abs().mean())


def test_launch_count_test_mode(model_sd):
    """test mode runs the mask head and the up-sampling once; each further iteration costs the same launches"""
    m, _ = model_sd
    set_precision("bf16x3")
    i1, i2 = images(1, 128, 128, 4)
    i1, i2 = i1.to(DEV), i2.to(DEV)
    counts = []
    for it in (2, 3):
        with torch.no_grad():
            n0 = launch_count()
            m(i1, i2, iters=it, test_mode=True)
            counts.append(launch_count() - n0)
    with torch.no_grad():
        n0 = launch_count()
        m(i1, i2, iters=3)
        full = launch_count() - n0
    print(f"RAFT launches: iters=2 {counts[0]}, iters=3 {counts[1]}, iters=3 non-test {full}")
    assert counts[1] - counts[0] == 18          # one iteration: lookup, 5 motion convs + flow store, 2 x 4 GRU, 2 flow head, update
    assert full - counts[1] == 2 * 3            # a mask head (2 convolutions) and an up-sampling for each earlier iteration


def test_smoothing_size_against_device_restatement(model_sd):
    """11 pairs at 800x800, 20 iterations, bf16x3, against the restatement in fp32 on cuDNN with TF32 off"""
    m, sd = model_sd
    set_precision("bf16x3")
    a, b = images(1, 800, 800, 11)
    i1 = a.repeat(11, 1, 1, 1).to(DEV)
    i2 = torch.cat([images(1, 800, 800, 20 + k)[1] for k in range(5)] + [b] + [images(1, 800, 800, 30 + k)[1] for k in range(5)]).to(DEV)
    with torch.no_grad():
        low, up = m(i1, i2, iters=20, test_mode=True)
        torch.cuda.synchronize()
        tf = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        try:
            rl, ru = O.raft_forward(sd, i1, i2, 20, None, True, every_mask=False)
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf
    assert up.shape == (11, 2, 800, 800) and torch.isfinite(up).all()
    err = max(_rel(low, rl), _rel(up, ru))
    print(f"RAFT 11x800x800 it20 bf16x3 vs fp32 restatement: relative L2 {err:.3e}, mean |flow_up| {float(ru.abs().mean()):.2f}")
    assert err <= 1e-4, err                      # measured 2.4e-5 (4x rounded up)
