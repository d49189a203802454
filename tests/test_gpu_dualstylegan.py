"""GPU: DualStyleGAN.forward against the reference outputs in tests/golden/dualstylegan64.npz, against Generator.forward where
the extrinsic path is off or has all weights 0 (bit for bit), at the VToonify-D teacher's batch-8 / 1024 shapes, and its
per-style caching."""
import pytest
import torch

from tests.oracle_dualstylegan import CASES, W_FIX_COLOR, W_RES, case_inputs, case_outputs, dualstylegan_forward, state_dict
from tests.test_gpu_layers import check

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture(params=["fp32", "bf16x3", "tf32"])
def prec(request):
    from vtoonify_b200 import ops
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(ops.DEFAULT_PRECISION)


@pytest.fixture(scope="module")
def model64():
    from vtoonify_b200.dualstylegan import DualStyleGAN
    m = DualStyleGAN(64, 512, 8)
    m.load_state_dict(state_dict(), strict=True)
    return m.cuda()


def codes(seed, B=2, L=10):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((B, L, 512), generator=g).cuda(), torch.randn((B, L, 512), generator=g).cuda()


@pytest.mark.parametrize("name", list(CASES))
def test_golden_cases(golden, model64, prec, name):
    g = golden("dualstylegan64")
    kw, inputs = CASES[name]
    styles, ex = case_inputs(g, inputs)
    y = model64([s.cuda() for s in styles], ex.cuda(), randomize_noise=False, **kw)
    y = (y[0][:, ::32], y[1]) if name == "feat" else (y[0],)
    for part, got, ref in zip(("", " skip"), y, case_outputs(g, name)):
        check(got, ref, prec, f"DualStyleGAN(64) {name}{part}")


def test_equals_generator_without_extrinsic_path(model64, prec):
    """use_res=False, and use_res=True with every weight 0 (ModRes blocks are the identity, blends the intrinsic code), run the
    generator's own launches: bit-identical to Generator.forward"""
    latent, ex = codes(3)
    ref, _ = model64.generator([latent], input_is_latent=True, randomize_noise=False)
    y, lat = model64([latent], ex, input_is_latent=True, randomize_noise=False, use_res=False, return_latents=True)
    assert torch.equal(y, ref)
    assert lat is latent
    y0, none = model64([latent], ex, input_is_latent=True, randomize_noise=False, interp_weights=[0] * 18)
    assert torch.equal(y0, ref) and none is None


def test_style_cache(model64):
    """the same tensors give the same result; an in-place change to exstyles or other interp_weights is picked up; a fresh
    code on every call (the training teacher) is right every time"""
    sd = state_dict()
    noises = [sd[f"generator.noises.noise_{i}"] for i in range(9)]
    kw = dict(input_is_latent=True, interp_weights=W_RES)        # + the stored noise buffers

    def run(latent, ex, **over):
        return model64([latent], ex, randomize_noise=False, **dict(kw, **over))[0]

    def uncached(latent, ex, **over):         # new tensor objects: nothing cached for them yet
        return run(latent.clone(), ex.clone(), **over)
    latent, ex = codes(4)
    y1 = run(latent, ex)
    assert torch.equal(run(latent, ex), y1)
    assert torch.equal(uncached(latent, ex), y1)
    ex.mul_(0.5)
    y2 = run(latent, ex)
    assert torch.equal(y2, uncached(latent, ex)) and not torch.equal(y2, y1)
    y3 = run(latent, ex, interp_weights=W_FIX_COLOR)
    assert torch.equal(y3, uncached(latent, ex, interp_weights=W_FIX_COLOR)) and not torch.equal(y3, y2)
    for seed in (5, 6, 7):
        latent, ex = codes(seed)
        y = run(latent, ex)
        check(y, dualstylegan_forward(sd, [latent.cpu()], ex.cpu(), noises, **kw), "bf16x3", f"fresh code {seed}")


def test_random_noise(model64):
    latent, ex = codes(8)
    y, _ = model64([latent], ex, input_is_latent=True, interp_weights=W_RES)
    assert tuple(y.shape) == (2, 3, 64, 64) and torch.isfinite(y).all()


def test_teacher_pretraining_call_1024_b8():
    """The pretraining teacher call of VToonify-D (train_vtoonify_d.py:132) at batch 8: 512-channel maps of 4², 8², 16² and
    32² with per-sample AdaIN and output statistics, on the automatic plans and with the ping-pong kernel forced onto launches of
    fewer items, with and without the 256-wide work items; against the fp32 mode and, for one sample, the CPU oracle.

    The bf16x3 mode is held to the whole-model bar of test_gpu_fullsize.py (1e-3 of max(1, rms)), not the per-layer TOL: after
    seven 512-channel layers the split-operand rounding alone reaches 5.6e-4 of the rms as the largest of 4M differences (measured on
    an H100 with every weight 0, i.e. on Generator's own launches; fused or separate statistics passes give the same)."""
    from vtoonify_b200 import _lib, ops
    from vtoonify_b200.dualstylegan import DualStyleGAN
    from vtoonify_b200.weights import det_state_dict
    m = DualStyleGAN(1024, 512, 8)
    sd = det_state_dict(m, seed=5)
    m.load_state_dict(sd, strict=True)
    m.cuda()
    ws, style = codes(9, B=8, L=18)
    kw = dict(input_is_latent=True, return_feat=True, truncation=0.5, truncation_latent=0, interp_weights=[0.75] * 7 + [1] * 11)
    ops.set_precision("fp32")
    try:
        ref_feat, ref_skip = (t.cpu() for t in m([ws], style, randomize_noise=False, **kw))
    finally:
        ops.set_precision(ops.DEFAULT_PRECISION)
    noises = [sd[f"generator.noises.noise_{i}"] for i in range(m.num_layers)]
    o_feat, o_skip = dualstylegan_forward(sd, [ws[:1].cpu()], style[:1].cpu(), noises, **kw)
    check(ref_feat[:1], o_feat, "fp32", "1024 feat [fp32 mode] vs oracle")
    check(ref_skip[:1], o_skip, "fp32", "1024 skip [fp32 mode] vs oracle")
    lib = _lib.load()
    for pp in (1, 2):
        for wide in (0, 1):
            old = lib.vt_set_option(b"tc_pingpong", pp), lib.vt_set_option(b"tc_wide", wide)
            try:
                feat, skip = m([ws], style, randomize_noise=False, **kw)
            finally:
                lib.vt_set_option(b"tc_pingpong", old[0]), lib.vt_set_option(b"tc_wide", old[1])
            assert tuple(feat.shape) == (8, 512, 32, 32) and tuple(skip.shape) == (8, 3, 32, 32)
            for name, y, ref in (("feat", feat, ref_feat), ("skip", skip, ref_skip)):
                err = (y.cpu() - ref).abs().max().item()
                rms = ref.pow(2).mean().sqrt().item()
                print(f"1024 {name} b8 (tc_pingpong {pp}, tc_wide {wide}) [bf16x3]: max err {err:.3e}  ref rms {rms:.3f}")
                assert err <= 1e-3 * max(1.0, rms), f"1024 {name} b8 (tc_pingpong {pp}, tc_wide {wide}): err {err:.3e}"


@pytest.mark.parametrize("hw", [4, 8])
def test_small_map_statistics_b8(hw):
    """The 512-channel ModRes convolution on a 4x4 / 8x8 map (smaller than one pixel tile) at batch 8: per-sample AdaIN applied
    inside the convolution and the output statistics from its epilogue, on every ping-pong / wide-item mode, against F.conv2d
    and a separate statistics pass over the output"""
    import torch.nn.functional as F
    from vtoonify_b200 import _lib, ops
    from vtoonify_b200._lib import ACT_LRELU
    B, C = 8, 512
    g = torch.Generator().manual_seed(hw)
    x = torch.randn((B, C, hw, hw), generator=g) + 0.3
    aff = torch.randn((B, C, 2), generator=g) * 0.5
    w = torch.randn((C, C, 3, 3), generator=g) / (3 * C ** 0.5)
    b = torch.randn(C, generator=g) * 0.1
    ref = F.leaky_relu(F.conv2d(x * aff[:, :, 0, None, None] + aff[:, :, 1, None, None], w, b, padding=1), 0.2) * 2 ** 0.5
    xn, wp, affc, bc = ops.to_nhwc(x.cuda(), round_tf32=False), ops.prep_weights(w.cuda(), cin_pad=C), aff.cuda(), b.cuda()
    lib = _lib.load()
    for pp in (0, 1, 2):
        for wide in (0, 1):
            old = lib.vt_set_option(b"tc_pingpong", pp), lib.vt_set_option(b"tc_wide", wide)
            try:
                y, st = ops.conv2d_nhwc([xn], wp, ops.conv_taps(3, 1), 1, hw, hw, bias=bc, act=ACT_LRELU, gain=2 ** 0.5,
                                        src_affine=[affc], want_stats=True)
            finally:
                lib.vt_set_option(b"tc_pingpong", old[0]), lib.vt_set_option(b"tc_wide", old[1])
            what = f"{hw}x{hw} (tc_pingpong {pp}, tc_wide {wide})"
            err = (ops.to_nchw(y).cpu() - ref).abs().max().item()
            assert err <= 3e-5 * max(1.0, ref.abs().max().item()), f"{what}: output err {err:.3e}"
            st_ref = ops.instnorm_stats(y)
            st_err = (st - st_ref).abs().max().item()
            assert st_err <= 1e-4 * max(1.0, st_ref.abs().max().item()), f"{what}: statistics err {st_err:.3e}"
