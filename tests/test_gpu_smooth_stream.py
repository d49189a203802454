"""Streaming parsing-map smoothing on the GPU: ParsingSmoother against a whole-clip restatement of the loop, the frame prep against torch
and the BiSeNet input, the fuse-and-downsample kernel against fuse + Downsample + 1/16 and float64, and FramePipeline(smoothing=...)
against the two-step library route (smooth_parsing_maps, then (frames, parse) batches)."""
import pytest
import torch
import torch.nn.functional as F

from tests.golden.make_golden_raft import images, raft_args
from tests.golden.make_golden_smooth import parsing_maps, parsing_seed
from vtoonify_b200 import ops, set_precision
from vtoonify_b200 import smooth_parsing as S
from vtoonify_b200.raft import RAFT
from vtoonify_b200.stylegan import make_kernel
from vtoonify_b200.weights import det_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def raft():
    torch.manual_seed(0)
    m = RAFT(raft_args()).eval()
    m.load_state_dict(det_state_dict(m, seed=0), strict=True)
    m.requires_grad_(False)
    return m.to(DEV)


@pytest.fixture(autouse=True)
def _restore_precision():
    yield
    set_precision(ops.DEFAULT_PRECISION)


def _clip(N, H, W, C=5, seed=0):
    Is = torch.cat([images(1, H, W, 70 + seed + k)[k % 2] for k in range(N)]) / 127.5 - 1.0
    Ps = parsing_maps(parsing_seed(N, 3 + seed)[:, :C], H, W)
    return Is.to(DEV), Ps.to(DEV)


def _whole_clip(Is, Ps, m, window, iters):
    """the smoothing loop with the whole clip at hand: per output, every slot's frame encoded from scratch"""
    N, C, H, W = Ps.shape
    R, wt = 2 * window + 1, S.temporal_weights(window).tolist()
    kernel = make_kernel([1, 3, 3, 1]).to(DEV)
    rin = torch.add(Is, 1).mul_(255.0).div_(2)
    out = torch.empty((N, C, H // 2, W // 2), device=DEV)
    for i, fr in enumerate(S.slot_frames(N, window)):
        flows = [None] * R
        if window:
            c = fr[window]
            nb = [fr[k] for k in range(R) if k != window]
            f1 = m._features(m._input_s2d(rin[c:c + 1])).expand(len(nb), -1, -1, -1).contiguous()
            f2 = torch.cat([m._features(m._input_s2d(rin[f:f + 1])) for f in nb])
            net, x = m._context(m._input_s2d(rin[c:c + 1]))
            _, up = m._iterate(f1, f2, net.expand(len(nb), -1, -1, -1).contiguous(), x.expand(len(nb), -1, -1, -1).contiguous(), iters)
            flows = [up[k if k < window else k - 1] if k != window else None for k in range(R)]
        fused = S.parsing_fuse([Is[f] for f in fr], [Ps[f] for f in fr], flows, wt)
        out[i] = ops.upfirdn2d_planar(fused[None], kernel, (1, 1), (2, 2), (1, 1, 1, 1))[0]
    return out


@pytest.mark.parametrize("window", [0, 1, 2, 5])
def test_streaming_equals_whole_clip(raft, window):
    set_precision("bf16x3")
    H = W = 128
    for N in sorted({max(window, 1), window + 1, 2 * window + 1, 3 * window + 3}):
        Is, Ps = _clip(N, H, W, seed=N)
        with torch.no_grad():
            ref = _whole_clip(Is, Ps, raft, window, 3)
            lib = S.smooth_parsing_maps(Is, Ps, raft, window=window, iters=3)
            sm = S.ParsingSmoother(raft, window, 3)
            got, fused = {}, {}
            for f in range(N):
                outs = sm.push(Is[f], Ps[f])
                assert [r.index for r in outs] == S.release_schedule(N, window)[0][f]
                for r in outs:
                    got[r.index] = r.down()
                    fused[r.index] = r.fuse_down(torch.empty((Ps.shape[1], H // 2, W // 2), device=DEV), 1.0)
            for r in sm.finish():
                got[r.index] = r.down()
                fused[r.index] = r.fuse_down(torch.empty((Ps.shape[1], H // 2, W // 2), device=DEV), 1.0)
        assert sorted(got) == list(range(N))
        stream = torch.stack([got[i] for i in range(N)])
        assert torch.equal(stream, ref), (window, N, float((stream - ref).abs().max()))
        assert torch.equal(lib, ref), (window, N)
        assert torch.equal(torch.stack([fused[i] for i in range(N)]), ref), (window, N)


def _ulps(a, b):
    ia, ib = a.contiguous().view(torch.int32).long(), b.contiguous().view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return (ia - ib).abs()


@pytest.mark.parametrize("B,H,W,kind", [(2, 64, 64, "random"), (1, 7, 9, "random"), (3, 33, 17, "edges"), (1, 16, 24, "zero"),
                                        (1, 16, 24, "full")])
def test_frame_prep(raft, B, H, W, kind):
    g = torch.Generator().manual_seed(H * 100 + W)
    if kind == "random":
        fr = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    elif kind == "edges":
        fr = (torch.randint(0, 2, (B, H, W, 3), generator=g) * 255).to(torch.uint8)
    else:
        fr = torch.full((B, H, W, 3), 0 if kind == "zero" else 255, dtype=torch.uint8)
    Is, stem = S.frame_prep(fr.to(DEV))
    assert Is.shape == (B, 3, 2 * H, 2 * W) and stem.shape == (B, H, W, 32)
    # the script: F.interpolate(transform(frame)) on the CPU, transform = ToTensor + Normalize(0.5, 0.5)
    t = (fr.permute(0, 3, 1, 2).float().div(255) - 0.5) / 0.5
    ref = F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)
    u = _ulps(Is.cpu(), ref)
    err = (Is.cpu().double() - ref.double()).abs()
    print(f"frame prep {kind} {B}x{H}x{W}: Is against torch's CPU bilinear: {int((u > 0).sum())} of {u.numel()} values differ, "
          f"{int((u > 1).sum())} by more than 1 ulp, max |err| {float(err.max()):.2e}")
    # the sum's fmas are frame_s2d's, not ATen's CPU roundings: a difference is a few roundings of terms of magnitude <= 1, which near
    # a cancellation to ~0 is many ulp of the result
    assert float(err.max()) <= 2.0 ** -22
    # RAFT's stem input: _input_s2d of the script's (Is + 1) * 255.0 / 2 (three roundings)
    rin = torch.add(Is, 1).mul_(255.0).div_(2)
    assert torch.equal(stem, raft._input_s2d(rin))
    # BiSeNet sees exactly 2 * Is
    a = ops.frame_s2d(ops.frames_u8_to_f32(fr.to(DEV)), upsample2=True)
    b = ops.frame_s2d(2 * Is, upsample2=False)
    assert torch.equal(a, b)


def _fuse_case(nslot_window, H, W, C, seed, dup=False):
    g = torch.Generator().manual_seed(seed)
    R = 2 * nslot_window + 1
    imgs = [(torch.rand((3, H, W), generator=g) * 2 - 1).to(DEV) for _ in range(R)]
    pars = [(torch.randn((C, H, W), generator=g) * 3).to(DEV) for _ in range(R)]
    flows = [((torch.rand((2, H, W), generator=g) - 0.5) * 10).to(DEV) for _ in range(R)]
    if dup and R > 1:                  # a boundary centre: one frame fills two slots (the same tensors, flows of their own)
        imgs[0], pars[0] = imgs[1], pars[1]
    flows[nslot_window] = None
    return imgs, pars, flows


@pytest.mark.parametrize("window,H,W,dup", [(0, 64, 64, False), (2, 48, 80, False), (2, 66, 38, True), (5, 40, 72, True),
                                            (5, 37, 51, False), (31, 24, 40, True)])
@pytest.mark.parametrize("prec", ["bf16x3", "tf32"])
def test_fuse_down_bit_identical(window, H, W, dup, prec):
    set_precision(prec)
    C, B = 19, 3
    wt = S.temporal_weights(window).tolist()
    kernel = make_kernel([1, 3, 3, 1]).to(DEV)
    centres = [_fuse_case(window, H, W, C, 10 * window + b, dup) for b in range(B)]
    Ho, Wo = H // 2, W // 2
    x = torch.full((B, 22, Ho, Wo), float("nan"), device=DEV)
    S.parsing_fuse_down(centres, wt, x[:, 3:], 1.0 / 16.0)
    assert torch.isnan(x[:, :3]).all()
    for b, (imgs, pars, flows) in enumerate(centres):
        fused = S.parsing_fuse(imgs, pars, flows, wt)
        down = ops.upfirdn2d_planar(fused[None], kernel, (1, 1), (2, 2), (1, 1, 1, 1))[0]
        ref = ops.axpby(down, None, 1.0 / 16.0)
        assert torch.equal(x[b, 3:], ref), (b, float((x[b, 3:] - ref).abs().max()))
        # float64 bar of the 16-term down-sampling sum of the fp32 fused map
        f64 = F.pad(fused.double()[None], (1, 1, 1, 1))
        k64 = kernel.double()[None, None].expand(C, 1, 4, 4)
        ref64 = F.conv2d(f64, k64, stride=2, groups=C)[0] / 16.0
        terms = F.conv2d(f64.abs(), k64, stride=2, groups=C)[0] / 16.0
        bar = 17 * 2.0 ** -24 * terms + (2.0 ** -10 * ref64.abs() if prec == "tf32" else 0) + 1e-30
        err = (x[b, 3:].double() - ref64).abs()
        print(f"fuse_down window {window} {H}x{W} {prec} centre {b}: worst err/bar {float((err / bar).max()):.3f}")
        assert bool((err <= bar).all())


def _nets():
    from vtoonify_b200.bisenet import BiSeNet
    from vtoonify_b200.vtoonify import VToonify
    m = VToonify(backbone="dualstylegan").eval()
    m.load_state_dict(det_state_dict(m, seed=0), strict=True)
    p = BiSeNet(19).eval()
    p.load_state_dict(det_state_dict(p, seed=21), strict=True)
    return m.to(DEV), p.to(DEV)


@pytest.fixture(scope="module")
def nets():
    return _nets()


def _frames(N, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 256, (1, H, W, 3), generator=g).float()
    drift = torch.randint(-20, 21, (N, 1, 1, 3), generator=g).float()
    noise = torch.randint(-6, 7, (N, H, W, 3), generator=g).float()
    return (base + drift + noise).clamp(0, 255).to(torch.uint8)


def _batches(frames, B):
    return [frames[i:i + B].pin_memory() for i in range(0, frames.shape[0], B)]


def _two_step(m, p, raft, style, frames, B, window, iters, prefilter=None):
    """the two-step library route: whole-clip Is / Ps on the host, smooth_parsing_maps, then (frames, parse) batches"""
    from vtoonify_b200.frame_loop import FramePipeline
    with torch.no_grad():
        fr = frames.to(DEV)
        if prefilter is not None:
            fr = ops.frame_prefilter_resize(fr, prefilter[0], prefilter[1], prefilter[2])
        Is = torch.cat([S.frame_prep(fr[i:i + 1])[0] for i in range(fr.shape[0])]).cpu()
        Ps = torch.cat([p(2 * Is[i:i + 1].to(DEV))[0] for i in range(Is.shape[0])]).cpu()
        parse = S.smooth_parsing_maps(Is, Ps, raft, window=window, iters=iters)
        fr = fr.cpu()
    pipe = FramePipeline(m, style, d_s=0.5)
    return list(pipe.run([(fr[i:i + B].pin_memory(), parse[i:i + B].pin_memory()) for i in range(0, fr.shape[0], B)]))


@pytest.mark.parametrize("B,N,prefilter", [(1, 7, False), (3, 8, False), (4, 10, True), (3, 5, True)])
def test_pipeline_matches_two_step_route(nets, raft, B, N, prefilter):
    from vtoonify_b200.frame_loop import FramePipeline
    from vtoonify_b200.weights import det_inputs
    set_precision("bf16x3")
    m, p = nets
    window, iters, H, W = 2, 3, 64, 64
    style = det_inputs(1, 32, 32, seed=5)[1]
    pf = (1, (W, H), (0, H, 0, W)) if prefilter else None
    frames = _frames(N, 80 if prefilter else H, 72 if prefilter else W, seed=B * 10 + N)
    pipe = FramePipeline(m, style, d_s=0.5, parsing_net=p, smoothing=(raft, window, iters), prefilter=pf)
    outs = list(pipe.run(_batches(frames, B)))
    ref = _two_step(m, p, raft, style, frames, B, window, iters, pf)
    assert len(outs) == len(ref) == (N + B - 1) // B
    for k, (o, r) in enumerate(zip(outs, ref)):
        assert o.shape == r.shape and torch.equal(o, r), (B, N, k)


def test_pipeline_device_memory_flat(nets, raft):
    from vtoonify_b200.frame_loop import FramePipeline
    from vtoonify_b200.weights import det_inputs
    set_precision("bf16x3")
    m, p = nets
    window, iters, H, W, B = 2, 2, 64, 64, 2
    R = 2 * window + 1
    style = det_inputs(1, 32, 32, seed=5)[1]
    peaks = []
    for N in (2 * R, 4 * R, 2 * R):
        frames = _frames(N, H, W, seed=N)
        pipe = FramePipeline(m, style, d_s=0.5, parsing_net=p, smoothing=(raft, window, iters))
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        n = sum(1 for _ in pipe.run(_batches(frames, B)))
        assert n == (N + B - 1) // B
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
    print(f"smoothed pipeline peak device memory above the models: N={2 * R} {peaks[0] / 2 ** 20:.1f} MB, N={4 * R} "
          f"{peaks[1] / 2 ** 20:.1f} MB")
    assert peaks[1] <= 1.05 * min(peaks[0], peaks[2]) + 4 * 2 ** 20


def test_pipeline_misuse(nets, raft):
    from vtoonify_b200.frame_loop import FramePipeline
    from vtoonify_b200.weights import det_inputs
    m, p = nets
    style = det_inputs(1, 32, 32, seed=5)[1]
    sm = (raft, 2, 2)
    with pytest.raises(ValueError, match="parsing_net"):
        FramePipeline(m, style, smoothing=sm)
    with pytest.raises(ValueError, match="graph"):
        FramePipeline(m, style, parsing_net=p, smoothing=sm, graph=True)
    with pytest.raises(ValueError, match="window"):
        FramePipeline(m, style, parsing_net=p, smoothing=(raft, -1, 2))
    pipe = FramePipeline(m, style, parsing_net=p, smoothing=sm)
    with pytest.raises(ValueError, match="uint8"):
        list(pipe.run([torch.zeros((1, 22, 64, 64))]))
    with pytest.raises(ValueError, match="multiples of 8"):
        list(pipe.run([_frames(3, 60, 64)]))
    with pytest.raises(ValueError, match="multiples of 8"):
        list(pipe.run([_frames(3, 56, 64)]))
    with pytest.raises(ValueError, match="fewer than the window"):
        list(pipe.run([_frames(1, 64, 64)]))


def test_smoother_misuse_is_an_error(raft):
    """a handle read after a later push, a push after finish, and bad arguments (checked before the ring changes)"""
    set_precision("bf16x3")
    window, H = 1, 128
    Is, Ps = _clip(4, H, H, seed=2)
    with torch.no_grad():
        sm = S.ParsingSmoother(raft, window, 2)
        assert sm.push(Is[0], Ps[0]) == []
        (r1,) = sm.push(Is[1], Ps[1])
        (r2,) = sm.push(Is[2], Ps[2])
        with pytest.raises(RuntimeError, match="later push"):
            r1.down()
        r2.down()
        ring = sm._img.clone(), sm._par.clone()
        bad = [((Is[3].double(), Ps[3]), "fp32"), ((Is[3], Ps[3][:3]), "differs"), ((Is[3], Ps[3], torch.zeros((1, 64, 64, 32),
               device=DEV)[:, :, :, :16]), "stem"), ((Is[3], Ps[3], torch.zeros((1, 32, 64, 32), device=DEV)), "stem")]
        for args, msg in bad:
            with pytest.raises((ValueError, RuntimeError), match=msg):
                sm.push(*args)
        assert sm.n == 3 and torch.equal(sm._img, ring[0]) and torch.equal(sm._par, ring[1])
        r2.down()                                              # still valid: nothing was pushed
        sm.push(Is[3], Ps[3])
        outs = sm.finish()
        assert [r.index for r in outs] == [3]
        with pytest.raises(RuntimeError, match="finish"):
            sm.push(Is[3], Ps[3])
        torch.testing.assert_close(outs[0].down(), outs[0].down(), rtol=0, atol=0)
