"""Segmented parsing-map smoothing on the GPU: ParsingSmoother(first=...) over the segments of segment_plan against smooth_parsing_maps,
FramePipeline.smooth_segment over a plan against FramePipeline(smoothing=...).run, and ShardedSmoothedVideo over NCCL against the
one-GPU pass, with rank 0's device peak flat in the clip's length."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

from tests.golden.make_golden_raft import raft_args
from tests.test_gpu_smooth_stream import _batches, _clip, _frames, _nets
from tests.test_smooth_host import case
from vtoonify_b200 import ops, set_precision
from vtoonify_b200 import smooth_parsing as S
from vtoonify_b200.raft import RAFT
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


def _segmented(Is, Ps, m, window, iters, length):
    """smooth_parsing_maps segment by segment: each segment's frames pushed into a ParsingSmoother(first=seg.lo), its own outputs read"""
    N, C, H, W = Ps.shape
    out = torch.full((N, C, H // 2, W // 2), float("nan"), device=DEV)
    for seg in S.segment_plan(N, window, length):
        sm = S.ParsingSmoother(m, window, iters, first=seg.lo)
        for f in range(seg.lo, seg.hi):
            for r in sm.push(Is[f].to(DEV), Ps[f].to(DEV)):
                if seg.a <= r.index < seg.b:
                    out[r.index] = r.down()
        for r in (sm.finish() if seg.finish else []):
            if seg.a <= r.index < seg.b:
                out[r.index] = r.down()
    return out


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", ["w2", "w5"])
def test_segments_equal_smooth_parsing_maps_on_fixtures(raft, golden, name, prec):
    Is, Ps, window, _, _ = case(golden, name)
    set_precision(prec)
    with torch.no_grad():
        ref = S.smooth_parsing_maps(Is, Ps, raft, window=window, iters=20)
        for length in (1, 2, 4, Is.shape[0]):
            got = _segmented(Is, Ps, raft, window, 20, length)
            assert torch.equal(got.cpu(), ref), (name, prec, length, float((got.cpu() - ref).abs().nan_to_num(1e30).max()))


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
@pytest.mark.parametrize("window", [0, 1, 2, 5])
def test_segments_equal_smooth_parsing_maps_on_seeded_clips(raft, window, prec):
    set_precision(prec)
    N = 3 * window + 4
    Is, Ps = _clip(N, 128, 128, seed=window)
    with torch.no_grad():
        ref = S.smooth_parsing_maps(Is, Ps, raft, window=window, iters=3)
        for length in sorted({1, 3, max(window, 1) - 1 or 1, window + 2, N - 1}):
            got = _segmented(Is, Ps, raft, window, 3, length)
            assert torch.equal(got, ref), (window, prec, length)


@pytest.fixture(scope="module")
def nets():
    return _nets()


def _pipe(nets, raft, window, iters, prefilter=None):
    from vtoonify_b200.frame_loop import FramePipeline
    from vtoonify_b200.weights import det_inputs
    m, p = nets
    style = det_inputs(1, 32, 32, seed=5)[1]
    return FramePipeline(m, style, d_s=0.5, parsing_net=p, smoothing=(raft, window, iters), prefilter=prefilter)


# (B, N, window, length, prefilter): clips that are not multiples of length, a last segment shorter than the window, one segment
@pytest.mark.parametrize("B,N,window,length,prefilter", [(1, 7, 2, 3, False), (2, 11, 2, 4, True), (4, 10, 2, 8, False),
                                                          (2, 9, 5, 2, False), (4, 13, 1, 4, True), (1, 6, 5, 6, False),
                                                          (2, 6, 0, 4, False)])
def test_smooth_segment_equals_run(nets, raft, B, N, window, length, prefilter):
    set_precision("bf16x3")
    iters, H, W = 3, 64, 64
    pf = (1, (W, H), (0, H, 0, W)) if prefilter else None
    frames = _frames(N, 80 if prefilter else H, 72 if prefilter else W, seed=B * 10 + N)
    pipe = _pipe(nets, raft, window, iters, pf)
    ref = torch.cat(list(pipe.run(_batches(frames, B))))
    dev = frames.to(DEV)
    got = []
    for seg in S.segment_plan(N, window, length):
        out = pipe.smooth_segment(dev[seg.lo:seg.hi], seg, B)
        assert out.is_cuda and out.dtype == torch.uint8 and out.shape == (seg.b - seg.a, 4 * H, 4 * W, 3)
        got.append(out.cpu())
    got = torch.cat(got)
    assert got.shape == ref.shape and torch.equal(got, ref), (B, N, window, length, prefilter)


def test_smooth_segment_misuse(nets, raft):
    from vtoonify_b200.frame_loop import FramePipeline
    from vtoonify_b200.weights import det_inputs
    pipe = _pipe(nets, raft, 2, 2)
    plan = S.segment_plan(12, 2, 4)
    fr = _frames(12, 64, 64).to(DEV)
    seg = plan[1]
    bad = [((fr[seg.lo:seg.hi].float(), seg, 2), "uint8"), ((fr[seg.lo:seg.hi + 1], seg, 2), "uint8"),
           ((fr[seg.lo:seg.hi].cpu(), seg, 2), "CUDA"), ((fr[seg.lo:seg.hi], tuple(seg), 2), "Segment"),
           ((fr[seg.lo:seg.hi], seg._replace(lo=seg.lo + 1), 2), "not a segment"),
           ((fr[seg.lo:seg.hi], seg._replace(hi=seg.hi - 1), 2), "not a segment"),
           ((fr[seg.lo:seg.hi], seg, 3), "batch"), ((fr[seg.lo:seg.hi], seg, 0), "batch"),
           ((_frames(8, 60, 64).to(DEV), seg, 2), "multiples of 8")]
    for args, msg in bad:
        with pytest.raises(ValueError, match=msg):
            pipe.smooth_segment(*args)
    m, _ = nets
    plain = FramePipeline(m, det_inputs(1, 32, 32, seed=5)[1])
    with pytest.raises(ValueError, match="no smoothing"):
        plain.smooth_segment(fr[seg.lo:seg.hi], seg, 2)


# ---- the sharded driver over NCCL ---------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, q):
    try:
        import torch.distributed as dist
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        torch.set_grad_enabled(False)
        set_precision("bf16x3")
        from vtoonify_b200.frame_loop import FramePipeline, ShardedSmoothedVideo
        from vtoonify_b200.weights import det_inputs
        torch.manual_seed(0)
        raft_m = RAFT(raft_args()).eval()
        raft_m.load_state_dict(det_state_dict(raft_m, seed=0), strict=True)
        raft_m.requires_grad_(False)
        m, p = _nets()
        raft_m.to(dev)
        m.to(dev)
        p.to(dev)
        window, iters, H, W, B, length = 2, 2, 64, 64, 2, 4
        style = det_inputs(1, 32, 32, seed=5)[1]
        pipe = FramePipeline(m, style, d_s=0.5, device=dev, parsing_net=p, smoothing=(raft_m, window, iters))
        d2h = torch.cuda.Stream(dev)
        ok, msgs, peaks = True, [], []
        # 9 frames: N not a multiple of length, a last segment shorter than the window; then 2 * length, 4 * length, 2 * length
        for N in (9, 2 * length, 4 * length, 2 * length):
            frames = _frames(N, H, W, seed=N)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            drv = ShardedSmoothedVideo(pipe, N, length, (H, W), B, dev)
            if rank == 0:
                results = {}

                def sink(i, buf, ready):
                    with torch.cuda.stream(d2h):
                        ready()
                        results[i] = buf.to("cpu", non_blocking=True)
                        ev = torch.cuda.Event()
                        ev.record(d2h)
                    return ev

                # single frames for the short clip, batches of 3 for the others
                src = [frames[f] for f in range(N)] if N == 9 else [frames[f:f + 3] for f in range(0, N, 3)]
                drv.run(src, sink)
            else:
                drv.run()
            torch.cuda.synchronize()
            del drv
            peaks.append(torch.cuda.max_memory_allocated() - base)
            if rank == 0:
                got = torch.cat([results[i] for i in sorted(results)])
                ref = torch.cat(list(pipe.run(_batches(frames, B))))
                if sorted(results) != list(range(0, N, length)) or not torch.equal(got, ref):
                    ok = False
                    msgs.append(f"N={N}: sinks {sorted(results)}, frames equal {got.shape == ref.shape and torch.equal(got, ref)}")
        if rank == 0:
            print(f"rank 0 device peak above the models at world {world}: N={2 * length} {peaks[1] / 2 ** 20:.1f} MB, "
                  f"N={4 * length} {peaks[2] / 2 ** 20:.1f} MB, N={2 * length} again {peaks[3] / 2 ** 20:.1f} MB")
            if peaks[2] > 1.05 * min(peaks[1], peaks[3]) + 4 * 2 ** 20:
                ok = False
                msgs.append(f"rank 0 peak grows with the clip: {peaks}")
        q.put((rank, ok, "; ".join(msgs)))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, False, traceback.format_exc()))
        raise


def test_sharded_smoothed_video_nccl():
    world = min(2, torch.cuda.device_count())
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=900) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    assert all(ok for _, ok, _ in res), "\n".join(msg for _, _, msg in res)
