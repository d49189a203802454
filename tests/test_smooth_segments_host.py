"""Segmented parsing-map smoothing on the host: segment_plan against the whole-clip slot_frames (every output once, in order, each slot
pushed by its segment, each output released by a push or by its segment's finish(), halos no wider than the window), the release rule
of a stream that starts at frame ``first`` against release_schedule, and the sharded driver over gloo at world 2 and 3 with a stub
segment function."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from vtoonify_b200 import smooth_parsing as S

WINDOWS = [0, 1, 2, 3, 4, 5, 6, 7, 31]


def _released(seg, N, window):
    """the outputs a ParsingSmoother(first=seg.lo) releases over the segment's pushes and, with seg.finish, its finish()"""
    out = [i for f in range(seg.lo, seg.hi) for i in S.released_by_push(f, window, seg.lo)]
    if seg.finish:
        assert seg.hi == N
        out += S.released_at_finish(N, window, seg.lo)
    return out


@pytest.mark.parametrize("window", WINDOWS)
def test_segment_plan_against_slot_frames(window):
    for N in range(max(window, 1), 151):
        slots = S.slot_frames(N, window)
        lo_slot, hi_slot = [min(s) for s in slots], [max(s) for s in slots]
        for length in range(1, 41):
            plan = S.segment_plan(N, window, length)
            assert [i for seg in plan for i in range(seg.a, seg.b)] == list(range(N)), (N, length)
            for seg in plan:
                assert seg.b - seg.a == length or seg.b == N
                assert 0 <= seg.lo <= seg.a < seg.b <= seg.hi <= N
                assert seg.a - seg.lo <= window and (seg.hi - seg.b <= window)
                # a segment calls finish() exactly when one of its outputs is a tail output, and then pushes to the clip's end
                assert seg.finish == any(i + window >= N for i in range(seg.a, seg.b))
                if not seg.finish:
                    assert seg.hi == seg.b + window
                for i in range(seg.a, seg.b):
                    assert seg.lo <= lo_slot[i] and hi_slot[i] < seg.hi, (N, length, seg, i)
                released = _released(seg, N, window)
                assert len(released) == len(set(released))
                assert set(range(seg.a, seg.b)) <= set(released), (N, length, seg)
                # a released output's slots are all pushed
                for i in released:
                    assert seg.lo <= lo_slot[i] and hi_slot[i] < seg.hi


def test_segment_plan_examples_and_errors():
    P = S.Segment
    assert S.segment_plan(20, 5, 8) == [P(0, 8, 0, 13, False), P(8, 16, 3, 20, True), P(16, 20, 11, 20, True)]
    assert S.segment_plan(7, 0, 3) == [P(0, 3, 0, 3, False), P(3, 6, 3, 6, False), P(6, 7, 6, 7, False)]
    assert S.segment_plan(5, 5, 16) == [P(0, 5, 0, 5, True)]
    for N, window in ((0, 0), (4, 5), (30, 31)):
        with pytest.raises(ValueError, match="fewer than the window"):
            S.segment_plan(N, window, 4)
    for length in (0, -1, 2.5):
        with pytest.raises(ValueError, match="length"):
            S.segment_plan(10, 2, length)
    for window in (-1, S.MAX_WINDOW + 1, 1.5):
        with pytest.raises(ValueError, match="window"):
            S.segment_plan(40, window, 4)


@pytest.mark.parametrize("window", [0, 1, 2, 5, 31])
def test_release_rule_with_first_against_release_schedule(window):
    """a stream from frame ``first`` releases what the whole clip's schedule releases, less the outputs with a slot before ``first``;
    ``first = 0`` is the whole clip's schedule itself"""
    for N in sorted({max(window, 1), window + 1, 2 * window + 1, 3 * window + 3, 4 * window + 7}):
        per_push, at_finish = S.release_schedule(N, window)
        slots = S.slot_frames(N, window)
        for first in range(N):
            for f in range(first, N):
                want = [i for i in per_push[f] if min(slots[i]) >= first]
                assert S.released_by_push(f, window, first) == want, (N, first, f)
                if first == 0:
                    assert S.released_by_push(f, window) == per_push[f]
            want = [i for i in at_finish if min(slots[i]) >= first]
            assert S.released_at_finish(N, window, first) == want, (N, first)
            if first == 0:
                assert S.released_at_finish(N, window) == at_finish
            if first > 0:
                assert all(i >= first + window for f in range(first, N) for i in S.released_by_push(f, window, first))


def test_smoother_first_is_checked():
    from tests.golden.make_golden_raft import raft_args
    from vtoonify_b200.raft import RAFT
    m = RAFT(raft_args()).eval()
    m.requires_grad_(False)
    for first in (-1, 1.5):
        with pytest.raises(ValueError, match="first"):
            S.ParsingSmoother(m, 2, 2, first=first)
    sm = S.ParsingSmoother(m, 2, 2, first=7)
    assert sm.finish() == []                  # N = 7 frames, none pushed here: nothing of this stream is computable


# ---- the sharded driver over gloo, with a stub segment function ---------------------------------------------------------------
H, W = 3, 2


def _frame(f):
    g = torch.Generator().manual_seed(1000 + f)
    return torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8)


def _checksum(frames_by_index, slots, i):
    """a stand-in for a smoothed, synthesised output: depends on which frames fill output i's slots, in order"""
    acc = torch.zeros((H, W, 3), dtype=torch.int64)
    for k, f in enumerate(slots):
        acc += (k + 1) * frames_by_index(f).long()
    acc += i
    return (acc % 251).to(torch.uint8).repeat_interleave(4, 0).repeat_interleave(4, 1)


class _StubPipe:
    """what ShardedSmoothedVideo uses of a FramePipeline: ``smoothing``, ``prefilter`` and ``smooth_segment``"""

    def __init__(self, N, window, batch):
        self.smoothing, self.prefilter = (None, window, 1), None
        self.N, self.window, self.batch = N, window, batch
        self.received = []

    def smooth_segment(self, frames, seg, batch):
        assert batch == self.batch and seg.a % batch == 0
        assert frames.dtype == torch.uint8 and frames.shape == (seg.hi - seg.lo, H, W, 3)
        self.received.append((seg, frames.clone()))
        slots = S.slot_frames(self.N, self.window)
        return torch.stack([_checksum(lambda f: frames[f - seg.lo], slots[i], i) for i in range(seg.a, seg.b)])


def _driver_worker(rank, world, port, N, window, length, batch, items, q):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from vtoonify_b200.frame_loop import ShardedSmoothedVideo
        pipe = _StubPipe(N, window, batch)
        drv = ShardedSmoothedVideo(pipe, N, length, (H, W), batch, "cpu")
        plan = S.segment_plan(N, window, length)
        ok, msg = True, ""
        if rank == 0:
            clip = torch.stack([_frame(f) for f in range(N)])
            reads = []

            def frames():                      # single frames or uneven batches, read once and in order
                f = 0
                for n in items:
                    n = min(n, N - f)
                    if n <= 0:
                        break
                    reads.append(f)
                    yield clip[f] if n == 1 else clip[f:f + n]
                    f += n
                while f < N:
                    reads.append(f)
                    yield clip[f]
                    f += 1

            got = []

            def sink(i, buf, ready):
                ready()
                got.append((i, buf.clone()))

            mine = drv.run(frames(), sink)
            slots = S.slot_frames(N, window)
            want = torch.stack([_checksum(lambda f: clip[f], slots[i], i) for i in range(N)])
            ok = [i for i, _ in got] == [seg.a for seg in plan]
            ok = ok and torch.equal(torch.cat([b for _, b in got]), want)
            ok = ok and reads == sorted(set(reads))
            if not ok:
                msg = f"rank 0: sinks at {[i for i, _ in got]}, plan {plan}"
        else:
            clip = torch.stack([_frame(f) for f in range(N)])
            mine = drv.run()
        # each rank received exactly its segments, each with its halo'd frames
        want_segs = [plan[i] for i in range(rank, len(plan), world)]
        ok = ok and mine == len(want_segs) and [s for s, _ in pipe.received] == want_segs
        ok = ok and all(torch.equal(fr, clip[s.lo:s.hi]) for s, fr in pipe.received)
        if not ok and not msg:
            msg = f"rank {rank}: received {[s for s, _ in pipe.received]}, want {want_segs}"
        q.put((rank, bool(ok), msg))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, False, traceback.format_exc()))
        raise


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# (world, N, window, length, batch, items): N not a multiple of length, a last segment shorter than the window, more ranks than
# segments, window 0, and frames arriving as single frames and as uneven batches
CASES = [(2, 23, 2, 4, 2, [1]), (2, 21, 5, 8, 4, [3, 5, 1, 7]), (3, 26, 3, 6, 3, [4]), (3, 10, 2, 8, 2, [10]),
         (3, 7, 0, 2, 1, [2, 2]), (2, 5, 5, 4, 2, [5]), (3, 40, 7, 4, 4, [6, 1])]


@pytest.mark.parametrize("world,N,window,length,batch,items", CASES)
def test_sharded_smoothed_video_gloo(world, N, window, length, batch, items):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_driver_worker, args=(r, world, port, N, window, length, batch, items, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _ in res), "\n".join(msg for _, _, msg in res)


def test_sharded_smoothed_video_argument_errors():
    pipe = _StubPipe(10, 2, 2)
    from vtoonify_b200.frame_loop import ShardedSmoothedVideo
    bad = [((pipe, 10, 3, (H, W), 2), "multiple of the batch"), ((pipe, 10, 0, (H, W), 1), "length"),
           ((pipe, 1, 4, (H, W), 2), "fewer than the window"), ((pipe, 10, 4, (H,), 2), "frame_shape"),
           ((pipe, 10, 4, (H, 0), 2), "frame_shape")]
    for args, msg in bad:
        with pytest.raises(ValueError, match=msg):
            ShardedSmoothedVideo(*args, "cpu")
    nosmooth = _StubPipe(10, 2, 2)
    nosmooth.smoothing = None
    with pytest.raises(ValueError, match="no smoothing"):
        ShardedSmoothedVideo(nosmooth, 10, 4, (H, W), 2, "cpu")


def test_halo_reader_checks_the_clip():
    from vtoonify_b200.frame_loop import _HaloReader
    clip = torch.stack([_frame(f) for f in range(6)])
    r = _HaloReader([clip[:2], clip[2], clip[3:6]], 6, (H, W))
    assert all(torch.equal(r.frame(f), clip[f]) for f in range(6))
    r.drop_before(4)
    assert r.base == 4 and len(r.kept) == 2
    for frames, msg in (([clip[:3]], "ended after 3"), ([clip[:4], clip[4:6], clip[:1]], "more than"),
                        ([clip[:2].float()], "uint8"), ([clip[:2, :, :1]], "uint8")):
        r = _HaloReader(frames, 5, (H, W))
        with pytest.raises(ValueError, match=msg):
            for f in range(5):
                r.frame(f)
