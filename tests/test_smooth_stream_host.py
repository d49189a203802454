"""Streaming parsing-map smoothing on the host: the release schedule of ParsingSmoother against slot_frames (every output once, only
when the frames its slots read are in the ring, with the slots the whole clip gives it) and the argument errors that need no GPU."""
import pytest
import torch

from tests.golden.make_golden_raft import raft_args
from vtoonify_b200 import smooth_parsing as S
from vtoonify_b200.raft import RAFT


def _lengths(window):
    return sorted({max(window, 1), window + 1, 2 * window + 1, 3 * window + 3})


@pytest.mark.parametrize("window", [0, 1, 2, 5])
def test_release_schedule_against_slot_frames(window):
    R = 2 * window + 1
    for N in _lengths(window):
        per_push, at_finish = S.release_schedule(N, window)
        assert len(per_push) == N
        slots = S.slot_frames(N, window)
        released = []
        for f, outs in enumerate(per_push):
            for i in outs:
                # frames 0..f are in; the ring holds f - R + 1 .. f
                assert max(slots[i]) <= f and min(slots[i]) >= f - R + 1, (N, f, i, slots[i])
                # before the end, the slots of output i do not depend on the clip length
                assert S.slot_frames(i + window + 1, window)[i] == slots[i]
            released += outs
        assert len(at_finish) == window
        for i in at_finish:
            assert min(slots[i]) >= N - R
        released += at_finish
        assert released == list(range(N)), (N, released)


@pytest.mark.parametrize("window", [1, 2, 5])
def test_finish_outputs_need_the_tail(window):
    """the outputs held back for finish() are exactly those whose slots reach past the last frame of the clip"""
    for N in _lengths(window):
        slots = S.slot_frames(N, window)
        _, at_finish = S.release_schedule(N, window)
        ext = list(range(window)) + list(range(N)) + list(range(N))[-window:]
        tail_users = [i for i in range(N) if i + 2 * window >= window + N]
        assert at_finish == tail_users
        for i in at_finish:
            assert slots[i] == ext[i:i + 2 * window + 1]


def _model():
    torch.manual_seed(0)
    m = RAFT(raft_args()).eval()
    m.requires_grad_(False)
    return m


def test_smoother_argument_errors():
    m = _model()
    with pytest.raises(ValueError, match="window"):
        S.ParsingSmoother(m, window=-1)
    with pytest.raises(ValueError, match="window"):
        S.ParsingSmoother(m, window=S.MAX_WINDOW + 1)
    with pytest.raises(ValueError, match="iters"):
        S.ParsingSmoother(m, window=2, iters=0)
    with pytest.raises(NotImplementedError, match="vtoonify_b200.raft.RAFT"):
        S.ParsingSmoother(torch.nn.Identity(), window=2)
    with pytest.raises(NotImplementedError, match="train mode"):
        S.ParsingSmoother(_model().train(), window=2)
    for window in (0, 1, 3):
        sm = S.ParsingSmoother(m, window=window)
        with pytest.raises(ValueError, match="fewer than the window"):
            sm.finish()                       # no frame pushed: fewer than max(window, 1)
    sm = S.ParsingSmoother(m, window=2)
    with pytest.raises(ValueError, match=r"\[3, H, W\]"):
        sm.push(torch.zeros(4, 128, 128), torch.zeros(19, 128, 128))
    with pytest.raises(ValueError, match=r"\[C, H, W\]"):
        sm.push(torch.zeros(3, 128, 128), torch.zeros(19, 128, 120))


def test_frame_prep_and_fuse_down_reject_bad_inputs():
    with pytest.raises(ValueError, match="uint8"):
        S.frame_prep(torch.zeros(1, 8, 8, 3))
    with pytest.raises(ValueError, match="at least one centre"):
        S.parsing_fuse_down([], [1.0], torch.zeros(1, 4, 4, 4))
    img, par = torch.zeros(3, 8, 8), torch.zeros(4, 8, 8)
    with pytest.raises(ValueError, match="slots"):
        S.parsing_fuse_down([([img, img], [par, par], [None, None])], [1.0, 1.0], torch.zeros(1, 4, 4, 4))
    with pytest.raises(ValueError, match="slot 0"):
        S.parsing_fuse_down([([img], [torch.zeros(4, 8, 9)], [None])], [1.0], torch.zeros(1, 4, 4, 4))


@pytest.mark.parametrize("window", [0, 1, 2, 5, 31])
def test_per_push_helpers_equal_the_whole_clip_schedule(window):
    """what a push and finish compute in O(window) equals the whole-clip oracle: released_by_push against release_schedule, and
    output_slots against slot_frames for every output released before finish (without N) and at finish (with N)"""
    for N in sorted({max(window, 1), window + 1, 2 * window + 1, 3 * window + 3, 4 * window + 7}):
        per_push, at_finish = S.release_schedule(N, window)
        slots = S.slot_frames(N, window)
        for f in range(N):
            assert S.released_by_push(f, window) == per_push[f]
            for i in per_push[f]:
                assert S.output_slots(i, window) == slots[i], (N, i)
        for i in range(N):
            assert S.output_slots(i, window, N) == slots[i], (N, i)
        assert at_finish == list(range(N - window, N))


def test_per_push_helpers_do_not_grow_with_the_clip():
    """the helpers a push calls take the same work at frame 10^9 as at frame 10: their results are O(window) lists computed from the
    indices alone"""
    w = 5
    f = 10 ** 9
    assert S.released_by_push(f, w) == [f - w]
    assert S.output_slots(f - w, w) == list(range(f - 2 * w, f + 1))
    assert S.output_slots(f - 1, w, f) == [f - 1 - w + k for k in range(w + 1)] + list(range(f - w, f))
