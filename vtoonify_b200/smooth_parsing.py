"""Temporal smoothing of face-parsing maps (smooth_parsing_map.py) on the library.

``warp(x, flo)`` is a drop-in for the script's ``warp``: the same ``(output * mask, mask)``, the mask materialised at ``[B, C, H, W]``.

``smooth_parsing_maps(Is, Ps, raft_model, window=5, iters=20)`` is the script's whole smoothing loop (lines 143-167): it returns its
``parse`` ``[N, C, H/2, W/2]`` on ``Ps``'s device, given the script's ``Is`` (the 2x up-sampled frames in [-1, 1], ``[N, 3, H, W]``) and
``Ps`` (the parsing logits, ``[N, C, H, W]``), on the CPU or on the device.  ``raft_model`` is a ``vtoonify_b200.raft.RAFT``.

The loop streams (DESIGN.md section 12):
  * a device ring of the ``2 * window + 1`` frames of the current window holds each frame's image, its RAFT input
    ``(I + 1) * 255.0 / 2``, its parsing map and its ``fnet`` features; every frame is uploaded and encoded once, and device memory does
    not grow with ``N``;
  * slot ``k`` of output frame ``i`` reads frame ``slot_frames(N, window)[i][k]``, the reference's ``cat((Is[0:w], Is, Is[-w:]))``
    indexing, boundary windows included (a frame may fill two slots, or the centre's own frame a non-centre slot: those pairs run);
  * per output frame: ``cnet`` once on the centre, the RAFT iterations on the ``2 * window`` non-centre pairs as one batch, one fusion
    launch (warp, spatial weights, normalisation and the weighted sum; nothing ``[11, 22, H, W]``-sized is materialised) and one
    ``Downsample([1, 3, 3, 1], 2)`` launch.  The centre pair RAFT(I_i, I_i) of the script is skipped: the script overwrites both of
    its results.
The RAFT convolutions follow ``set_precision``; the warp and the fusion are fp32 in every mode.

``ParsingSmoother`` is that loop as a stream (``smooth_parsing_maps`` is a loop over its ``push`` and ``finish``): one frame in, the
outputs that have become computable out, so neither side holds the clip.  ``FramePipeline(smoothing=...)`` runs it between the face
parsing and the synthesis, with ``frame_prep`` (uint8 frames -> ``Is`` and RAFT's stem input in one launch) and
``parsing_fuse_down`` (fusion, ``Downsample`` and the ``/ 16`` of style_transfer.py in one launch) (DESIGN.md section 13).
``segment_plan`` cuts a clip into segments that smooth independently, each pushing its frames and a halo of ``window`` frames on
each side into a ``ParsingSmoother(first=...)`` (DESIGN.md section 14).
"""
import collections

import torch

from . import ops
from ._lib import c_float, c_void_p, check, load
from .raft import MIN_SIZE, RAFT
from .stylegan import make_kernel

MAX_WINDOW = 31             # the fusion kernel's slot table holds 2 * 31 + 1 slots


def temporal_weights(window: int) -> torch.Tensor:
    """the script's ``wt`` (line 144), float32 on the CPU, ``[2 * window + 1]``"""
    return torch.exp(-(torch.arange(2 * window + 1).float() - window) ** 2 / (2 * ((window + 0.5) ** 2))).reshape(2 * window + 1)


def slot_frames(N: int, window: int):
    """for each output frame i, the frame index behind each of its ``2 * window + 1`` slots: ``Is_[i : i + 2w + 1]`` with
    ``Is_ = cat((Is[0:w], Is, Is[-w:]))`` (``Is[-0:]`` is all of ``Is``, as in Python)"""
    head = list(range(0, min(window, N)))
    tail = list(range(N))[-window:] if window else list(range(N))
    ext = head + list(range(N)) + tail
    return [ext[i:i + 2 * window + 1] for i in range(N)]


def _check_no_grad(name, *ts):
    if torch.is_grad_enabled():
        for t in ts:
            if t is not None and t.requires_grad:
                raise NotImplementedError(f"{name}: inputs that require grad are not supported (forward only; run under torch.no_grad())")


def warp(x: torch.Tensor, flo: torch.Tensor):
    """smooth_parsing_map.py:38-74 on planar fp32 CUDA tensors: x [B, C, H, W], flo [B, 2, H, W] -> (warped x * mask, mask)"""
    _check_no_grad("warp", x, flo)
    if x.dim() != 4 or flo.dim() != 4 or flo.shape[1] != 2 or flo.shape[0] != x.shape[0] or flo.shape[2:] != x.shape[2:]:
        raise ValueError(f"warp: x {tuple(x.shape)} must be [B, C, H, W] and flo {tuple(flo.shape)} [B, 2, H, W]")
    ops._req_cuda(x, flo)
    B, C, H, W = x.shape
    x, flo = x.contiguous(), flo.contiguous()
    out = torch.empty_like(x)
    mask = torch.empty_like(x)
    check(load().vt_flow_warp_f32(x.data_ptr(), flo.data_ptr(), out.data_ptr(), mask.data_ptr(), B, C, H, W, ops._stream()))
    return out, mask


def parsing_fuse(imgs, pars, flows, wt, out=None):
    """one centre of the window fusion (script lines 155-165 before ``down``): per-slot planar CUDA tensors imgs[k] [3, H, W],
    pars[k] [C, H, W], flows[k] [2, H, W] (``flows[window]`` is ignored and may be None), host weights wt [2 * window + 1] ->
    fused [C, H, W]"""
    n = len(imgs)
    if n % 2 != 1 or n > 2 * MAX_WINDOW + 1 or len(pars) != n or len(flows) != n or len(wt) != n:
        raise ValueError(f"parsing_fuse: need 2 * window + 1 <= {2 * MAX_WINDOW + 1} slots in every list")
    C, H, W = pars[0].shape
    for k in range(n):
        ok = tuple(imgs[k].shape) == (3, H, W) and tuple(pars[k].shape) == (C, H, W)
        ok = ok and (k == n // 2 or tuple(flows[k].shape) == (2, H, W))
        if not ok:
            raise ValueError(f"parsing_fuse: slot {k} must hold [3, {H}, {W}], [{C}, {H}, {W}] and [2, {H}, {W}] tensors")
        ops._req_cuda(imgs[k], pars[k], None if k == n // 2 else flows[k])
        if not (imgs[k].is_contiguous() and pars[k].is_contiguous() and (k == n // 2 or flows[k].is_contiguous())):
            raise ValueError(f"parsing_fuse: slot {k} tensors must be contiguous")
    if out is None:
        out = torch.empty((C, H, W), device=pars[0].device, dtype=torch.float32)
    ptrs = [(c_void_p * n)(*[None if t is None else t.data_ptr() for t in ts]) for ts in (imgs, pars, flows)]
    w = (c_float * n)(*[float(v) for v in wt])
    check(load().vt_parsing_fuse_f32(ptrs[0], ptrs[1], ptrs[2], w, n, out.data_ptr(), C, H, W, ops._stream()))
    return out


def parsing_fuse_down(centres, wt, out, scale=1.0):
    """``len(centres)`` centres of the window fusion, each followed by ``Downsample([1, 3, 3, 1], 2)`` and ``* scale``, in one launch
    that never writes the fused 2x map: ``centres[b] = (imgs, pars, flows)`` as for :func:`parsing_fuse`, host weights wt, and
    ``out`` [B, C, H/2, W/2] (each sample contiguous, any batch stride: e.g. ``x[:, 3:]`` of VToonify's input).  Bit-identical to
    :func:`parsing_fuse`, then ``ops.upfirdn2d_planar`` and ``ops.axpby(.., scale)`` (TF32-rounded under ``set_precision('tf32')``
    like ``axpby``)."""
    B = len(centres)
    if B < 1:
        raise ValueError("parsing_fuse_down: need at least one centre")
    n = len(centres[0][0])
    if n % 2 != 1 or n > 2 * MAX_WINDOW + 1 or len(wt) != n:
        raise ValueError(f"parsing_fuse_down: need 2 * window + 1 <= {2 * MAX_WINDOW + 1} slots and as many weights")
    C, H, W = centres[0][1][0].shape
    for imgs, pars, flows in centres:
        if len(imgs) != n or len(pars) != n or len(flows) != n:
            raise ValueError("parsing_fuse_down: every centre needs the same number of slots")
        for k in range(n):
            ok = tuple(imgs[k].shape) == (3, H, W) and tuple(pars[k].shape) == (C, H, W)
            ok = ok and (k == n // 2 or tuple(flows[k].shape) == (2, H, W))
            if not ok:
                raise ValueError(f"parsing_fuse_down: slot {k} must hold [3, {H}, {W}], [{C}, {H}, {W}] and [2, {H}, {W}] tensors")
            ops._req_cuda(imgs[k], pars[k], None if k == n // 2 else flows[k])
            if not (imgs[k].is_contiguous() and pars[k].is_contiguous() and (k == n // 2 or flows[k].is_contiguous())):
                raise ValueError(f"parsing_fuse_down: slot {k} tensors must be contiguous")
    Ho, Wo = H // 2, W // 2
    ops._req_cuda(out)
    if (out.dim() != 4 or tuple(out.shape) != (B, C, Ho, Wo) or out.stride()[1:] != (Ho * Wo, Wo, 1)
            or (B > 1 and out.stride(0) < C * Ho * Wo)):
        raise ValueError(f"parsing_fuse_down: out must be [{B}, {C}, {Ho}, {Wo}] with contiguous samples (got {tuple(out.shape)}, "
                         f"strides {out.stride()})")
    ptrs = [(c_void_p * (B * n))(*[None if t is None else t.data_ptr() for c in centres for t in c[j]]) for j in range(3)]
    w = (c_float * n)(*[float(v) for v in wt])
    check(load().vt_parsing_fuse_down_f32(ptrs[0], ptrs[1], ptrs[2], w, n, B, out.data_ptr(), out.stride(0), C, H, W, float(scale),
                                          ops._round_flag(), ops._stream()))
    return out


def frame_prep(frames: torch.Tensor, cpad: int = 32):
    """uint8 RGB frames [B, H, W, 3] on the device -> (Is [B, 3, 2H, 2W], stem [B, H, W, cpad]) in one launch: the script's
    ``F.interpolate(transform(frame), scale_factor=2, mode='bilinear')`` and RAFT's stem input ``raft._input_s2d((Is + 1) * 255.0 / 2)``
    with the script's three roundings.  The up-sampling is ``ops.frame_s2d``'s: ``frame_s2d(frames_u8_to_f32(frames), upsample2=True)``
    equals ``frame_s2d(2 * Is, upsample2=False)`` bit for bit."""
    if not frames.is_cuda or frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError("frame_prep: frames must be a CUDA uint8 [B, H, W, 3] tensor")
    frames = frames.contiguous()
    B, H, W, _ = frames.shape
    img = torch.empty((B, 3, 2 * H, 2 * W), device=frames.device, dtype=torch.float32)
    stem = torch.empty((B, H, W, cpad), device=frames.device, dtype=torch.float32)
    check(load().vt_smooth_frame_prep_u8(frames.data_ptr(), img.data_ptr(), stem.data_ptr(), B, H, W, cpad, ops._stream()))
    return img, stem


def _check_model_window(name, raft_model, window, iters):
    if not isinstance(raft_model, RAFT):
        raise NotImplementedError(f"{name}: raft_model must be a vtoonify_b200.raft.RAFT")
    raft_model._check_model()
    if int(window) != window or window < 0 or window > MAX_WINDOW:
        raise ValueError(f"{name}: window must be an integer in 0..{MAX_WINDOW} (got {window})")
    if int(iters) < 1:
        raise ValueError(f"{name}: iters must be at least 1")


def release_schedule(N: int, window: int):
    """which outputs :class:`ParsingSmoother` hands back: ``(per_push, at_finish)`` with ``per_push[f]`` the output indices the push of
    frame f returns (output i once frame i + window is in) and ``at_finish`` the last ``window`` (their tail slots repeat
    ``Is[-window:]``, known only at the end).  The whole clip's schedule; a push computes its own entry with
    :func:`released_by_push`."""
    per_push = [[f - window] if f >= window else [] for f in range(N)]
    return per_push, list(range(max(N - window, 0), N)) if window else []


def released_by_push(f: int, window: int, first: int = 0):
    """the outputs the push of frame f releases, ``release_schedule(N, window)[0][f]`` for any N > f, in O(1).  For a stream whose
    first frame is ``first``, only the outputs whose slots are all pushed: those with i >= first + window when first > 0."""
    i = f - window
    return [i] if i >= 0 and max(0, i - window) >= first else []


def released_at_finish(N: int, window: int, first: int = 0):
    """the outputs ``finish()`` releases for a clip of N frames, ``release_schedule(N, window)[1]``; for a stream whose first frame is
    ``first``, only those whose slots are all pushed, as for :func:`released_by_push`"""
    return list(range(max(N - window, first + window if first else 0), N))


Segment = collections.namedtuple("Segment", "a b lo hi finish")
Segment.__doc__ = """one segment of :func:`segment_plan`: outputs ``[a, b)``, frames ``[lo, hi)`` pushed into a
``ParsingSmoother(first=lo)``, and whether the segment ends with ``finish()`` (then ``hi`` is the clip's N)"""


def segment_plan(N: int, window: int, length: int):
    """Cut the outputs ``0..N-1`` of a clip into consecutive segments of ``length`` outputs (the last may be shorter) that can be
    smoothed independently: a segment pushes its outputs' frames and up to ``window`` frames on each side (its halo), so every slot of
    its outputs is pushed.  A segment with a tail output (``i + window >= N``, released only by ``finish()``) pushes to the clip's
    end and calls ``finish()``.  Returns a list of :class:`Segment` (DESIGN.md section 14)."""
    if int(N) != N or int(window) != window or window < 0 or window > MAX_WINDOW:
        raise ValueError(f"segment_plan: N must be an integer and window an integer in 0..{MAX_WINDOW} (got {N}, {window})")
    if int(length) != length or length < 1:
        raise ValueError(f"segment_plan: length must be a positive integer (got {length})")
    N, window, length = int(N), int(window), int(length)
    if N < max(window, 1):
        raise ValueError(f"segment_plan: {N} frames are fewer than the window {window} (the script's RAFT batches would not match)")
    plan = []
    for a in range(0, N, length):
        b = min(a + length, N)
        finish = b - 1 + window >= N
        plan.append(Segment(a, b, max(0, a - window), N if finish else b + window, finish))
    return plan


def output_slots(i: int, window: int, N: int = None):
    """``slot_frames(N, window)[i]`` in O(window): slot k of output i is frame i + k - window, or frame i + k in the head
    (i + k < window: ``Is[0:w]``); with N given, the tail (i + k >= window + N: ``Is[-w:]``) is frame i + k - 2 * window.  Without N,
    i must be released before the end of the clip (i + window < N for the clip's N), where the tail is never reached."""
    out = []
    for j in range(i, i + 2 * window + 1):
        if j < window:
            out.append(j)
        elif N is None or j < window + N:
            out.append(j - window)
        else:
            out.append(j - 2 * window)
    return out


class SmoothedFrame:
    """one output frame of :class:`ParsingSmoother`, computable from the ring: ``down()`` gives its parsing map [C, H/2, W/2]
    (``parsing_fuse`` then ``Downsample``, the route of ``smooth_parsing_maps``), ``fuse_down(out, scale)`` writes ``scale`` times
    the same map into ``out`` in one launch.  The RAFT flows of the centre run on the first of them.  A handle returned by ``push``
    is valid until the next ``push``; those returned by ``finish`` stay valid."""

    def __init__(self, smoother, index, pos):
        self.index = index
        self._sm, self._pos, self._flows = smoother, pos, None
        self._pushed = smoother.n            # the ring holds this handle's frames while no further frame is pushed

    def _slots(self):
        sm, pos = self._sm, self._pos
        if sm.n != self._pushed:
            raise RuntimeError(f"SmoothedFrame {self.index}: read after a later push (frame {sm.n - 1}) has overwritten its window; "
                               "read each handle before pushing the next frame")
        if self._flows is None:
            self._flows = sm._flows(self.index, pos)
        return [sm._img[p] for p in pos], [sm._par[p] for p in pos], self._flows

    def down(self):
        imgs, pars, flows = self._slots()
        sm = self._sm
        parsing_fuse(imgs, pars, flows, sm.wt, out=sm._fused)
        return ops.upfirdn2d_planar(sm._fused[None], sm._kernel, (1, 1), (2, 2), (1, 1, 1, 1))[0]

    def fuse_down(self, out, scale=1.0):
        parsing_fuse_down([self._slots()], self._sm.wt, out[None], scale)
        return out


class ParsingSmoother:
    """The smoothing loop of smooth_parsing_map.py as a stream: ``push(I, P)`` takes one frame's 2x image ``I`` [3, H, W] in [-1, 1] and
    parsing logits ``P`` [C, H, W] on the device and returns the :class:`SmoothedFrame` handles that have become computable (output i
    once frame i + window is in); ``finish()`` returns the last ``window`` outputs, whose tail slots repeat the clip's last frames.
    Device memory is a ring of the ``2 * window + 1`` frames of the current window and does not grow with the clip (DESIGN.md
    section 12).  ``push(I, P, stem)`` takes RAFT's stem input of ``(I + 1) * 255.0 / 2`` precomputed ([1, H/2, W/2, 32], e.g.
    from :func:`frame_prep`) instead of computing it.  Each output's cnet state and flows are computed when its handle is first
    read, so a consumer reads every handle before pushing the next frame: a handle read after a later push raises
    ``RuntimeError``, and so does a push after ``finish``.  Host work per frame is O(window), whatever the clip's length.

    ``first`` numbers the pushed frames from that clip index (a segment of :func:`segment_plan`): output i is released only once every
    frame of its slots is in, i.e. i >= first + window when first > 0, and ``finish()`` applies the tail rule to the clip's
    N = first + frames pushed."""

    def __init__(self, raft_model: RAFT, window: int = 5, iters: int = 20, first: int = 0):
        _check_model_window("ParsingSmoother", raft_model, window, iters)
        if int(first) != first or first < 0:
            raise ValueError(f"ParsingSmoother: first must be a non-negative integer (got {first})")
        self.model, self.window, self.iters = raft_model, int(window), int(iters)
        self.first = int(first)
        self.R = 2 * self.window + 1
        self.wt = temporal_weights(self.window).tolist()
        self.n = 0                          # frames pushed
        self.finished = False
        self.flow_sink = None               # tests: flow_sink(i, up) receives output i's up-sampled flows [2 * window, 2, H, W]
        self._img = None

    def _alloc(self, I, P):
        R, dev = self.R, I.device
        C, H, W = P.shape
        self.shape = (C, H, W)
        # the ring: frame f lives at position f % R (the frames one output reads span at most R consecutive indices)
        self._img = torch.empty((R, 3, H, W), device=dev, dtype=torch.float32)
        self._par = torch.empty((R, C, H, W), device=dev, dtype=torch.float32)
        self._fmap = [None] * R
        self._stem = [None] * R             # pushed stem inputs; frames pushed without one keep (I + 1) * 255 / 2 in _rin
        self._rin = None
        self._fused = torch.empty((C, H, W), device=dev, dtype=torch.float32)
        self._kernel = make_kernel([1, 3, 3, 1]).to(dev)

    def push(self, I: torch.Tensor, P: torch.Tensor, stem: torch.Tensor = None):
        # every argument is checked before any state changes
        if self.finished:
            raise RuntimeError("ParsingSmoother.push: the clip has ended (finish() was called)")
        if I.dim() != 3 or I.shape[0] != 3 or P.dim() != 3 or P.shape[1:] != I.shape[1:]:
            raise ValueError(f"ParsingSmoother.push: I {tuple(I.shape)} must be [3, H, W] and P {tuple(P.shape)} [C, H, W]")
        ops._req_cuda(I, P, stem)
        H, W = I.shape[1:]
        if H % 8 or W % 8 or H < MIN_SIZE or W < MIN_SIZE:
            raise ValueError(f"ParsingSmoother.push: H and W must be multiples of 8 and at least {MIN_SIZE} (got {H}x{W})")
        if self._img is not None and tuple(P.shape) != self.shape:
            raise ValueError(f"ParsingSmoother.push: P {tuple(P.shape)} differs from the clip's {self.shape}")
        if stem is not None and (tuple(stem.shape) != (1, H // 2, W // 2, 32) or not stem.is_contiguous()):
            raise ValueError(f"ParsingSmoother.push: stem must be contiguous [1, {H // 2}, {W // 2}, 32]")
        if self._img is None:
            self._alloc(I, P)
        f, m = self.first + self.n, self.model
        r = f % self.R
        with torch.no_grad():
            self._img[r].copy_(I)
            self._par[r].copy_(P)
            if self.window:
                if stem is None:
                    if self._rin is None:
                        self._rin = torch.empty_like(self._img)
                    torch.add(self._img[r], 1, out=self._rin[r]).mul_(255.0).div_(2)    # the script's (I + 1) * 255.0 / 2
                    self._stem[r] = None
                    self._fmap[r] = m._features(m._input_s2d(self._rin[r:r + 1]))
                else:
                    self._stem[r] = stem
                    self._fmap[r] = m._features(stem)
        self.n += 1
        return [self._ready(i) for i in released_by_push(f, self.window, self.first)]

    def finish(self):
        N = self.first + self.n
        if N < max(self.window, 1):
            raise ValueError(f"ParsingSmoother: {N} frames are fewer than the window {self.window} (the script's RAFT batches would "
                             "not match)")
        self.finished = True
        return [self._ready(i, N) for i in released_at_finish(N, self.window, self.first)]

    def _ready(self, i, N=None):
        # before the end, output i's slots never reach the tail, so they do not depend on the clip's length
        return SmoothedFrame(self, i, [f % self.R for f in output_slots(i, self.window, N)])

    def _flows(self, i, pos):
        """cnet once on the centre, the RAFT iterations on the 2 * window non-centre pairs as one batch (the script's centre pair is
        skipped: the script overwrites both of its results)"""
        w, R, m = self.window, self.R, self.model
        if not w:
            return [None]
        c = pos[w]
        nb = [pos[k] for k in range(R) if k != w]
        B = len(nb)
        with torch.no_grad():
            f1 = self._fmap[c].expand(B, -1, -1, -1)
            if ops.get_option("raft_corr") != "on_demand":      # the on-demand lookup reads one map at batch stride 0
                f1 = f1.contiguous()
            f2 = torch.cat([self._fmap[p] for p in nb], 0)
            stem = self._stem[c] if self._stem[c] is not None else m._input_s2d(self._rin[c:c + 1])
            net, x = m._context(stem)
            _, up = m._iterate(f1, f2, net.expand(B, -1, -1, -1).contiguous(), x.expand(B, -1, -1, -1).contiguous(), self.iters)
        if self.flow_sink is not None:
            self.flow_sink(i, up)
        return [up[k if k < w else k - 1] if k != w else None for k in range(R)]


def _check_args(Is, Ps, raft_model, window, iters):
    _check_model_window("smooth_parsing_maps", raft_model, window, iters)
    _check_no_grad("smooth_parsing_maps", Is, Ps)
    if Is.dim() != 4 or Is.shape[1] != 3 or Ps.dim() != 4 or Ps.shape[0] != Is.shape[0] or Ps.shape[2:] != Is.shape[2:]:
        raise ValueError(f"smooth_parsing_maps: Is {tuple(Is.shape)} must be [N, 3, H, W] and Ps {tuple(Ps.shape)} [N, C, H, W]")
    if Is.dtype != torch.float32 or Ps.dtype != torch.float32:
        raise ValueError(f"smooth_parsing_maps: Is and Ps must be float32 (got {Is.dtype}, {Ps.dtype})")
    N, _, H, W = Is.shape
    if N < max(window, 1):
        raise ValueError(f"smooth_parsing_maps: {N} frames are fewer than the window {window} (the script's RAFT batches would not match)")
    if H % 8 or W % 8 or H < MIN_SIZE or W < MIN_SIZE:
        raise ValueError(f"smooth_parsing_maps: H and W must be multiples of 8 and at least {MIN_SIZE} (got {H}x{W})")


def smooth_parsing_maps(Is: torch.Tensor, Ps: torch.Tensor, raft_model: RAFT, window: int = 5, iters: int = 20) -> torch.Tensor:
    """smooth_parsing_map.py:143-167: the temporally fused, down-sampled parsing maps [N, C, H/2, W/2] on ``Ps``'s device"""
    return _smooth(Is, Ps, raft_model, window, iters)


def _smooth(Is, Ps, raft_model, window, iters, flow_sink=None):
    """smooth_parsing_maps as a loop over ParsingSmoother.push and finish; ``flow_sink(i, up)`` (tests) receives output frame i's
    up-sampled flows [2 * window, 2, H, W]"""
    _check_args(Is, Ps, raft_model, window, iters)
    N, C, H, W = Ps.shape
    dev = Is.device if Is.is_cuda else (Ps.device if Ps.is_cuda else next(raft_model.parameters()).device)
    if dev.type != "cuda":
        raise ValueError("smooth_parsing_maps: the RAFT model (or Is / Ps) must be on a CUDA device")
    parse = torch.empty((N, C, H // 2, W // 2), device=Ps.device, dtype=torch.float32)
    sm = ParsingSmoother(raft_model, window, iters)
    sm.flow_sink = flow_sink
    with torch.no_grad():
        for f in range(N):
            for r in sm.push(Is[f].to(dev), Ps[f].to(dev)):
                parse[r.index].copy_(r.down())
        for r in sm.finish():
            parse[r.index].copy_(r.down())
    return parse
