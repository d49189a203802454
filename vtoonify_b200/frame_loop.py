"""Frame loop (the hot loop of style_transfer.py:99-183) for batches of frames.

Reference behaviour per batch: stack frames -> BiSeNet parsing of the 2x up-sampled frames -> ``inputs = cat(x, x_p/16)``
-> ``y = vtoonify(inputs, s_w.repeat(B,1,1), d_s)`` -> ``clamp(-1,1)`` -> per frame ``tensor2cv2(y[k].cpu())``
(style_transfer.py:160-179).  There the H2D copy is pageable and per-frame, the D2H is a blocking fp32 ``.cpu()`` per
frame and nothing overlaps.

Here a :class:`FramePipeline` owns pinned staging buffers and two side streams: batch i+1's host->device copy and
batch i-1's device->host copy overlap batch i's synthesis; ``ToTensor + Normalize``, the face parsing (``parsing_net``)
and the clamp + uint8 + RGB->BGR conversion (``util.tensor2cv2``) run on the device, so a frame crosses PCIe as uint8
in both directions (1.8 MB in / 28 MB out per 576x1024 frame instead of 52 MB / 113 MB of fp32).

Multi-GPU: frames are independent units (SURVEY.md §8e), so ranks take round-robin shards of the frame batches with no
collective inside the forward.  :class:`ShardedFrameLoop` implements the reference's single-decoder layout: rank 0 holds
the clip, every round it scatters one input batch per rank and gathers the uint8 frames back, over ``torch.distributed``
(NCCL on NVLink for CUDA tensors, gloo in the CPU tests), overlapped with the synthesis of the neighbouring rounds.
:func:`scatter_batches` / :func:`gather_frames` are the same collectives in their simple blocking form.
:class:`ShardedSmoothedVideo` runs smoothed video the same way, one segment of output frames with its halo of neighbouring
frames per rank (DESIGN.md §14).
"""
import collections
import contextlib
from typing import Callable, Iterable, Iterator, List, Optional, Sequence

import torch
import torch.distributed as dist

from . import ops
from . import smooth_parsing


def shard_indices(num_batches: int, rank: int, world: int) -> List[int]:
    """Round-robin ownership of frame batches: batch i belongs to rank i % world (BASELINE.json configs[3])."""
    return list(range(rank, num_batches, world))


def merge_order(num_batches: int, world: int) -> List[tuple]:
    """(rank, local_index) of every global batch, in output order."""
    return [(i % world, i // world) for i in range(num_batches)]


class FramePipeline:
    """``run(batches)`` yields one uint8 ``[B, 4H, 4W, 3]`` (BGR, like cv2 frames) host tensor per input batch.

    ``batches``: iterable of host tensors (pinned for real overlap), each one of
      * fp32 ``[B, 22, H, W]`` — the ``inputs`` of style_transfer.py:174;
      * a tuple ``(frames_u8 [B,H,W,3] RGB, parsing [B,19,H,W] fp32)`` — parsing computed elsewhere;
      * uint8 ``[B, H, W, 3]`` RGB frames alone — needs ``parsing_net`` (a :class:`vtoonify_b200.bisenet.BiSeNet`):
        the parsing maps are computed on the device (style_transfer.py:171-174); with ``prefilter`` the frames are the
        clip's full-resolution frames and the blur / resize / crop of style_transfer.py:151-156 also runs on the device.

    Temporally smoothed parsing (``smoothing=(raft_model, window, iters)``, smooth_parsing_map.py followed by
    ``style_transfer.py --parsing_map_path`` in one pass): batches are uint8 frames (``prefilter`` allowed) and ``parsing_net`` is
    required.  Per input batch the frames are up-sampled 2x with RAFT's stem input (``smooth_parsing.frame_prep``), BiSeNet gives
    the 2x logits (the script's ``parsingpredictor(2 * Is)``) and every frame is pushed into a ``smooth_parsing.ParsingSmoother``; each
    output it releases is fused, down-sampled and scaled by 1/16 straight into its frame's network input
    (``smooth_parsing.parsing_fuse_down``).  Output batch j holds the frames of input batch j: the first outputs wait ``window``
    frames and the end of the input flushes the rest.  Device memory holds the window, not the clip; no intermediate file is
    written.  H and W (after ``prefilter``) must be multiples of 8 and at least 64; ``graph`` is not supported (the launches of a
    batch depend on where it sits in the clip).

    Buffer ownership.  With ``copy=True`` (default) every yielded tensor is a fresh host tensor owned by the caller.
    With ``copy=False`` the yielded tensor is a *borrowed* view of one of ``ring`` pinned staging buffers: it stays valid
    until ``ring - 1`` further batches have been yielded (``ring=3``: the previous result is still intact while the
    current one is being consumed) — the zero-copy mode for a consumer that encodes / writes each batch before asking for
    the next one.
    """

    def __init__(self, model, style: torch.Tensor, d_s: Optional[float] = 0.5, device: Optional[torch.device] = None,
                 output: str = "u8", parsing_net=None, ring: int = 3, copy: bool = True, graph: bool = False,
                 prefilter=None, smoothing=None):
        if ring < 2:
            raise ValueError("FramePipeline: ring must be >= 2 (one buffer is being filled while one is being consumed)")
        if smoothing is not None:
            if graph:
                raise ValueError("FramePipeline: graph=True is not supported with smoothing (a batch's launches depend on its place "
                                 "in the clip)")
            if parsing_net is None:
                raise ValueError("FramePipeline: smoothing needs parsing_net (the 2x parsing logits are computed on the device)")
            raft_model, window, iters = smoothing
            with torch.no_grad():           # the run is forward only
                smooth_parsing._check_model_window("FramePipeline", raft_model, window, iters)
            smoothing = (raft_model, int(window), int(iters))
        self.smoothing = smoothing
        self.model = model
        self.device = device or next(model.parameters()).device
        self.style = style.to(self.device)
        self.d_s = d_s
        self.output = output
        self.parsing_net = parsing_net
        self.ring = ring
        self.copy = copy
        # (n_blur, (w, h), (top, bottom, left, right)): the reference's per-frame CPU pre-processing of high-resolution clips
        # (style_transfer.py:151-156: sepFilter2D x n_blur, resize, crop) applied on the device to uploaded uint8 frames
        self.prefilter = prefilter
        self.graph = graph          # replay one captured CUDA graph per input geometry instead of ~130 launches per batch
        self._graphs = {}
        self._style_b = {}
        self.h2d = torch.cuda.Stream(self.device)
        self.d2h = torch.cuda.Stream(self.device)
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        self._host_out = {}

    # ---- device-side assembly of the network input -------------------------------------------------
    def assemble(self, item_dev):
        """device tensors of one batch (same forms as ``run``'s items) -> ``inputs`` fp32 ``[B,22,H,W]``."""
        if isinstance(item_dev, (tuple, list)):
            frames, parsing = item_dev
            B, H, W, _ = frames.shape
            x = torch.empty((B, 22, H, W), device=self.device, dtype=torch.float32)
            ops.frames_u8_to_f32(frames, out=x)                       # channels 0..2: ToTensor + Normalize(0.5, 0.5)
            for b in range(B):
                ops.axpby(parsing[b], None, 1.0 / 16.0, out=x[b, 3:])  # style_transfer.py:174 (x[b, 3:] is contiguous)
            return x
        if item_dev.dtype == torch.uint8:
            if self.prefilter is not None:
                n_blur, size, crop = self.prefilter
                item_dev = ops.frame_prefilter_resize(item_dev, n_blur, size, crop)
            if self.parsing_net is None:
                raise ValueError("FramePipeline: uint8 frames need parsing_net (face parsing on the device)")
            B, H, W, _ = item_dev.shape
            x = torch.empty((B, 22, H, W), device=self.device, dtype=torch.float32)
            ops.frames_u8_to_f32(item_dev, out=x)
            rgb = ops.frames_u8_to_f32(item_dev)                      # dense planar copy for the parsing network
            self.parsing_net.parsing_for_frames(rgb, scale=1.0 / 16.0, out=x[:, 3:])
            return x
        return item_dev

    def _style_for(self, B):
        # the SAME expanded (stride-0) tensor object on every call: the model recognises a style it has already prepared by
        # identity, and a stride-0 batch as "one style for all frames" without looking at the data
        st = self._style_b.get(B)
        if st is None:
            st = self.style.expand(B, -1, -1) if self.style.shape[0] == 1 else self.style
            self._style_b[B] = st
        return st

    def synthesize(self, x):
        """``inputs`` -> device uint8 BGR frames (or clamped fp32 images when ``output != 'u8'``)"""
        y = self.model(x, self._style_for(x.shape[0]), d_s=self.d_s)
        return ops.f32_to_frames_u8(y, swap_rb=True) if self.output == "u8" else y.clamp(-1, 1)

    def process(self, item_dev):
        """device item (any of the input forms) -> device result; with ``graph=True`` through a CUDA graph captured once per
        input geometry (static input / output buffers; the result is copied out so that the next replay may start while the
        previous result is still being downloaded)"""
        if not self.graph:
            return self.synthesize(self.assemble(item_dev))
        items = item_dev if isinstance(item_dev, (tuple, list)) else (item_dev,)
        key = tuple((tuple(t.shape), t.dtype) for t in items)
        g = self._graphs.get(key)
        if g is None:
            static_in = tuple(torch.empty_like(t) for t in items)
            for a, b in zip(static_in, items):
                a.copy_(b)
            arg = static_in if isinstance(item_dev, (tuple, list)) else static_in[0]
            side = torch.cuda.Stream(self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):
                for _ in range(2):                                   # warm-up outside the capture: weight caches, attributes
                    self.synthesize(self.assemble(arg))
            torch.cuda.current_stream(self.device).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_out = self.synthesize(self.assemble(arg))
            g = (graph, static_in, static_out)
            self._graphs[key] = g
        graph, static_in, static_out = g
        for a, b in zip(static_in, items):
            a.copy_(b, non_blocking=True)
        graph.replay()
        return static_out.clone()

    def _upload(self, item):
        """Host -> device on the h2d stream; returns (device item, ready_event)."""
        with torch.cuda.stream(self.h2d):
            if isinstance(item, (tuple, list)):
                dev = tuple(t.to(self.device, non_blocking=True) for t in item)
                self.h2d_bytes += sum(t.numel() * t.element_size() for t in item)
            else:
                dev = item.to(self.device, non_blocking=True)
                self.h2d_bytes += item.numel() * item.element_size()
            ev = torch.cuda.Event()
            ev.record(self.h2d)
        return dev, ev

    def _host_buffer(self, shape, dtype, slot):
        key = (tuple(shape), dtype, slot)
        if key not in self._host_out:
            self._host_out[key] = torch.empty(shape, dtype=dtype, pin_memory=True)
        return self._host_out[key]

    def run(self, batches: Iterable) -> Iterator[torch.Tensor]:
        compute = self._compute_smoothed(batches) if self.smoothing is not None else self._compute(batches)
        main = torch.cuda.current_stream(self.device)
        pending = None  # (host_tensor, event) of the previous batch's download
        slot = 0
        with torch.no_grad():
            for out_dev in compute:
                done = torch.cuda.Event()
                done.record(main)
                host = self._host_buffer(out_dev.shape, out_dev.dtype, slot)
                slot = (slot + 1) % self.ring
                with torch.cuda.stream(self.d2h):
                    self.d2h.wait_event(done)
                    host.copy_(out_dev, non_blocking=True)
                    out_dev.record_stream(self.d2h)
                    dl = torch.cuda.Event()
                    dl.record(self.d2h)
                self.d2h_bytes += out_dev.numel() * out_dev.element_size()
                if pending is not None:
                    pending[1].synchronize()
                    yield pending[0].clone() if self.copy else pending[0]
                pending = (host, dl)
            if pending is not None:
                pending[1].synchronize()
                yield pending[0].clone() if self.copy else pending[0]

    def _uploaded(self, batches: Iterable):
        """the device items of ``batches`` in order, each made ready on the current stream; the next batch's upload is issued before
        the current one is handed out, so it overlaps the current batch's compute"""
        main = torch.cuda.current_stream(self.device)
        it = iter(batches)
        nxt = next(it, None)
        up = self._upload(nxt) if nxt is not None else None
        while up is not None:
            x, ev = up
            nxt = next(it, None)
            up = self._upload(nxt) if nxt is not None else None   # prefetch the next batch while this one computes
            main.wait_event(ev)
            for t in (x if isinstance(x, tuple) else (x,)):
                t.record_stream(main)
            yield x

    def _compute(self, batches: Iterable):
        """one device result per input batch"""
        for x in self._uploaded(batches):
            yield self.process(x)

    def _smoothing_frames(self, item):
        """a device item of a smoothed run -> its uint8 frames after ``prefilter``, with the checks of the smoothed route"""
        if isinstance(item, (tuple, list)) or item.dtype != torch.uint8 or item.dim() != 4 or item.shape[3] != 3:
            raise ValueError("FramePipeline: with smoothing, batches must be uint8 [B, H, W, 3] RGB frames")
        frames = item
        if self.prefilter is not None:
            n_blur, size, crop = self.prefilter
            frames = ops.frame_prefilter_resize(frames, n_blur, size, crop)
        _, H, W, _ = frames.shape
        if H % 8 or W % 8 or H < 64 or W < 64:
            raise ValueError(f"FramePipeline: smoothing needs frames whose H and W are multiples of 8 and at least 64 (RAFT runs "
                             f"at 2H x 2W); got {H}x{W}")
        return frames

    def _compute_smoothed(self, batches: Iterable):
        """one device result per input batch through the streaming smoother"""
        return self._smoothed((self._smoothing_frames(item) for item in self._uploaded(batches)), 0, None, True)

    def _smoothed(self, batches, first, outputs, finish):
        """the streaming smoother between the face parsing and the synthesis.  ``batches`` yields uint8 frames after ``prefilter`` in
        clip order from frame ``first``.  A batch whose first frame is in ``outputs`` (a range; None: every frame) is synthesised: its
        network input is allocated (with its RGB channels) when it arrives, its parsing channels are filled as the smoother releases
        its frames, and it is yielded once all of them are in.  The other batches (halo frames) are prepped, parsed and pushed only,
        and the outputs outside ``outputs`` are not read.  ``finish`` ends the stream with ``finish()``."""
        raft_model, window, iters = self.smoothing
        sm = smooth_parsing.ParsingSmoother(raft_model, window, iters, first)
        net = self.parsing_net
        waiting = collections.deque()       # [x [B, 22, H, W], index of its first frame, frames filled] in clip order
        n_in = first

        def fill(r):
            if outputs is not None and r.index not in outputs:
                return
            for item in waiting:
                k = r.index - item[1]
                if 0 <= k < item[0].shape[0]:
                    r.fuse_down(item[0][k, 3:], 1.0 / 16.0)      # style_transfer.py:174's x_p / 16
                    item[2] += 1
                    return
            raise AssertionError(f"smoothed frame {r.index} has no waiting batch")

        for frames in batches:
            B, H, W, _ = frames.shape
            if outputs is None or n_in in outputs:
                x = torch.empty((B, 22, H, W), device=self.device, dtype=torch.float32)
                ops.frames_u8_to_f32(frames, out=x)                    # channels 0..2: ToTensor + Normalize(0.5, 0.5)
                waiting.append([x, n_in, 0])
            n_in += B
            Is, stem = smooth_parsing.frame_prep(frames)
            fuse, _, _ = net._features(ops.frame_s2d(ops.frames_u8_to_f32(frames), upsample2=True))
            Ps = ops.logits_readout(net.conv_out.logits_nhwc(fuse), net.n_classes, 2 * H, 2 * W, step=1)   # parsingpredictor(2*Is)[0]
            for b in range(B):
                for r in sm.push(Is[b], Ps[b], stem[b:b + 1]):
                    fill(r)
            del Is, stem, Ps
            while waiting and waiting[0][2] == waiting[0][0].shape[0]:
                yield self.synthesize(waiting.popleft()[0])
        if n_in == first:
            return
        if finish:
            for r in sm.finish():
                fill(r)
        while waiting:
            x, _, filled = waiting.popleft()
            assert filled == x.shape[0]
            yield self.synthesize(x)

    def smooth_segment(self, frames_dev: torch.Tensor, seg, batch: int) -> torch.Tensor:
        """One segment of a smoothed clip (``seg`` from ``smooth_parsing.segment_plan(N, window, length)``): ``frames_dev`` holds the
        clip's uint8 RGB frames ``[seg.lo, seg.hi)`` on the device, ``[seg.hi - seg.lo, H, W, 3]`` (``prefilter`` applies as in
        ``run``).  Returns the device uint8 BGR frames of outputs ``[seg.a, seg.b)``, ``[seg.b - seg.a, 4H, 4W, 3]``: the same bytes
        as those frames of ``run`` over the whole clip in batches of ``batch``, so ``seg.a`` must be a multiple of ``batch`` (a
        ``length`` that is).  The halo frames are prepped, parsed and pushed, not synthesised (DESIGN.md section 14)."""
        if self.smoothing is None:
            raise ValueError("FramePipeline.smooth_segment: the pipeline has no smoothing")
        window = self.smoothing[1]
        if not isinstance(seg, smooth_parsing.Segment):
            raise ValueError("FramePipeline.smooth_segment: seg must be a smooth_parsing.Segment (from segment_plan)")
        a, b, lo, hi, finish = seg
        # the plan's halos: window frames before a (fewer at the clip's head), window after b or, with finish, up to the clip's end
        if not (0 <= lo == max(0, a - window) and a < b and (b <= hi < b + window if finish else hi == b + window)):
            raise ValueError(f"FramePipeline.smooth_segment: {seg} is not a segment of a plan with window {window}")
        if int(batch) != batch or batch < 1 or a % batch:
            raise ValueError(f"FramePipeline.smooth_segment: batch must be a positive integer that divides the first output {a} "
                             f"(got {batch})")
        if (not isinstance(frames_dev, torch.Tensor) or not frames_dev.is_cuda or frames_dev.dtype != torch.uint8
                or frames_dev.dim() != 4 or frames_dev.shape[0] != hi - lo or frames_dev.shape[3] != 3):
            raise ValueError(f"FramePipeline.smooth_segment: frames must be a CUDA uint8 [{hi - lo}, H, W, 3] tensor (the segment's "
                             f"frames {lo}..{hi - 1})")
        # batches of `batch` frames from a (those of run over the whole clip), the halos cut likewise
        cuts = sorted({*range(lo, a, int(batch)), *range(a, b, int(batch)), *range(b, hi, int(batch)), hi})
        batches = (self._smoothing_frames(frames_dev[s - lo:e - lo]) for s, e in zip(cuts[:-1], cuts[1:]))
        with torch.no_grad():
            outs = list(self._smoothed(batches, lo, range(a, b), finish))
        return outs[0] if len(outs) == 1 else torch.cat(outs)


# ----------------------------------------------------------------------------------------------
# rank-0 ingest / egress over torch.distributed (NCCL over NVLink on the GPU box, gloo in CPU tests)
# ----------------------------------------------------------------------------------------------
def scatter_batches(batches: Optional[Sequence[torch.Tensor]], num_batches: int, example_shape, dtype, device,
                    src: int = 0, group=None) -> List[torch.Tensor]:
    """Rank ``src`` holds all ``num_batches`` input batches; every rank returns its round-robin shard.
    One ``dist.scatter`` per round of ``world`` batches (the only input-side collective of the path)."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    mine = []
    rounds = (num_batches + world - 1) // world
    for r in range(rounds):
        recv = torch.empty(example_shape, dtype=dtype, device=device)
        if rank == src:
            chunk = []
            for k in range(world):
                i = r * world + k
                chunk.append(batches[i].to(device) if i < num_batches else torch.zeros(example_shape, dtype=dtype, device=device))
            dist.scatter(recv, chunk, src=src, group=group)
        else:
            dist.scatter(recv, None, src=src, group=group)
        if r * world + rank < num_batches:
            mine.append(recv)
    return mine


def gather_frames(local_outputs: Sequence[torch.Tensor], num_batches: int, example_shape, dtype, device, dst: int = 0,
                  group=None) -> Optional[List[torch.Tensor]]:
    """Inverse of :func:`scatter_batches` for the uint8 output frames: returns the ordered list on ``dst``."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    rounds = (num_batches + world - 1) // world
    ordered = [] if rank == dst else None
    for r in range(rounds):
        have = r * world + rank < num_batches
        send = local_outputs[r].to(device) if have else torch.zeros(example_shape, dtype=dtype, device=device)
        if rank == dst:
            bufs = [torch.empty(example_shape, dtype=dtype, device=device) for _ in range(world)]
            dist.gather(send, bufs, dst=dst, group=group)
            for k in range(world):
                if r * world + k < num_batches:
                    ordered.append(bufs[k])
        else:
            dist.gather(send, None, dst=dst, group=group)
    return ordered


class _Pending:
    """An asynchronous collective: ``wait()`` orders the CURRENT stream (CUDA) / the caller (CPU) behind the communication
    work and behind everything the issuing stream had enqueued when the collective was issued (the local piece)."""

    def __init__(self, work, event, device=None):
        self.work, self.event, self.device = work, event, device

    def wait(self):
        self.work.wait()
        if self.event is not None:
            torch.cuda.current_stream(self.device).wait_event(self.event)


class ShardedFrameLoop:
    """The reference's single-decoder frame loop over ``world`` GPUs: rank 0 owns the clip (input batches in, frames out),
    every round ``r`` it scatters batch ``r*world + k`` to rank ``k`` and gathers the ``world`` result batches back.

    Per round and rank:  [rank 0: stage the round's inputs on its device] -> ``dist.scatter`` -> ``fn(inputs)`` ->
    ``dist.gather`` of the results to rank 0 -> [rank 0: hand the ordered results to ``sink``].  The collectives are issued
    asynchronously and double-buffered: the scatter of round r+1 is in flight while round r is synthesised, the gather of
    round r while round r+1 is; ``fn`` is the only thing on the compute stream.

    ``fn``: device batch -> device result (e.g. ``lambda t: pipe.synthesize(pipe.assemble(t))``); with ``indexed=True``,
    ``fn(batch, i)`` also gets the global index ``i`` of the batch.
    ``stage``: rank 0 only, ``stage(i) -> device tensor`` of global batch ``i`` (from host memory: an H2D copy; from device
    memory: a lookup).  ``sink``: rank 0 only, ``sink(i, result_dev, ready)`` — called in order for every global batch once its
    gather has been *issued*; ``ready()`` makes the current stream wait for the data (CUDA) / blocks (CPU).  ``result_dev`` is
    a borrowed gather buffer, reused two rounds later: a sink that reads it asynchronously (a D2H copy on its own stream)
    returns a ``torch.cuda.Event`` recorded after its read and the loop orders the buffer's next use behind it.
    Works on CPU tensors with the gloo backend (tests) and on CUDA tensors with NCCL.
    """

    def __init__(self, fn: Callable, in_shape, in_dtype, out_shape, out_dtype, device, group=None, src: int = 0,
                 indexed: bool = False):
        self.fn, self.group, self.src, self.indexed = fn, group, src, indexed
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        self.in_shape, self.in_dtype, self.out_shape, self.out_dtype = tuple(in_shape), in_dtype, tuple(out_shape), out_dtype
        n = 2
        self._recv = [torch.empty(self.in_shape, dtype=in_dtype, device=self.device) for _ in range(n)]
        self._send = [torch.empty(self.out_shape, dtype=out_dtype, device=self.device) for _ in range(n)]
        self._gath = ([[torch.empty(self.out_shape, dtype=out_dtype, device=self.device) for _ in range(self.world)]
                       for _ in range(n)] if self.rank == src else None)
        self._zero_in = torch.zeros(self.in_shape, dtype=in_dtype, device=self.device) if self.rank == src else None
        self.side = torch.cuda.Stream(self.device) if self.cuda else None
        self.scatter_bytes = 0
        self.gather_bytes = 0

    def _side(self):
        return torch.cuda.stream(self.side) if self.cuda else contextlib.nullcontext()

    def _event_on(self, stream):
        if not self.cuda:
            return None
        ev = torch.cuda.Event()
        ev.record(stream)
        return ev

    def _issue_scatter(self, r, num_batches, stage):
        """stage + scatter round r on the side stream; returns the Work handle (None past the last round)."""
        if r * self.world >= num_batches:
            return None
        recv = self._recv[r % 2]
        with self._side():
            if self.rank == self.src:
                chunk = []
                for k in range(self.world):
                    i = r * self.world + k
                    chunk.append(stage(i) if i < num_batches else self._zero_in)
                work = dist.scatter(recv, chunk, src=self.src, group=self.group, async_op=True)
                self._keep = chunk                      # keep the staged tensors alive until the next round's scatter
                self.scatter_bytes += sum(c.numel() * c.element_size() for c in chunk[1:])
            else:
                work = dist.scatter(recv, None, src=self.src, group=self.group, async_op=True)
            # a rank's OWN piece of a scatter / gather is a plain device copy that the backend may enqueue on the issuing stream
            # instead of its communication stream: consumers wait for the Work AND for this event
            ev = None
            if self.cuda:
                ev = torch.cuda.Event()
                ev.record(self.side)
        return _Pending(work, ev, self.device if self.cuda else None)

    def run(self, num_batches: int, stage: Optional[Callable] = None, sink: Optional[Callable] = None) -> int:
        """Process ``num_batches`` global batches; returns the number of batches this rank synthesised."""
        rounds = (num_batches + self.world - 1) // self.world
        mine = 0
        pend_scatter = self._issue_scatter(0, num_batches, stage)
        pend_gather = [None, None]                      # Work of the gather that last used slot s
        sink_done = [[], []]                            # events after which slot s's gather buffers may be overwritten
        cur = torch.cuda.current_stream(self.device) if self.cuda else None
        for r in range(rounds):
            s = r % 2
            pend_scatter.wait()                         # compute stream waits for this round's inputs
            if self.cuda and r + 1 < rounds:
                self.side.wait_stream(cur)              # recv[(r+1)%2] was read by round r-1's fn: order the next scatter after it
            nxt = self._issue_scatter(r + 1, num_batches, stage)
            have = r * self.world + self.rank < num_batches
            if pend_gather[s] is not None:
                pend_gather[s].wait()                   # the gather of round r-2 has consumed send[s] / filled gath[s]
            if have:
                out = self.fn(self._recv[s], r * self.world + self.rank) if self.indexed else self.fn(self._recv[s])
                self._send[s].copy_(out)
                mine += 1
            else:
                self._send[s].zero_()
            if self.rank == self.src:
                for ev in sink_done[s]:
                    cur.wait_event(ev)                  # round r-2's results have left these gather buffers
                sink_done[s] = []
                work = dist.gather(self._send[s], self._gath[s], dst=self.src, group=self.group, async_op=True)
                work = _Pending(work, self._event_on(cur), self.device if self.cuda else None)
                self.gather_bytes += (self.world - 1) * self._send[s].numel() * self._send[s].element_size()
                if sink is not None:
                    for k in range(self.world):
                        i = r * self.world + k
                        if i < num_batches:
                            tok = sink(i, self._gath[s][k], work.wait)
                            if tok is not None and self.cuda:
                                sink_done[s].append(tok)
            else:
                work = _Pending(dist.gather(self._send[s], None, dst=self.src, group=self.group, async_op=True), self._event_on(cur),
                                self.device if self.cuda else None)
            pend_gather[s] = work
            pend_scatter = nxt
        for w in pend_gather:
            if w is not None:
                w.wait()
        return mine


class ShardedSmoothedVideo:
    """Smoothed video over ``world`` GPUs, one process per GPU: the clip's N outputs are cut into segments of ``length`` outputs
    (``smooth_parsing.segment_plan``), and segment ``r * world + k`` is smoothed and synthesised on rank k by
    ``pipe.smooth_segment(frames, seg, batch)`` (a ``FramePipeline`` with ``smoothing``), which gives the bytes of the one-GPU
    ``pipe.run`` over the clip in batches of ``batch``.  Built on :class:`ShardedFrameLoop`: every round, rank 0 scatters one
    zero-padded ``[length + 2 * window, H, W, 3]`` uint8 segment (its frames with their halos) per rank and gathers the
    ``[length, 4h, 4w, 3]`` uint8 BGR outputs back (h, w: the frame size after ``prefilter``).

    ``run(frames, sink)`` on rank 0, ``run()`` on the others.  ``frames`` is an iterable of the clip's N uint8 RGB frames, each item
    one ``[H, W, 3]`` frame or a batch ``[n, H, W, 3]``, read once and in order; rank 0 keeps the 2 * window frames the next
    segment's halo shares with the last one, so its host and device memory are bounded by ``world``, ``length`` and the frame size,
    whatever N (DESIGN.md section 14).  ``sink(i, frames, ready)`` is called in clip order, once per segment, with the segment's
    first output index ``i`` and its device frames ``[b - a, 4h, 4w, 3]``, with the contract of :class:`ShardedFrameLoop`'s sink
    (``ready()`` before reading; the buffer is reused two rounds later unless the sink returns an event)."""

    def __init__(self, pipe, N: int, length: int, frame_shape, batch: int, device, group=None, src: int = 0):
        if pipe.smoothing is None:
            raise ValueError("ShardedSmoothedVideo: the pipeline has no smoothing")
        window = pipe.smoothing[1]
        self.plan = smooth_parsing.segment_plan(N, window, length)
        if int(batch) != batch or batch < 1 or length % batch:
            raise ValueError(f"ShardedSmoothedVideo: length {length} must be a multiple of the batch size (got {batch}), so that "
                             "every batch holds the frames it holds in the one-GPU run")
        if len(frame_shape) != 2 or any(int(s) != s or s < 1 for s in frame_shape):
            raise ValueError(f"ShardedSmoothedVideo: frame_shape must be (H, W) (got {frame_shape})")
        self.pipe, self.N, self.length, self.batch = pipe, int(N), int(length), int(batch)
        self.frame_shape = tuple(int(s) for s in frame_shape)
        H, W = self.frame_shape
        if pipe.prefilter is None:
            h, w = H, W
        else:
            _, (dw, dh), crop = pipe.prefilter
            top, bottom, left, right = (0, dh, 0, dw) if crop is None else crop
            h, w = bottom - top, right - left
        self.loop = ShardedFrameLoop(self._segment, (self.length + 2 * window, H, W, 3), torch.uint8, (self.length, 4 * h, 4 * w, 3),
                                     torch.uint8, device, group=group, src=src, indexed=True)

    def _segment(self, x, i):
        seg = self.plan[i]
        out = self.pipe.smooth_segment(x[:seg.hi - seg.lo], seg, self.batch)
        if out.shape[0] < self.length:                # the clip's last segment
            out = torch.cat([out, out.new_zeros((self.length - out.shape[0],) + tuple(out.shape[1:]))])
        return out

    def run(self, frames: Optional[Iterable] = None, sink: Optional[Callable] = None) -> int:
        """Smooth and synthesise the clip; returns the number of segments this rank computed."""
        loop = self.loop
        if loop.rank != loop.src:
            return loop.run(len(self.plan))
        if frames is None or sink is None:
            raise ValueError("ShardedSmoothedVideo.run: rank 0 needs the clip's frames and a sink")
        reader = _HaloReader(frames, self.N, self.frame_shape)
        plan, cuda = self.plan, loop.cuda

        def stage(i):
            seg = plan[i]
            buf = torch.empty(loop.in_shape, dtype=torch.uint8, pin_memory=cuda)
            n = seg.hi - seg.lo
            buf[n:].zero_()
            for f in range(seg.lo, seg.hi):
                buf[f - seg.lo].copy_(reader.frame(f))
            reader.drop_before(plan[i + 1].lo if i + 1 < len(plan) else self.N)
            return buf.to(loop.device, non_blocking=True)

        def seg_sink(i, buf, ready):
            a, b = plan[i].a, plan[i].b
            return sink(a, buf[:b - a], ready)

        return loop.run(len(plan), stage=stage, sink=seg_sink)


class _HaloReader:
    """rank 0's view of the clip for :class:`ShardedSmoothedVideo`: frames read once, in order, from an iterable of ``[H, W, 3]``
    frames or ``[n, H, W, 3]`` batches; it holds copies of the frames from the oldest one still needed"""

    def __init__(self, frames: Iterable, N: int, frame_shape):
        self.it, self.N, self.shape = iter(frames), N, tuple(frame_shape) + (3,)
        self.kept = collections.deque()              # copies of frames base, base + 1, ...
        self.base = 0
        self.item, self.off = None, 0

    def _read(self):
        f = self.base + len(self.kept)
        while self.item is None or self.off == self.item.shape[0]:
            item = next(self.it, None)
            if item is None:
                raise ValueError(f"ShardedSmoothedVideo: the clip ended after {f} frames; {self.N} were announced")
            item = torch.as_tensor(item)
            if item.dim() == 3:
                item = item[None]
            if item.dtype != torch.uint8 or item.dim() != 4 or tuple(item.shape[1:]) != self.shape:
                raise ValueError(f"ShardedSmoothedVideo: frames must be uint8 {list(self.shape)} or batches [n, "
                                 f"{', '.join(map(str, self.shape))}] (got {item.dtype} {list(item.shape)})")
            if f + item.shape[0] > self.N:
                raise ValueError(f"ShardedSmoothedVideo: the clip has more than the {self.N} frames announced")
            self.item, self.off = item, 0
        self.kept.append(self.item[self.off].clone())
        self.off += 1

    def frame(self, f: int) -> torch.Tensor:
        while self.base + len(self.kept) <= f:
            self._read()
        return self.kept[f - self.base]

    def drop_before(self, f: int):
        while self.kept and self.base < f:
            self.kept.popleft()
            self.base += 1
