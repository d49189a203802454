"""Times segmented smoothed video (DESIGN.md section 14): 400x400 uint8 frames (smoothing at 800x800), window 5, 20 iterations, batch 4,
bf16x3, det_state_dict weights (VToonify-D, BiSeNet, RAFT).  The card's name and power limit are read in the same run; one JSON line on
stdout (rank 0).

Halo overhead (one GPU, the default), arms alternated round by round:
  * ``unsegmented``: ``FramePipeline(..., smoothing=(raft, 5, 20)).run`` on uint8 batches, ms per interior frame as
    (T(N) - T(N - K)) / K over whole clips, as tools/smooth_video_bench.py;
  * ``segment_L`` for L in ``--lengths``: ``FramePipeline.smooth_segment`` on an interior segment of ``segment_plan(3 L, 5, L)`` (its
    L outputs with a halo of 5 frames on each side), ms per output as T / L.
A host clock around work that ends in a device synchronise.

    python tools/smooth_sharded_bench.py [--frames 16] [--delta 8] [--lengths 8 16 32] [--rounds 2]

Sharded (``--sharded``, one process per GPU under ``torchrun --nproc-per-node N``; without torchrun, one rank on this GPU):
``ShardedSmoothedVideo`` over a ``--frames``-frame clip in segments of ``--length`` outputs, frames read from host memory and written
back to pinned host memory on rank 0.  Frames per second on rank 0 after a warm-up clip, and rank 0's peak device memory above the
models and peak host RSS above the run's start.

    torchrun --nproc-per-node 8 tools/smooth_sharded_bench.py --sharded [--frames 256] [--length 16]
"""
import argparse
import json
import os
import socket
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from smooth_video_bench import RssPeak, card, clip  # noqa: E402
from tests.golden.make_golden_raft import raft_args  # noqa: E402
from vtoonify_b200 import set_precision  # noqa: E402
from vtoonify_b200 import smooth_parsing as S  # noqa: E402
from vtoonify_b200.bisenet import BiSeNet  # noqa: E402
from vtoonify_b200.frame_loop import FramePipeline, ShardedSmoothedVideo  # noqa: E402
from vtoonify_b200.raft import RAFT  # noqa: E402
from vtoonify_b200.vtoonify import VToonify  # noqa: E402
from vtoonify_b200.weights import det_inputs, det_state_dict  # noqa: E402


def pipeline(dev, window, iters):
    torch.manual_seed(0)
    with torch.no_grad():
        model = VToonify(backbone="dualstylegan").eval()
        model.load_state_dict(det_state_dict(model, seed=0), strict=True)
        parser = BiSeNet(19).eval()
        parser.load_state_dict(det_state_dict(parser, seed=21), strict=True)
        raft = RAFT(raft_args()).eval()
        raft.load_state_dict(det_state_dict(raft, seed=0), strict=True)
    for m in (model, parser, raft):
        m.requires_grad_(False)
        m.to(dev)
    set_precision("bf16x3")
    style = det_inputs(1, 32, 32, seed=5)[1]
    return FramePipeline(model, style, d_s=0.5, device=dev, parsing_net=parser, smoothing=(raft, window, iters))


def halo_overhead(args):
    dev = torch.device("cuda")
    pipe = pipeline(dev, args.window, args.iters)
    N, B, w = args.frames, args.batch, args.window
    lengths = (N - args.delta, N)
    frames = clip(max(N, 3 * max(args.lengths)), args.size, args.size)
    frames_dev = frames.to(dev)

    def unsegmented(n):
        list(pipe.run([frames[i:min(i + B, n)].pin_memory() for i in range(0, n, B)]))

    def segment(L):
        seg = S.segment_plan(3 * L, w, L)[1]
        assert not seg.finish and seg.a - seg.lo == w and seg.hi - seg.b == w
        pipe.smooth_segment(frames_dev[seg.lo:seg.hi], seg, B)

    arms = {f"unsegmented_{n}": (unsegmented, n) for n in lengths}
    arms.update({f"segment_{L}": (segment, L) for L in args.lengths})
    times = {a: [] for a in arms}
    for f, n in arms.values():                                # warm-up
        f(min(n, lengths[0]) if f is unsegmented else n)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for a, (f, n) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f(n)
            torch.cuda.synchronize()
            times[a].append((time.perf_counter() - t0) * 1e3)
    K = lengths[1] - lengths[0]
    un = [(t1 - t0) / K for t0, t1 in zip(times[f"unsegmented_{lengths[0]}"], times[f"unsegmented_{N}"])]
    per = {"unsegmented": round(statistics.median(un), 2)}
    spread = {"unsegmented": [round(min(un), 2), round(max(un), 2)]}
    for L in args.lengths:
        v = [t / L for t in times[f"segment_{L}"]]
        per[f"segment_{L}"] = round(statistics.median(v), 2)
        spread[f"segment_{L}"] = [round(min(v), 2), round(max(v), 2)]
    overhead = {k: round(v / per["unsegmented"] - 1, 4) for k, v in per.items() if k != "unsegmented"}
    return {"workload": f"{args.size}x{args.size} uint8 frames, smoothing at {2 * args.size}x{2 * args.size}, window {w}, "
                        f"{args.iters} iterations, batch {B}, bf16x3; unsegmented from {N}- and {lengths[0]}-frame clips",
            "card": card(), "gpu": torch.cuda.get_device_properties(0).name, "rounds": args.rounds,
            "ms_per_interior_frame": per, "ms_per_interior_frame_spread": spread, "halo_overhead": overhead}


def sharded(args):
    if "RANK" not in os.environ:                              # one rank on this GPU
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        os.environ.update(RANK="0", LOCAL_RANK="0", WORLD_SIZE="1", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    torch.set_grad_enabled(False)
    pipe = pipeline(dev, args.window, args.iters)
    N, L, Sz = args.frames, args.length, args.size
    frames = clip(N, Sz, Sz) if rank == 0 else None
    host = [torch.empty((L, 4 * Sz, 4 * Sz, 3), dtype=torch.uint8).pin_memory() for _ in range(2)] if rank == 0 else None
    d2h = torch.cuda.Stream(dev)
    done = [None, None]

    def sink(i, buf, ready):                                  # a D2H copy per segment into two alternating pinned buffers
        k = (i // L) % 2
        if done[k] is not None:
            done[k].synchronize()
        with torch.cuda.stream(d2h):
            ready()
            host[k][:buf.shape[0]].copy_(buf, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(d2h)
        done[k] = ev
        return ev

    def run(n):
        drv = ShardedSmoothedVideo(pipe, n, L, (Sz, Sz), args.batch, dev)
        if rank == 0:
            drv.run((frames[f] for f in range(n)), sink)
        else:
            drv.run()
        torch.cuda.synchronize()
        dist.barrier()

    run(min(N, world * L))                                    # warm-up: one round
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with RssPeak() as rss:
        t0 = time.perf_counter()
        run(N)
        t = time.perf_counter() - t0
    res = None
    if rank == 0:
        res = {"workload": f"{N}-frame {Sz}x{Sz} uint8 clip, smoothing at {2 * Sz}x{2 * Sz}, window {args.window}, {args.iters} "
                           f"iterations, batch {args.batch}, segments of {L}, bf16x3",
               "card": card(), "gpu": torch.cuda.get_device_properties(dev).name, "world": world,
               "seconds": round(t, 2), "frames_per_s": round(N / t, 3), "frames_per_s_per_gpu": round(N / t / world, 3),
               "rank0_peak_device_gb_above_models": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3),
               "rank0_peak_host_rss_gb_above_start": round(rss.above / 2 ** 30, 3)}
    dist.destroy_process_group()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sharded", action="store_true")
    ap.add_argument("--frames", type=int, default=None, help="halo: the longer unsegmented clip (16); sharded: the clip (64)")
    ap.add_argument("--delta", type=int, default=8)
    ap.add_argument("--lengths", type=int, nargs="+", default=[8, 16, 32])
    ap.add_argument("--length", type=int, default=16)
    ap.add_argument("--size", type=int, default=400)
    ap.add_argument("--window", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("smooth_sharded_bench.py needs a CUDA device")
    if args.frames is None:
        args.frames = 64 if args.sharded else 16
    res = sharded(args) if args.sharded else halo_overhead(args)
    if res is not None:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
