"""Times RAFT's two correlation paths (ops.set_option("raft_corr", ...)): the all-pairs ``volume`` and the ``on_demand`` lookup.

Legs (bf16x3, det_state_dict weights, random fnet-sized features; one JSON line on stdout):
  * ``iterate``: ``RAFT._iterate`` (correlation set-up, ``--iters`` updates, test-mode up-sampling) for the smoothing batch at 800x800
    (h, w = 100; 11 pairs), both arms alternated round by round: ms per call (host clock around work that ends in a device
    synchronise), peak device memory above the inputs (torch.cuda.max_memory_allocated), library launches per call, and the largest
    difference of the up-sampled flows between the arms;
  * ``iterate_hd``: the same call on demand at 1152x2048 and 1440x2560 (10 pairs, the 576x1024 and 720x1280 frames' smoothing
    batch); the volume arm gives only its analytic bytes, 4 * pairs * (h*w)^2 * (1 + 1/4 + 1/16 + 1/64);
  * ``pipeline``: ``FramePipeline(..., smoothing=(raft, 5, iters))`` on demand for 576x1024 and 720x1280 uint8 clips, batch 1: ms per
    interior frame as (T(N) - T(N - delta)) / delta over whole clips, and the peak device memory above the models.
The card's name and power limit are read in the same run.

    python tools/raft_ondemand_bench.py [--rounds 3] [--iters 20] [--frames 14] [--delta 4] [--skip-pipeline]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests.golden.make_golden_raft import raft_args  # noqa: E402
from tools.smooth_video_bench import card, clip  # noqa: E402
from vtoonify_b200 import ops, set_precision  # noqa: E402
from vtoonify_b200._lib import launch_count  # noqa: E402
from vtoonify_b200.raft import RAFT  # noqa: E402
from vtoonify_b200.weights import det_inputs, det_state_dict  # noqa: E402

DEV = "cuda"


def volume_bytes(pairs, h, w):
    return 4 * pairs * (h * w) ** 2 * (1 + 1 / 4 + 1 / 16 + 1 / 64)


def inputs(pairs, h, w, seed=0):
    """fmap1 (one map at batch stride 0, as ParsingSmoother passes it on demand), fmap2, net and x of a smoothing batch"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    f1 = torch.randn(1, h, w, 256, device=DEV, generator=g)
    # fmap2: fmap1 shifted by a smooth few-pixel flow plus noise, so the flows are coherent as in a video
    f2 = torch.roll(f1, shifts=(2, -3), dims=(1, 2)).expand(pairs, -1, -1, -1) + 0.3 * torch.randn(pairs, h, w, 256, device=DEV,
                                                                                                  generator=g)
    net = torch.tanh(torch.randn(1, h, w, 128, device=DEV, generator=g))
    x = torch.relu(torch.randn(1, h, w, 256, device=DEV, generator=g))
    return f1, f2.contiguous(), net, x


def run_iterate(raft, mode, pairs, f1, f2, net, x, iters):
    ops.set_option("raft_corr", mode)
    fm1 = f1.expand(pairs, -1, -1, -1)
    if mode == "volume":
        fm1 = fm1.contiguous()
    n, xx = net.expand(pairs, -1, -1, -1).contiguous(), x.expand(pairs, -1, -1, -1).contiguous()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    l0 = launch_count()
    t0 = time.perf_counter()
    with torch.no_grad():
        _, up = raft._iterate(fm1, f2, n, xx, iters)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return ms, torch.cuda.max_memory_allocated() - base, launch_count() - l0, up


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--frames", type=int, default=14)
    ap.add_argument("--delta", type=int, default=4)
    ap.add_argument("--skip-pipeline", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("raft_ondemand_bench.py needs a CUDA device")
    torch.manual_seed(0)
    raft = RAFT(raft_args()).eval()
    raft.load_state_dict(det_state_dict(raft, seed=0), strict=True)
    raft.requires_grad_(False)
    raft.to(DEV)
    set_precision("bf16x3")
    res = {"card": card(), "precision": "bf16x3", "iters": args.iters}

    # 800x800: both arms, alternated
    pairs, h, w = 11, 100, 100
    ins = inputs(pairs, h, w)
    for mode in ("volume", "on_demand"):
        run_iterate(raft, mode, pairs, *ins, 2)          # warm-up: modules, weight caches, allocator
    t = {"volume": [], "on_demand": []}
    out = {}
    for _ in range(args.rounds):
        for mode in ("volume", "on_demand"):
            ms, peak, nl, up = run_iterate(raft, mode, pairs, *ins, args.iters)
            t[mode].append(ms)
            out[mode] = (peak, nl, up)
    res["iterate_800"] = {m: {"ms_per_call": sorted(v)[len(v) // 2], "ms_all": [round(a, 2) for a in v], "peak_gb": out[m][0] / 1e9,
                              "launches": out[m][1]} for m, v in t.items()}
    res["iterate_800"]["pairs"] = pairs
    res["iterate_800"]["volume_analytic_gb"] = volume_bytes(pairs, h, w) / 1e9
    res["iterate_800"]["max_abs_flow_diff"] = float((out["volume"][2] - out["on_demand"][2]).abs().max())
    del ins, out

    # HD: on demand only
    res["iterate_hd"] = {}
    for (H, W) in ((1152, 2048), (1440, 2560)):
        pairs, h, w = 10, H // 8, W // 8
        ins = inputs(pairs, h, w)
        run_iterate(raft, "on_demand", pairs, *ins, 2)
        v = [run_iterate(raft, "on_demand", pairs, *ins, args.iters) for _ in range(args.rounds)]
        res["iterate_hd"][f"{H}x{W}"] = {"pairs": pairs, "ms_per_call": sorted(a[0] for a in v)[len(v) // 2],
                                         "peak_gb": v[-1][1] / 1e9, "launches": v[-1][2],
                                         "volume_analytic_gb": volume_bytes(pairs, h, w) / 1e9}
        del ins, v
    ops.set_option("raft_corr", "volume")
    print(json.dumps(res), flush=True)

    if not args.skip_pipeline:
        from vtoonify_b200.bisenet import BiSeNet
        from vtoonify_b200.frame_loop import FramePipeline
        from vtoonify_b200.vtoonify import VToonify
        with torch.no_grad():
            model = VToonify(backbone="dualstylegan").eval()
            model.load_state_dict(det_state_dict(model, seed=0), strict=True)
            parser = BiSeNet(19).eval()
            parser.load_state_dict(det_state_dict(parser, seed=21), strict=True)
        for m in (model, parser):
            m.requires_grad_(False)
            m.to(DEV)
        style = det_inputs(1, 32, 32, seed=5)[1]
        ops.set_option("raft_corr", "on_demand")
        res["pipeline"] = {}
        for (H, W) in ((576, 1024), (720, 1280)):
            frames = clip(args.frames, H, W)

            def one(n):
                pipe = FramePipeline(model, style, d_s=0.5, parsing_net=parser, smoothing=(raft, 5, args.iters))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for o in pipe.run([frames[i:i + 1].pin_memory() for i in range(n)]):
                    pass
                torch.cuda.synchronize()
                return time.perf_counter() - t0
            one(args.frames - args.delta)                   # warm-up at this size
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            ta, tb = one(args.frames - args.delta), one(args.frames)
            res["pipeline"][f"{H}x{W}"] = {"ms_per_frame": (tb - ta) / args.delta * 1e3, "frames": [args.frames - args.delta, args.frames],
                                           "peak_gb_above_models": (torch.cuda.max_memory_allocated() - base) / 1e9}
        ops.set_option("raft_corr", "volume")
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
