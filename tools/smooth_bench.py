"""Times parsing-map smoothing (smooth_parsing_map.py:143-167) per output frame: 800x800 frames, window 5, 20 iterations, det_state_dict
weights, bf16x3, a clip long enough to have interior frames.

Arms, alternated round by round:
  * ``script``: the script's loop as it stands, with the drop-in RAFT on the 11 pairs of every output frame and the warp, fusion and
    ``Downsample`` as torch statements (tests/oracle_smooth.py, library ``Downsample``);
  * ``library``: ``vtoonify_b200.smooth_parsing.smooth_parsing_maps``.
Both take the clip CPU-resident, as the script holds it.  The cost of an interior frame is (T(N) - T(N - K)) / K over whole clips of N
and N - K frames (CUDA events), so each frame's one-time upload and encode is included; launches per frame likewise.  Also reported:
peak memory above the inputs, the warp + fusion + down-sampling of one centre on its own against the torch statements, the relative
difference of the two arms' outputs, and the card's name and power limit read in the same run.  One JSON line on stdout.

    python tools/smooth_bench.py [--frames 16] [--delta 6] [--size 800] [--window 5] [--iters 20] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests import oracle_smooth as O  # noqa: E402
from tests.golden.make_golden_raft import images, raft_args  # noqa: E402
from tests.golden.make_golden_smooth import parsing_maps, parsing_seed  # noqa: E402
from vtoonify_b200 import set_precision  # noqa: E402
from vtoonify_b200 import smooth_parsing as S  # noqa: E402
from vtoonify_b200._lib import launch_count  # noqa: E402
from vtoonify_b200.raft import RAFT  # noqa: E402
from vtoonify_b200.stylegan import Downsample  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402


def script_loop(Is, Ps, raft_model, down, window, iters, dev):
    """the script's loop with the drop-in RAFT (11 pairs per output frame) and torch statements for the rest"""
    w = window
    Is_ = torch.cat((Is[0:w], Is, Is[-w:]), 0)
    Ps_ = torch.cat((Ps[0:w], Ps, Ps[-w:]), 0)
    wt = O.temporal_weights(w, device=dev).reshape(2 * w + 1, 1, 1, 1)
    parse = []
    for ii in range(Is.shape[0]):
        i = ii + w
        image2 = Is_[i - w:i + w + 1].to(dev)
        image1 = Is_[i].repeat(2 * w + 1, 1, 1, 1).to(dev)
        _, flow_up = raft_model((image1 + 1) * 255.0 / 2, (image2 + 1) * 255.0 / 2, iters=iters, test_mode=True)
        parse.append(down(fusion_statements(image1, image2, Ps_[i - w:i + w + 1].to(dev), flow_up, wt, w)).cpu())
    return torch.cat(parse, 0)


def fusion_statements(image1, image2, ps, flow_up, wt, w):
    output, mask = O.warp(torch.cat((image2, ps), 1), flow_up)
    aligned_Is, aligned_Ps = output[:, 0:3], output[:, 3:]
    ws = torch.exp(-((aligned_Is - image1) ** 2).mean(dim=1, keepdim=True) / (2 * (0.2 ** 2))) * mask[:, 0:1]
    aligned_Ps[w] = ps[w]
    ws[w] = 1.0
    weights = ws * wt
    weights = weights / weights.sum(dim=0, keepdim=True)
    return (aligned_Ps * weights).sum(dim=0, keepdim=True)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--delta", type=int, default=6, help="the shorter clip has frames - delta frames")
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--window", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("smooth_bench.py needs a CUDA device")
    dev = torch.device("cuda")
    torch.manual_seed(0)
    m = RAFT(raft_args()).eval()
    m.load_state_dict(det_state_dict(m, seed=0), strict=True)
    m.requires_grad_(False)
    m.to(dev)
    down = Downsample(kernel=[1, 3, 3, 1], factor=2).to(dev).eval()
    set_precision("bf16x3")
    N, Sz, w = args.frames, args.size, args.window
    Is = torch.cat([images(1, Sz, Sz, 70 + k)[k % 2] for k in range(N)]) / 127.5 - 1.0
    Ps = parsing_maps(parsing_seed(N, 3), Sz, Sz)
    lengths = (N - args.delta, N)

    def arm(name, n):
        def run():
            with torch.no_grad():
                if name == "script":
                    return script_loop(Is[:n], Ps[:n], m, down, w, args.iters, dev)
                return S.smooth_parsing_maps(Is[:n], Ps[:n], m, window=w, iters=args.iters)
        return run

    names = ("script", "library")
    times = {(a, n): [] for a in names for n in lengths}
    launches, peak, outs = {}, {}, {}
    base = torch.cuda.memory_allocated()
    for a in names:                                      # warm-up
        arm(a, lengths[0])()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for a in names:
            for n in lengths:
                torch.cuda.reset_peak_memory_stats()
                n0 = launch_count()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = arm(a, n)()
                e1.record()
                torch.cuda.synchronize()
                times[(a, n)].append(e0.elapsed_time(e1))
                launches[(a, n)] = launch_count() - n0
                peak[a] = max(peak.get(a, 0.0), (torch.cuda.max_memory_allocated() - base) / 2 ** 30)
                if n == N:
                    outs[a] = out
    K = lengths[1] - lengths[0]
    per_frame = {a: round((statistics.median(times[(a, N)]) - statistics.median(times[(a, lengths[0])])) / K, 2) for a in names}
    per_frame_spread = {a: [round((min(times[(a, N)]) - max(times[(a, lengths[0])])) / K, 2),
                            round((max(times[(a, N)]) - min(times[(a, lengths[0])])) / K, 2)] for a in names}
    launches_per_frame = {a: (launches[(a, N)] - launches[(a, lengths[0])]) / K for a in names}
    diff = float((outs["library"].double() - outs["script"].double()).norm() / outs["script"].double().norm())

    # warp + fusion + down-sampling of one centre on its own, given the flows of its 2w pairs
    R = 2 * w + 1
    img = Is[:R].to(dev).contiguous()
    par = Ps[:R].to(dev).contiguous()
    flows = (torch.rand((R, 2, Sz, Sz), generator=torch.Generator().manual_seed(1)) - 0.5).mul_(30.0).to(dev)
    kernel = torch.tensor([1.0, 3.0, 3.0, 1.0])
    kernel = (kernel[None] * kernel[:, None] / 64.0).to(dev)
    wt_dev = O.temporal_weights(w, device=dev).reshape(R, 1, 1, 1)
    wt = S.temporal_weights(w).tolist()
    image1 = img[w:w + 1].repeat(R, 1, 1, 1)
    from vtoonify_b200 import ops

    def lib_fuse():
        f = S.parsing_fuse(list(img), list(par), list(flows), wt)
        return ops.upfirdn2d_planar(f[None], kernel, (1, 1), (2, 2), (1, 1, 1, 1))

    def torch_fuse():
        return down(fusion_statements(image1, img, par, flows, wt_dev, w))
    fuse_ms = {}
    with torch.no_grad():
        for name, f in (("library", lib_fuse), ("torch", torch_fuse)):
            f()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                f()
            e1.record()
            torch.cuda.synchronize()
            fuse_ms[name] = round(e0.elapsed_time(e1) / 20, 3)
        fuse_diff = float((lib_fuse().double() - torch_fuse().double()).norm() / torch_fuse().double().norm())

    res = {"workload": f"{N}- and {lengths[0]}-frame clips at {Sz}x{Sz}, window {w}, {args.iters} iterations, bf16x3",
           "card": card(), "gpu": torch.cuda.get_device_properties(0).name,
           "ms_per_interior_frame": per_frame, "ms_per_interior_frame_spread": per_frame_spread,
           "ms_per_clip": {f"{a}_{n}": round(statistics.median(v), 1) for (a, n), v in times.items()},
           "library_launches_per_frame": launches_per_frame, "peak_gb_above_inputs": {a: round(v, 2) for a, v in peak.items()},
           "warp_fusion_down_ms_per_centre": fuse_ms, "warp_fusion_rel_diff": fuse_diff, "arms_rel_diff": diff}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
