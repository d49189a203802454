"""Times a temporally smoothed video through the library: 400x400 uint8 frames (smoothing at 800x800), window 5, 20 iterations, batch
4, bf16x3, det_state_dict weights (VToonify-D, BiSeNet, RAFT).

Arms, alternated round by round:
  * ``one_pass``: ``FramePipeline(..., parsing_net, smoothing=(raft, 5, 20))`` on uint8 batches;
  * ``two_step``: the whole clip's ``Is`` / ``Ps`` held on the host as smooth_parsing_map.py holds them (``Is`` from
    ``smooth_parsing.frame_prep``, ``Ps = parsing_net(2 * Is[i])[0]``), then ``smooth_parsing_maps``, then ``FramePipeline`` on
    ``(frames, parse)`` batches (style_transfer.py --parsing_map_path, without the file).
Per arm: ms per interior frame as (T(N) - T(N - K)) / K over whole clips (a host clock around work that ends in a device synchronise),
peak device memory above the models (torch.cuda.max_memory_allocated) and peak host RSS above the arm's start (sampled every 2 ms) for
both clip lengths, and whether the two arms' frames are bit-identical.  The card's name and power limit are read in the same run.  One
JSON line on stdout.

    python tools/smooth_video_bench.py [--frames 16] [--delta 8] [--size 400] [--rounds 2]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests.golden.make_golden_raft import raft_args  # noqa: E402
from vtoonify_b200 import set_precision  # noqa: E402
from vtoonify_b200 import smooth_parsing as S  # noqa: E402
from vtoonify_b200.bisenet import BiSeNet  # noqa: E402
from vtoonify_b200.frame_loop import FramePipeline  # noqa: E402
from vtoonify_b200.raft import RAFT  # noqa: E402
from vtoonify_b200.vtoonify import VToonify  # noqa: E402
from vtoonify_b200.weights import det_inputs, det_state_dict  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def rss_bytes():
    with open("/proc/self/statm") as f:
        return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")


class RssPeak:
    """the peak resident set size while the block runs, above its value at the start"""

    def __enter__(self):
        self.base = self.peak = rss_bytes()
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._watch, daemon=True)
        self._t.start()
        return self

    def _watch(self):
        while not self._stop.is_set():
            self.peak = max(self.peak, rss_bytes())
            time.sleep(0.002)

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()
        self.peak = max(self.peak, rss_bytes())
        self.above = self.peak - self.base


def clip(N, H, W, seed=0):
    """a moving colour ramp with noise: uint8 [N, H, W, 3]"""
    g = torch.Generator().manual_seed(seed)
    y = torch.arange(H).float()[:, None, None]
    x = torch.arange(W).float()[None, :, None]
    c = torch.tensor([0.7, 1.0, 1.3])[None, None, :]
    out = []
    for t in range(N):
        v = 127.5 + 100 * torch.sin((x * c + 2.0 * t) / 37.0) * torch.cos((y / c + 1.5 * t) / 53.0)
        out.append((v + torch.randint(-8, 9, (H, W, 3), generator=g)).clamp(0, 255).to(torch.uint8))
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--delta", type=int, default=8, help="the shorter clip has frames - delta frames")
    ap.add_argument("--size", type=int, default=400)
    ap.add_argument("--window", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("smooth_video_bench.py needs a CUDA device")
    dev = torch.device("cuda")
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
    N, Sz, w, it, B = args.frames, args.size, args.window, args.iters, args.batch
    frames = clip(N, Sz, Sz)
    lengths = (N - args.delta, N)

    def one_pass(n):
        pipe = FramePipeline(model, style, d_s=0.5, parsing_net=parser, smoothing=(raft, w, it))
        return list(pipe.run([frames[i:min(i + B, n)].pin_memory() for i in range(0, n, B)]))

    def two_step(n):
        with torch.no_grad():
            Is, Ps = [], []
            for i in range(n):
                I = S.frame_prep(frames[i:i + 1].to(dev))[0]
                Is.append(I.cpu())
                Ps.append(parser(2 * I)[0].cpu())
            Is, Ps = torch.cat(Is), torch.cat(Ps)          # the script's whole-clip host tensors
            parse = S.smooth_parsing_maps(Is, Ps, raft, window=w, iters=it)
            del Is, Ps
        pipe = FramePipeline(model, style, d_s=0.5)
        return list(pipe.run([(frames[i:min(i + B, n)].pin_memory(), parse[i:min(i + B, n)].pin_memory()) for i in range(0, n, B)]))

    arms = {"one_pass": one_pass, "two_step": two_step}
    times = {(a, n): [] for a in arms for n in lengths}
    dev_peak, host_peak, outs = {}, {}, {}
    base = torch.cuda.memory_allocated()
    for f in arms.values():                              # warm-up
        f(lengths[0])
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for a, f in arms.items():
            for n in lengths:
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                with RssPeak() as rss:
                    t0 = time.perf_counter()
                    out = f(n)
                    torch.cuda.synchronize()
                    times[(a, n)].append((time.perf_counter() - t0) * 1e3)
                key = f"{a}_{n}"
                dev_peak[key] = max(dev_peak.get(key, 0.0), (torch.cuda.max_memory_allocated() - base) / 2 ** 30)
                host_peak[key] = max(host_peak.get(key, 0.0), rss.above / 2 ** 30)
                if n == N:
                    outs[a] = out
                del out
    K = lengths[1] - lengths[0]
    per_frame = {a: round((statistics.median(times[(a, N)]) - statistics.median(times[(a, lengths[0])])) / K, 2) for a in arms}
    spread = {a: [round((min(times[(a, N)]) - max(times[(a, lengths[0])])) / K, 2),
                  round((max(times[(a, N)]) - min(times[(a, lengths[0])])) / K, 2)] for a in arms}
    same = len(outs["one_pass"]) == len(outs["two_step"]) and all(torch.equal(x, y) for x, y in zip(outs["one_pass"], outs["two_step"]))
    res = {"workload": f"{N}- and {lengths[0]}-frame {Sz}x{Sz} uint8 clips, smoothing at {2 * Sz}x{2 * Sz}, window {w}, {it} "
                       f"iterations, batch {B}, bf16x3",
           "card": card(), "gpu": torch.cuda.get_device_properties(0).name,
           "ms_per_interior_frame": per_frame, "ms_per_interior_frame_spread": spread,
           "ms_per_clip": {f"{a}_{n}": round(statistics.median(v), 1) for (a, n), v in times.items()},
           "peak_device_gb_above_models": {k: round(v, 3) for k, v in dev_peak.items()},
           "peak_host_rss_gb_above_start": {k: round(v, 3) for k, v in host_peak.items()},
           "frames_bit_identical": same}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
