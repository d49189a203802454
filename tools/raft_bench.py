"""Times RAFT as smooth_parsing_map.py runs it per output frame: image1 repeated 11 times against its 11 neighbours at 800x800,
20 iterations, test mode, det_state_dict weights.

Arms, alternated round by round: the library in bf16x3 and tf32, and the plain-torch restatement (tests/oracle_raft.py) on cuDNN in
fp32 and with TF32.  Reports ms per call (CUDA events, median of the rounds), the library's forward split into encoders / correlation /
iterations (events between the phases of one call, from a separate instrumented run), launches per call, peak memory above the inputs,
and the analytic TFLOP per call from the layer shapes.  One JSON line on stdout.

    python tools/raft_bench.py [--pairs 11] [--size 800] [--iters 20] [--rounds 5] [--profile out.json]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests import oracle_raft as O  # noqa: E402
from tests.golden.make_golden_raft import images, raft_args  # noqa: E402
from vtoonify_b200 import ops, set_precision  # noqa: E402
from vtoonify_b200._lib import launch_count  # noqa: E402
from vtoonify_b200.raft import RAFT  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402


def tflop(B, H, W, iters):
    """multiply-adds x 2 of every convolution and the correlation, from the layer shapes (test mode: one mask head)"""
    def conv(n, h, w, cin, cout, k):
        return 2.0 * n * h * w * cin * cout * k
    h2, w2, h4, w4, h8, w8 = H // 2, W // 2, H // 4, W // 4, H // 8, W // 8

    def enc(n, cout):
        f = conv(n, h2, w2, 3, 64, 49) + 4 * conv(n, h2, w2, 64, 64, 9)
        f += conv(n, h4, w4, 64, 96, 9) + conv(n, h4, w4, 64, 96, 1) + 3 * conv(n, h4, w4, 96, 96, 9)
        f += conv(n, h8, w8, 96, 128, 9) + conv(n, h8, w8, 96, 128, 1) + 3 * conv(n, h8, w8, 128, 128, 9)
        return f + conv(n, h8, w8, 128, cout, 1)
    e = enc(2 * B, 256) + enc(B, 256)
    corr = 2.0 * B * (h8 * w8) ** 2 * 256
    it = (conv(B, h8, w8, 324, 256, 1) + conv(B, h8, w8, 256, 192, 9) + conv(B, h8, w8, 2, 128, 49) + conv(B, h8, w8, 128, 64, 9)
          + conv(B, h8, w8, 256, 126, 9) + 2 * (conv(B, h8, w8, 384, 256, 5) + conv(B, h8, w8, 384, 128, 5))
          + conv(B, h8, w8, 128, 256, 9) + conv(B, h8, w8, 256, 2, 9))
    mask = conv(B, h8, w8, 128, 256, 9) + conv(B, h8, w8, 256, 576, 1)
    return {"encoders": e / 1e12, "correlation": corr / 1e12, "iterations": iters * it / 1e12, "mask_head": mask / 1e12,
            "total": (e + corr + iters * it + mask) / 1e12}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=11)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", default=None, help="write a torch.profiler kernel table of one library call (bf16x3) here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("raft_bench.py needs a CUDA device")
    dev = torch.device("cuda")
    m = RAFT(raft_args()).eval()
    sd = det_state_dict(m, seed=0)
    m.load_state_dict(sd, strict=True)
    m.requires_grad_(False)
    m.to(dev)
    sd = {k: v.to(dev) for k, v in sd.items()}
    P, S = args.pairs, args.size
    a, _ = images(1, S, S, 11)
    i1 = a.repeat(P, 1, 1, 1).to(dev)
    i2 = torch.cat([images(1, S, S, 20 + k)[1] for k in range(P)]).to(dev)

    def lib(prec):
        def run():
            set_precision(prec)
            with torch.no_grad():
                return m(i1, i2, iters=args.iters, test_mode=True)
        return run

    def ref(tf32):
        def run():
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
            with torch.no_grad():
                return O.raft_forward(sd, i1, i2, args.iters, None, True, every_mask=False)
        return run

    arms = {"library_bf16x3": lib("bf16x3"), "library_tf32": lib("tf32"), "cudnn_fp32": ref(False), "cudnn_tf32": ref(True)}
    times = {k: [] for k in arms}
    peak = {}
    launches = {}
    base = torch.cuda.memory_allocated()
    for k, f in arms.items():                   # warm-up: every arm and shape once
        f()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for k, f in arms.items():
            torch.cuda.reset_peak_memory_stats()
            n0 = launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            peak[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
            if k.startswith("library"):
                launches[k] = launch_count() - n0

    # phase split of one library call: CUDA events at the entry and exit of the forward's three ops.nvtx_range phases (a separate run)
    spans = []

    class timed(ops.nvtx_range):
        def __enter__(self):
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
            return super().__enter__()

        def __exit__(self, *exc):
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            spans.append((self.name.replace("raft.", ""), self.e0, e1))
            return super().__exit__(*exc)
    orig = ops.nvtx_range
    ops.nvtx_range = timed
    try:
        set_precision("bf16x3")
        with torch.no_grad():
            m(i1, i2, iters=args.iters, test_mode=True)
        torch.cuda.synchronize()
    finally:
        ops.nvtx_range = orig
    split = {n: round(a.elapsed_time(b), 2) for n, a, b in spans}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        set_precision("bf16x3")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with torch.no_grad():
                m(i1, i2, iters=args.iters, test_mode=True)
            torch.cuda.synchronize()
        with open(args.profile, "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))

    props = torch.cuda.get_device_properties(0)
    res = {"workload": f"{P} pairs {S}x{S}, {args.iters} iterations, test mode", "gpu": props.name,
           "ms_per_call": {k: round(statistics.median(v), 2) for k, v in times.items()},
           "ms_spread": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()},
           "library_phase_ms_bf16x3": split, "launches_per_call": launches,
           "peak_gb_above_inputs": {k: round(v, 2) for k, v in peak.items()}, "analytic_tflop": tflop(P, S, S, args.iters)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
