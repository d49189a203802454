"""The G step's perceptual term (train_vtoonify_d.py:311-312, train_vtoonify_t.py:253-254): LPIPS VGG16 net-lin on pred and target at
batch 8 and 512 x 512, forward plus backward into pred.

Arms, alternated within each run: the library (vtoonify_b200.lpips) in bf16x3 and in tf32; the plain-torch restatement
(tests/oracle_lpips.py) in fp32 on cuDNN with TF32 off and on.  Prints one JSON line per (run, arm) with ms per step (forward / backward
split from CUDA events), kernel launches (library arms) and max_memory_allocated; then, from a separate torch.profiler run, the kernels
that take the most of the library's bf16x3 step; and a summary line with the analytic TFLOP per step and the card name and power limit
from nvidia-smi in the same call.

    python tools/lpips_bench.py --steps 10 --warmup 2 --runs 2
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def analytic_tflop(B, S):
    """(forward, backward) TFLOP of one step from the layer shapes: the 13 convolutions on 2B images forward, their input gradients on
    the B pred images backward (conv1_1's included)."""
    from vtoonify_b200.lpips import VGG_CONVS
    fwd = bwd = 0.0
    side = S
    prev = 1
    for s, cin, cout in VGG_CONVS.values():
        if s != prev:
            side //= 2
            prev = s
        f = 2.0 * side * side * cin * cout * 9 / 1e12
        fwd += 2 * B * f
        bwd += B * f
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=512)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lpips_bench needs a CUDA device")
    from vtoonify_b200 import _lib, ops
    from tests import oracle_lpips as O
    from tests.test_gpu_lpips import make_loss

    B, S = args.batch, args.size
    percept = make_loss()
    sd = {k: v.detach().clone() for k, v in percept.model.net.state_dict().items()}
    pred, target = O.inputs((B, 3, S, S), 12)
    pred, target = pred.float().cuda(), target.float().cuda()
    arms = {"lib_bf16x3": ("bf16x3", None), "lib_tf32": ("tf32", None), "cudnn_fp32_tf32off": (None, False),
            "cudnn_fp32_tf32on": (None, True)}

    def step(arm, ev=None):
        prec, tf32 = arms[arm]
        if prec:
            ops.set_precision(prec)
        if tf32 is not None:
            torch.backends.cudnn.allow_tf32 = tf32
        p = pred.clone().requires_grad_()
        if ev:
            ev[0].record()
        loss = percept(p, target) if prec else O.perceptual_loss(sd, p, target)
        loss = loss.sum()
        if ev:
            ev[1].record()
        loss.backward()
        if ev:
            ev[2].record()

    results = {}
    torch.set_grad_enabled(True)
    for run in range(args.runs):
        for arm in arms:
            for _ in range(args.warmup):
                step(arm)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            n0 = _lib.launch_count()
            evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.steps)]
            for e in evs:
                step(arm, e)
            torch.cuda.synchronize()
            f = sorted(e[0].elapsed_time(e[1]) for e in evs)
            b = sorted(e[1].elapsed_time(e[2]) for e in evs)
            t = sorted(e[0].elapsed_time(e[2]) for e in evs)
            r = {"run": run, "arm": arm, "ms_step_median": t[len(t) // 2], "ms_fwd_median": f[len(f) // 2],
                 "ms_bwd_median": b[len(b) // 2],
                 "launches_per_step": (_lib.launch_count() - n0) / args.steps if arm.startswith("lib") else None,
                 "max_mem_GB": torch.cuda.max_memory_allocated() / 1e9}
            results.setdefault(arm, []).append(r["ms_step_median"])
            print(json.dumps(r), flush=True)
    ops.set_precision(ops.DEFAULT_PRECISION)
    torch.backends.cudnn.allow_tf32 = True

    from torch.profiler import ProfilerActivity, profile
    step("lib_bf16x3")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            step("lib_bf16x3")
        torch.cuda.synchronize()
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if t and not ev.key.startswith(("cudaLaunch", "cudaMemcpy", "cudaStream", "cudaEvent")):
            rows.append((t / 2e3, ev.count // 2, ev.key[:90]))
    total = sum(r[0] for r in rows)
    rows.sort(reverse=True)
    print(json.dumps({"profile": "lib_bf16x3 step", "kernel_ms_per_step": round(total, 2),
                      "top": [{"ms": round(t, 2), "share": round(t / total, 3), "launches": n, "kernel": k} for t, n, k in rows[:12]]}))
    ops.set_precision(ops.DEFAULT_PRECISION)
    fw, bw = analytic_tflop(B, S)
    print(json.dumps({"card": card(), "batch": B, "size": S, "analytic_TFLOP": {"fwd": round(fw, 3), "bwd": round(bw, 3)},
                      "ms_step_median_per_run": results}))


if __name__ == "__main__":
    main()
