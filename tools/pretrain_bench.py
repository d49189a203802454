"""Encoder pretraining step (train_vtoonify_d.py:132-148, the student half): VToonify-D forward(return_feat=True) + MSE on feat and
skip + backward at batch 8, 256 x 256, d_s = 0 and 0.5.

Arms, alternated within each run: the library in bf16x3 and in tf32, and the float64-oracle restatement (tests/oracle_vtoonify_feat.py)
run in fp32 through cuDNN with TF32 on (PyTorch's default for cuDNN convolutions) and off.  Reports ms per step with the
forward / backward split (CUDA events), kernel launches per step (library), max_memory_allocated, the analytic work per step, and,
from a separate torch.profiler run, the share of the library step spent in the weight-gradient kernel.  Prints one JSON line per
(run, arm, d_s) and a summary line; card name and power limit come from nvidia-smi in the same call.

    python tools/pretrain_bench.py --steps 20 --warmup 3 --runs 2
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def analytic_tflop(B, S, d_s):
    """(forward, backward, of which weight gradients) TFLOP of one step, from the layer shapes (x does not require grad)."""
    layers = [(S, 22, 32, 9, 1, True), (S, 32, 128, 9, 1, True), (S // 2, 128, 256, 9, 2, True), (S // 2, 256, 256, 9, 1, True),
              (S // 4, 256, 512, 9, 2, True), (S // 4, 512, 512, 9, 1, True), (S // 8, 512, 512, 9, 2, True),
              (S // 8, 512, 512, 9, 1, True)]            # (output size, Cin, Cout, taps, stride, trainable)
    layers += [(S // 8, 512, 512, 9, 1, True)] * 12 + [(S // 8, 512, 3, 1, 1, True)]
    if d_s:
        layers += [(S // 8, 512, 512, 9, 1, False)] * 12
    fwd = bwd = wg = 0.0
    for i, (o, cin, cout, taps, _, train) in enumerate(layers):
        f = 2.0 * B * o * o * cin * cout * taps / 1e12
        fwd += f
        if i > 0:
            bwd += f                      # input gradient (none for the first layer: x is data)
        if train:
            bwd += f
            wg += f
    return fwd, bwd, wg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pretrain_bench needs a CUDA device")
    from vtoonify_b200 import _lib, ops
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict
    from tests.oracle_vtoonify_feat import case_inputs, feat_forward, targets

    B, S = args.batch, args.size
    m = VToonify(backbone="dualstylegan")
    m.load_state_dict(det_state_dict(m, seed=0), strict=True)
    m = m.cuda()
    m.res.requires_grad_(False)
    m.generator.requires_grad_(False)
    sd = {k: v.detach().clone().requires_grad_(k.startswith("encoder.")) for k, v in m.state_dict().items()}
    x, style = case_inputs(B, S, S)
    x, style = x.cuda(), style.cuda()
    t_f, t_s = targets((B, 512, S // 8, S // 8), (B, 3, S // 8, S // 8))
    t_f, t_s = t_f.cuda(), t_s.cuda()

    def lib_fwd(d_s):
        return m(x, style, d_s=d_s, return_feat=True)

    def ora_fwd(d_s):
        return feat_forward(sd, x, style, d_s, "dualstylegan")

    arms = {"lib_bf16x3": (lib_fwd, "bf16x3", None), "lib_tf32": (lib_fwd, "tf32", None),
            "cudnn_fp32_tf32on": (ora_fwd, None, True), "cudnn_fp32_tf32off": (ora_fwd, None, False)}

    def step(arm, d_s, ev=None):
        fwd, prec, tf32 = arms[arm]
        if prec:
            ops.set_precision(prec)
        else:
            torch.backends.cudnn.allow_tf32 = tf32
        for p in list(m.parameters()) + list(sd.values()):
            p.grad = None
        if ev:
            ev[0].record()
        feat, skip = fwd(d_s)
        loss = F.mse_loss(feat, t_f) + F.mse_loss(skip, t_s)
        if ev:
            ev[1].record()
        loss.backward()
        if ev:
            ev[2].record()

    info = {"card": card(), "batch": B, "size": S}
    results = {}
    torch.set_grad_enabled(True)
    for run in range(args.runs):
        for d_s in (0.0, 0.5):
            for arm in arms:
                for _ in range(args.warmup):
                    step(arm, d_s)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                n0 = _lib.launch_count()
                evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.steps)]
                for e in evs:
                    step(arm, d_s, e)
                torch.cuda.synchronize()
                f = sorted(e[0].elapsed_time(e[1]) for e in evs)
                b = sorted(e[1].elapsed_time(e[2]) for e in evs)
                t = sorted(e[0].elapsed_time(e[2]) for e in evs)
                r = {"run": run, "arm": arm, "d_s": d_s, "ms_step_median": t[len(t) // 2], "ms_fwd_median": f[len(f) // 2],
                     "ms_bwd_median": b[len(b) // 2], "launches_per_step": (_lib.launch_count() - n0) / args.steps,
                     "max_mem_GB": torch.cuda.max_memory_allocated() / 1e9}
                results.setdefault((arm, d_s), []).append(r["ms_step_median"])
                print(json.dumps(r), flush=True)
    ops.set_precision(ops.DEFAULT_PRECISION)
    torch.backends.cudnn.allow_tf32 = True

    # weight-gradient share of the library step: a separate profiled run
    shares = {}
    from torch.profiler import ProfilerActivity, profile
    for d_s in (0.0, 0.5):
        step("lib_bf16x3", d_s)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                step("lib_bf16x3", d_s)
            torch.cuda.synchronize()
        tot = wg = 0.0
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            if ev.key.startswith(("cudaLaunch", "cudaMemcpy", "cudaStream", "cudaEvent")):
                continue
            tot += t
            if "wgrad" in ev.key:
                wg += t
        shares[d_s] = wg / tot if tot else float("nan")
    summary = dict(info)
    for d_s in (0.0, 0.5):
        fw, bw, wgf = analytic_tflop(B, S, d_s)
        summary[f"d_s={d_s}"] = {"analytic_TFLOP": {"fwd": round(fw, 3), "bwd": round(bw, 3), "wgrad": round(wgf, 3)},
                                 "wgrad_kernel_share_lib_bf16x3": round(shares[d_s], 3),
                                 "ms_step_median_per_run": {a: results[(a, d_s)] for a in arms}}
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
