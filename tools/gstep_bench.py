"""VToonify G step (train_vtoonify_d.py:299-338, train_vtoonify_t.py:242-270): forward(return_mask=True) at 256 x 256 plus a second
call on the 224 x 224 crop, an image loss and the mask terms, backward into x-free encoder and fusion parameters, at batch 8, D (d_s 0.5)
and T.

Arms, alternated within each run: the library in bf16x3 and in tf32; the float64-oracle restatement (oracle/vt_oracle.py through
tests/oracle_vtoonify_gstep.py) run in fp32 through cuDNN with TF32 on and off; and level (b), the reference module's own statements
(``restated_forward``: grouped modulated convolutions, nn.Conv2d on cuDNN) on vtoonify_b200.op's conv2d_gradfix, upfirdn2d and
fused_leaky_relu in bf16x3.  Prints one JSON line per (run, arm, case) with ms per step (forward / backward split from CUDA events),
kernel launches (library ops) and max_memory_allocated; then, from a separate torch.profiler run, the kernels that take the most of
the library's bf16x3 D step; and a summary line with the analytic TFLOP per step and the card name and power limit from nvidia-smi
in the same call.

    python tools/gstep_bench.py --steps 10 --warmup 2 --runs 2
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


def analytic_tflop(B, S, D):
    """(forward, backward) TFLOP of one model call at input S x S, from the layer shapes: encoder (with the frozen ModRes blocks on D),
    five generator levels (the up-conv counted as the transposed conv's MACs, input pixels x Cin x Cout x 9; conv2; ToRGB), the fusion
    convolutions.  The backward counts an input gradient for every layer but the first and a weight gradient for the trained ones."""
    ch = {S: 128, S // 2: 256, S // 4: 512, S // 8: 512}
    layers = [(S, 22, 32, 9, True), (S, 32, 128, 9, True), (S // 2, 128, 256, 9, True), (S // 2, 256, 256, 9, True),
              (S // 4, 256, 512, 9, True), (S // 4, 512, 512, 9, True), (S // 8, 512, 512, 9, True), (S // 8, 512, 512, 9, True)]
    layers += [(S // 8, 512, 512, 9, True)] * 12 + [(S // 8, 512, 3, 1, True)]
    if D:
        layers += [(S // 8, 512, 512, 9, False)] * 12
    gen = {0: (512, 512), 1: (512, 256), 2: (256, 128), 3: (128, 64), 4: (64, 32)}
    for lvl in range(5):
        o = S // 8 * 2 ** lvl
        cin, cout = gen[lvl]
        if o in ch:
            c = ch[o]
            layers += [(o, 2 * c, c, 9, True), (o, c + 3, 3, 9, True)] + ([(o, 2 * c, 1, 9, True)] if D else [])
        layers += [(o, cin, cout, 9, False), (2 * o, cout, cout, 9, False), (2 * o, cout, 3, 1, False)]
    fwd = bwd = 0.0
    for i, (o, cin, cout, taps, train) in enumerate(layers):
        f = 2.0 * B * o * o * cin * cout * taps / 1e12
        fwd += f
        bwd += (f if i > 0 else 0.0) + (f if train else 0.0)
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gstep_bench needs a CUDA device")
    from vtoonify_b200 import _lib, ops
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict
    from tests.oracle_vtoonify_gstep import O, image_target, library_ops, loss_of, restated_forward, trained
    from tests.oracle_vtoonify_feat import case_inputs

    B, S = args.batch, 256
    x, style = case_inputs(B, S, S)
    x, style = x.cuda(), style.cuda()
    crop = x[:, :, 16:240, 16:240].contiguous()
    models, sds = {}, {}
    for bb in ("dualstylegan", "toonify"):
        m = VToonify(backbone=bb)
        m.load_state_dict(det_state_dict(m, seed=0), strict=True)
        m = m.cuda().requires_grad_(False)
        for n, p in m.named_parameters():
            p.requires_grad_(trained(n))
        models[bb] = m
        sds[bb] = {k: v.detach().clone().requires_grad_(trained(k)) for k, v in m.state_dict().items()}
    t1, t2 = image_target((B, 3, 4 * S, 4 * S)).cuda(), image_target((B, 3, 4 * 224, 4 * 224), seed=1).cuda()

    def call(arm, bb, xin, d_s):
        if arm.startswith("lib"):
            r = models[bb](xin, style, d_s=d_s, return_mask=True)
        elif arm == "level_b":
            return restated_forward(sds[bb], xin, style, d_s, bb, ops=lib_ops)
        else:
            r = O.vtoonify_forward(sds[bb], xin, style, d_s, bb, return_mask=True)
        return r if bb == "dualstylegan" else (r, [])

    lib_ops = library_ops()
    arms = {"lib_bf16x3": ("bf16x3", None), "lib_tf32": ("tf32", None), "level_b": ("bf16x3", True), "cudnn_fp32_tf32on": (None, True),
            "cudnn_fp32_tf32off": (None, False)}
    cases = {"D": ("dualstylegan", 0.5), "T": ("toonify", 0.5)}

    def step(arm, case, ev=None):
        prec, tf32 = arms[arm]
        bb, d_s = cases[case]
        if prec:
            ops.set_precision(prec)
        if tf32 is not None:
            torch.backends.cudnn.allow_tf32 = tf32
        for p in list(models[bb].parameters()) + list(sds[bb].values()):
            p.grad = None
        if ev:
            ev[0].record()
        img, masks = call(arm, bb, x, d_s)
        img2, masks2 = call(arm, bb, crop, d_s)
        loss = loss_of(img, masks, t1) + loss_of(img2, masks2, t2)
        if ev:
            ev[1].record()
        loss.backward()
        if ev:
            ev[2].record()

    info = {"card": card(), "batch": B, "calls": "256^2 + 224^2 crop"}
    results = {}
    torch.set_grad_enabled(True)
    for run in range(args.runs):
        for case in cases:
            for arm in arms:
                for _ in range(args.warmup):
                    step(arm, case)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                n0 = _lib.launch_count()
                evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.steps)]
                for e in evs:
                    step(arm, case, e)
                torch.cuda.synchronize()
                f = sorted(e[0].elapsed_time(e[1]) for e in evs)
                b = sorted(e[1].elapsed_time(e[2]) for e in evs)
                t = sorted(e[0].elapsed_time(e[2]) for e in evs)
                r = {"run": run, "arm": arm, "case": case, "ms_step_median": t[len(t) // 2], "ms_fwd_median": f[len(f) // 2],
                     "ms_bwd_median": b[len(b) // 2], "launches_per_step": (_lib.launch_count() - n0) / args.steps,
                     "max_mem_GB": torch.cuda.max_memory_allocated() / 1e9}
                results.setdefault((arm, case), []).append(r["ms_step_median"])
                print(json.dumps(r), flush=True)
    ops.set_precision(ops.DEFAULT_PRECISION)
    torch.backends.cudnn.allow_tf32 = True

    # where the library's bf16x3 D step spends its time: a separate profiled run
    from torch.profiler import ProfilerActivity, profile
    step("lib_bf16x3", "D")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            step("lib_bf16x3", "D")
        torch.cuda.synchronize()
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if t and not ev.key.startswith(("cudaLaunch", "cudaMemcpy", "cudaStream", "cudaEvent")):
            rows.append((t / 2e3, ev.count // 2, ev.key[:90]))
    total = sum(r[0] for r in rows)
    rows.sort(reverse=True)
    print(json.dumps({"profile": "lib_bf16x3 D step", "kernel_ms_per_step": round(total, 2),
                      "top": [{"ms": round(t, 2), "share": round(t / total, 3), "launches": n, "kernel": k} for t, n, k in rows[:12]]}))
    ops.set_precision(ops.DEFAULT_PRECISION)
    summary = dict(info)
    for case, (bb, _) in cases.items():
        fw = sum(analytic_tflop(B, s, bb == "dualstylegan")[0] for s in (256, 224))
        bw = sum(analytic_tflop(B, s, bb == "dualstylegan")[1] for s in (256, 224))
        summary[case] = {"analytic_TFLOP": {"fwd": round(fw, 3), "bwd": round(bw, 3)},
                         "ms_step_median_per_run": {a: results[(a, case)] for a in arms}}
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
