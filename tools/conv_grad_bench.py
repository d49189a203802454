"""Time the convolution's forward, input gradient and weight gradient on training-sized layers, against cuDNN.

    python tools/conv_grad_bench.py [--iters 20] [--warmup 3]

For each layer: this library's forward (conv2d_gradfix.conv2d under no_grad), input gradient (the transposed op on the forward
kernels, under the current precision, bf16x3 by default) and weight gradient (the wgmma weight-gradient kernel), then cuDNN's
F.conv2d and its two backward convolutions (torch.nn.grad.conv2d_input / conv2d_weight) with allow_tf32 False and True.
Times are CUDA-event means over --iters calls after --warmup calls; TFLOP/s are algorithmic (2 * B * Ho * Wo * Cout * Cin * kh * kw
per pass, the same for all three passes).  The card's name, power limit and top SM clock are read in the same run.
"""
import argparse
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (label, B or G, Cin, Cout, H, W, k, stride, padding, dilation, per_sample)
LAYERS = [
    ("AdaResBlock 512 3x3 d1 32x32", 4, 512, 512, 32, 32, 3, 1, 1, 1, False),
    ("AdaResBlock 512 3x3 d2 32x32", 4, 512, 512, 32, 32, 3, 1, 2, 2, False),
    ("AdaResBlock 512 3x3 d4 32x32", 4, 512, 512, 32, 32, 3, 1, 4, 4, False),
    ("256 3x3 128x128", 4, 256, 256, 128, 128, 3, 1, 1, 1, False),
    ("64 3x3 512x512", 2, 64, 64, 512, 512, 3, 1, 1, 1, False),
    ("down 256->512 3x3 s2 p0 66x66", 4, 256, 512, 66, 66, 3, 2, 0, 1, False),
    ("skip 256->512 1x1 s2 p0 66x66", 4, 256, 512, 66, 66, 1, 2, 0, 1, False),
    ("modulated 512 3x3 32x32 per-sample G=4", 4, 512, 512, 32, 32, 3, 1, 1, 1, True),
]


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        print("conv_grad_bench: needs a CUDA device", file=sys.stderr)
        return 2
    from vtoonify_b200.op import conv2d_gradfix as gf
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        card = f"nvidia-smi unavailable ({e})"
    print(f"card: {card}; torch {torch.__version__}, cuDNN {torch.backends.cudnn.version()}")
    print("| layer | pass | ours ms | ours TFLOP/s | cuDNN fp32 ms | cuDNN tf32 ms |")
    print("|---|---|---|---|---|---|")
    torch.backends.cudnn.benchmark = True
    for label, B, Cin, Cout, H, W, k, s, p, d, per_sample in LAYERS:
        g = torch.Generator(device="cuda").manual_seed(0)
        G = B if per_sample else 1
        x = torch.randn((1, B * Cin, H, W) if per_sample else (B, Cin, H, W), device="cuda", generator=g)
        w = torch.randn((G * Cout, Cin, k, k), device="cuda", generator=g) / (Cin * k * k) ** 0.5
        with torch.no_grad():
            y = gf.conv2d(x, w, stride=s, padding=p, dilation=d, groups=G)
            go = torch.randn(tuple(y.shape), device="cuda", generator=g)
        Ho, Wo = y.shape[2], y.shape[3]
        flops = 2.0 * B * Ho * Wo * Cout * Cin * k * k
        st, pd, dl = (s, s), (p, p), (d, d)
        op = tuple(x.shape[i + 2] - (Ho - 1) * s - (1 - 2 * p) - d * (k - 1) for i in range(2))
        tr = gf._conv2d_gradfix(True, tuple(w.shape), st, pd, op, dl, G)
        ours = {
            "forward": lambda: gf.conv2d(x, w, stride=s, padding=p, dilation=d, groups=G),
            "input grad": lambda: tr.apply(go, w, None),
            "weight grad": lambda: gf._weight_grad(False, tuple(w.shape), go, x, st, pd, dl, G),
        }
        ref = {
            "forward": lambda: F.conv2d(x, w, stride=s, padding=p, dilation=d, groups=G),
            "input grad": lambda: torch.nn.grad.conv2d_input(tuple(x.shape), w, go, stride=s, padding=p, dilation=d, groups=G),
            "weight grad": lambda: torch.nn.grad.conv2d_weight(x, tuple(w.shape), go, stride=s, padding=p, dilation=d, groups=G),
        }
        with torch.no_grad():
            for name in ("forward", "input grad", "weight grad"):
                t_ours = timed(ours[name], args.iters, args.warmup)
                t_ref = {}
                for tf32 in (False, True):
                    torch.backends.cudnn.allow_tf32 = tf32
                    t_ref[tf32] = timed(ref[name], args.iters, args.warmup)
                torch.backends.cudnn.allow_tf32 = True
                print(f"| {label} | {name} | {t_ours:.3f} | {flops / t_ours / 1e9:.1f} | {t_ref[False]:.3f} | {t_ref[True]:.3f} |", flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
