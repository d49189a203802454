"""Row-strip layers (vt_conv2d_rs) of VToonify-D at 576x1024, batch 4: conv_rs_kernel (rs_kernel=1) against the conv_tc_kernel route
(rs_kernel=0), alternated in one process.
   python tools/rs_bench.py [reps]      (on the GPU box)

Per layer: ms per launch of each route, issued TFLOP/s (3 bf16 products per multiply-add), the roofline floor (the larger of the
issued FLOPs at the 989 TFLOP/s bf16 data-sheet rate and the HBM bytes at 3.35 TB/s), and max|rs_kernel 1 - rs_kernel 0| over
max|rs_kernel 0| of the activation and of the ToRGB image.  With Cout = 32 the rs route hands both kernels the N-stacked weight split
(conv_rs_kernel's A operand), so the rs_kernel=0 column is conv_tc_kernel in its N-stacked mode, not its default 6-MMA bf16 mode."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vtoonify_b200 import _lib, ops  # noqa: E402

PEAK_BF16, HBM = 989e12, 3.35e12
# (label, Cin, Cout, H, W, per-sample weights, fused ToRGB: None / "skip" / "only")
LAYERS = [("32->32 k9 s1 2304x4096 (image-only ToRGB)", 32, 32, 2304, 4096, False, "only"),
          ("64->64 k9 s1 1152x2048 (noise, lrelu, ToRGB)", 64, 64, 1152, 2048, True, "skip"),
          ("32->32 k9 s1 576x1024 (noise, lrelu)", 32, 32, 576, 1024, False, None)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi not available"
    return q or torch.cuda.get_device_name()


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    dev = torch.device("cuda:0")
    lib = _lib.load()
    ops.set_precision("bf16x3")
    B = 4
    g = torch.Generator().manual_seed(0)
    k1 = torch.tensor([1., 3., 3., 1.])
    print(f"card: {card()}")
    with torch.no_grad():
        for label, cin, cout, H, W, per_sample, rgb_mode in LAYERS:
            wB = B if per_sample else 1
            x = torch.randn((B, H, W, cin), generator=g).to(dev)
            wt = torch.randn((wB, cout, cin, 3, 3), generator=g) / (3 * cin ** 0.5)
            w = torch.cat([ops.prep_weights(wt[i].to(dev), cin_pad=cin, round_tf32=False) for i in range(wB)], 0).contiguous()
            kw = dict(bias=(torch.randn(cout, generator=g) * 0.2).to(dev), act=ops.ACT_LRELU, slope=0.2, gain=2 ** 0.5,
                      noise=torch.randn((B, 1, H, W), generator=g).to(dev), noise_w=torch.tensor([0.3]).to(dev))
            rgb = None
            if rgb_mode is not None:
                rgb = {"w": (torch.randn((wB, 1, 3, cout), generator=g) * 0.2).to(dev), "bias": (torch.randn(3, generator=g) * 0.1).to(dev),
                       "skip": torch.randn((B, 3, H // 2, W // 2), generator=g).to(dev), "kernel": (k1[:, None] * k1[None, :] / 64 * 4).to(dev),
                       "only": rgb_mode == "only"}

            def run():
                return ops.conv2d_nhwc([x], w, ops.conv_taps(3, 1), 1, H, W, rgb=rgb, **kw)

            outs, times = {}, {0: [], 1: []}
            for route in (1, 0):
                lib.vt_set_option(b"rs_kernel", route)
                outs[route] = run()
            for _ in range(3):   # alternate the routes; each sample is the mean of `reps` back-to-back launches
                for route in (1, 0):
                    lib.vt_set_option(b"rs_kernel", route)
                    run(); torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        run()
                    e1.record(); torch.cuda.synchronize()
                    times[route].append(e0.elapsed_time(e1) / reps)
            lib.vt_set_option(b"rs_kernel", 1)
            issued = 3 * 2.0 * B * H * W * cin * cout * 9
            nbytes = 4.0 * (B * H * W * cin + (0 if rgb_mode == "only" else B * H * W * cout) + B * H * W + w.numel()
                            + (B * 3 * H * W * 5 // 4 if rgb_mode else 0))
            floor_ms = max(issued / PEAK_BF16, nbytes / HBM) * 1e3

            def rel(a, b):
                return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item() if a is not None and b is not None else float("nan")

            pair = [o if isinstance(o, tuple) else (o, None) for o in (outs[1], outs[0])]
            t1, t0 = min(times[1]), min(times[0])
            print(f"{label:48s} conv_rs {t1:7.3f} ms ({issued / t1 * 1e-9:5.0f} TFLOP/s) | conv_tc {t0:7.3f} ms ({issued / t0 * 1e-9:5.0f} TFLOP/s)"
                  f" | floor {floor_ms:.2f} ms | max diff act {rel(pair[0][0], pair[1][0]):.1e} rgb {rel(pair[0][1], pair[1][1]):.1e}")


if __name__ == "__main__":
    main()
