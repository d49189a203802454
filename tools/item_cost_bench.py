"""What a 128-pixel conv_tc work item costs beyond its main loop: a 3x3 / stride-1 layer with Cout = 128 at 576x1024, batch 4,
bf16x3, timed at Cin = 32, 64, 128 and 256 (1, 2, 4 and 8 K chunks of 32 channels per item).
   python tools/item_cost_bench.py [reps]      (on the GPU box)

Every Cin runs the same instantiation, conv_tc_kernel<128, 1, OP_BF16>, over the same 18432 work items, so the time per item on
one SM is linear in the K chunks per item: the slope is the main loop of one chunk (9 taps x 6 MMAs m64n128k16 per consumer
warpgroup) and the intercept is the fixed cost of an item (pipeline fill, wgmma drain, epilogue) that the tensor cores do not
overlap.  The intercept x items per SM is the most that overlapping the epilogue with the next item's MMAs can recover.
Times are the best of 3 samples, each the mean of `reps` back-to-back calls (CUDA events)."""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vtoonify_b200 import _lib, ops  # noqa: E402

B, H, W, COUT = 4, 576, 1024, 128
CINS = (32, 64, 128, 256)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi not available"
    return q or torch.cuda.get_device_name()


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    dev = torch.device("cuda:0")
    _lib.load()
    ops.set_precision("bf16x3")
    g = torch.Generator().manual_seed(0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    items = B * (H // 16) * (W // 8)
    per_sm = items / sms
    print(f"card: {card()}")
    print(f"{items} work items of 128 pixels x {COUT} channels, {per_sm:.1f} per SM on {sms} SMs")
    ks, us = [], []
    with torch.no_grad():
        for cin in CINS:
            x = ops.to_nhwc(torch.randn((B, cin, H, W), generator=g).to(dev), round_tf32=False)
            bias = (torch.randn(COUT, generator=g) * 0.2).to(dev)
            wt = (torch.randn((COUT, cin, 3, 3), generator=g) / (3 * cin ** 0.5)).to(dev)
            w = ops.prep_weights(wt, cin_pad=cin, round_tf32=False)

            def run():
                return ops.conv2d_nhwc([x], w, ops.conv_taps(3, 1), 1, H, W, bias=bias, act=ops.ACT_LRELU, gain=2 ** 0.5)
            for _ in range(3):
                run()
            torch.cuda.synchronize()
            times = []
            for _ in range(3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    run()
                e1.record(); torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1) / reps)
            t = min(times)
            issued = 3 * 2.0 * B * H * W * cin * COUT * 9
            ks.append(cin // 32); us.append(t * 1e3 / per_sm)
            print(f"Cin {cin:4d}: {cin // 32} K chunks/item  {t:7.3f} ms  {us[-1]:6.2f} us/item/SM  {issued / t * 1e-9:5.0f} TF/s issued")
    slope, icpt = np.polyfit(np.array(ks, float), np.array(us, float), 1)
    resid = np.array(us) - (slope * np.array(ks) + icpt)
    print(f"fit: us per item = {slope:.2f} x K chunks + {icpt:.2f}   (max residual {np.abs(resid).max():.2f} us)")
    print(f"fixed cost per SM: {icpt * per_sm / 1e3:.3f} ms per layer call ({icpt:.2f} us x {per_sm:.1f} items)")


if __name__ == "__main__":
    main()
