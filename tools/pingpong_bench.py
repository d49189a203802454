"""The conv_tc layers of VToonify-D at 576x1024, batch 4, that run 128 x 128 bf16-split work items: tc_pingpong 0 (both consumer
warpgroups on every item) against 1 (automatic: launches with more items than SMs) and 2 (ping-pong wherever it exists, one item
per CTA included), alternated in one process.
   python tools/pingpong_bench.py [reps]      (on the GPU box)

Per layer: ms per call of each mode (the best of 3 samples, each the mean of `reps` back-to-back calls, CUDA events), issued
TFLOP/s of mode 0 (3 bf16 products per multiply-add, 12 on the folded up-convolution) and whether the modes gave bit-identical
outputs.  Layers are labelled as in `bench.py --dump-layers`: Cin->Cout, taps, stride, input map.  The 512->512 72x128 layer is
the wide layer whose last partial round of items runs as a 128-wide launch; the k2 / k4 layers are timed as plain 2- and
4-tap convolutions."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vtoonify_b200 import _lib, ops  # noqa: E402

B = 4
MODES = (0, 1, 2)
# (Cin, Cout, taps, stride, H, W): the input map of each layer
LAYERS = [(64, 32, "up", 1, 1152, 2048), (256, 128, 9, 1, 576, 1024), (128, 128, 9, 1, 576, 1024), (32, 128, 9, 1, 576, 1024),
          (256, 128, 2, 1, 288, 512), (256, 128, 4, 1, 288, 512), (256, 128, 1, 1, 288, 512), (512, 512, 9, 1, 72, 128),
          (128, 256, 9, 2, 576, 1024), (256, 512, 9, 2, 288, 512), (512, 512, 9, 2, 144, 256)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi not available"
    return q or torch.cuda.get_device_name()


def taps_of(n):
    return {9: ops.conv_taps(3, 1), 4: [(0, 0, 0), (0, 1, 1), (1, 0, 2), (1, 1, 3)], 2: [(0, 0, 0), (0, 1, 1)], 1: [(0, 0, 0)]}[n]


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    dev = torch.device("cuda:0")
    lib = _lib.load()
    ops.set_precision("bf16x3")
    g = torch.Generator().manual_seed(0)
    print(f"card: {card()}")
    print(f"{'layer':28s} {'tc_pingpong 0':>22s} {'1':>10s} {'change':>7s} {'2':>10s} {'change':>7s}  identical")
    tot = {m: 0.0 for m in MODES}
    with torch.no_grad():
        for cin, cout, taps, stride, H, W in LAYERS:
            x = ops.to_nhwc(torch.randn((B, cin, H, W), generator=g).to(dev), round_tf32=False)
            bias = (torch.randn(cout, generator=g) * 0.2).to(dev)
            if taps == "up":
                k4 = torch.tensor([1., 3., 3., 1.])
                k4 = (k4[:, None] * k4[None, :] / 64 * 4).to(dev)
                wt = (torch.randn((cout, cin, 3, 3), generator=g) / (3 * cin ** 0.5)).to(dev)
                w = ops.fold_upconv_weights(ops.prep_weights(wt, cin_pad=cin, round_tf32=False), k4)
                noise = torch.randn((B, 1, 2 * H, 2 * W), generator=g).to(dev)

                def run():
                    return ops.conv_up2_folded_nhwc(x, w, bias=bias, noise=noise, noise_w=torch.tensor([0.3], device=dev),
                                                    act=ops.ACT_LRELU, gain=2 ** 0.5)
                label, issued = f"{cin}->{cout}x4up k9 s1 {H}x{W}", 12 * 2.0 * B * H * W * cin * cout * 9
            else:
                tp = taps_of(taps)
                k = 3 if taps == 9 else 2 if taps in (2, 4) else 1
                wt = (torch.randn((cout, cin, k, k), generator=g) / (k * cin ** 0.5)).to(dev)
                w = ops.prep_weights(wt, cin_pad=cin, round_tf32=False)
                if taps == 2:
                    w = w[:, :2].contiguous()
                Ho, Wo = (H, W) if stride == 1 else ((H - 1) // 2 + 1, (W - 1) // 2 + 1)

                def run():
                    return ops.conv2d_nhwc([x], w, tp, stride, Ho, Wo, bias=bias, act=ops.ACT_LRELU, gain=2 ** 0.5)
                label, issued = f"{cin}->{cout} k{taps} s{stride} {H}x{W}", 3 * 2.0 * B * Ho * Wo * cin * cout * taps
            outs, times = {}, {m: [] for m in MODES}
            for mode in MODES:
                lib.vt_set_option(b"tc_pingpong", mode)
                outs[mode] = run()
            for _ in range(3):
                for mode in MODES:
                    lib.vt_set_option(b"tc_pingpong", mode)
                    run(); torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        run()
                    e1.record(); torch.cuda.synchronize()
                    times[mode].append(e0.elapsed_time(e1) / reps)
            lib.vt_set_option(b"tc_pingpong", 1)
            t = {m: min(times[m]) for m in MODES}
            for m in MODES:
                tot[m] += t[m]
            same = all(torch.equal(outs[m], outs[0]) for m in MODES)
            print(f"{label:28s} {t[0]:7.3f} ms {issued / t[0] * 1e-9:5.0f} TF/s {t[1]:7.3f} ms {(t[1] / t[0] - 1) * 100:+6.1f}% "
                  f"{t[2]:7.3f} ms {(t[2] / t[0] - 1) * 100:+6.1f}%  {'yes' if same else 'NO'}")
            del outs, x, w
    print(f"{'sum (one call each)':28s} {tot[0]:7.3f} ms {'':10s} {tot[1]:7.3f} ms {(tot[1] / tot[0] - 1) * 100:+6.1f}% "
          f"{tot[2]:7.3f} ms {(tot[2] / tot[0] - 1) * 100:+6.1f}%")


if __name__ == "__main__":
    main()
