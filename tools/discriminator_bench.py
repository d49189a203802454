"""Times the ConditionalDiscriminator steps of VToonify training at batch 8, 256^2, channel multiplier 2, use_condition=True:
  * D step: d_logistic_loss over a fake and a real pass, backward into the parameters (the inputs need no gradient);
  * G-step share: forward + input gradient with the parameters frozen.
Arms, alternated per repetition: the library in bf16x3 and in tf32; the float64 restatement's statements (tests/oracle_discriminator.py)
in fp32 on cuDNN with TF32 on and off; the same statements on ``vtoonify_b200.op`` (integration level (b)).  Fresh inputs per step.
Reports ms per step (forward / backward split), kernel launches of the library arms, peak memory, and, from a separate
torch.profiler run, the weight-gradient kernel's share of the library D step.  Writes one JSON file to --out.

    python tools/discriminator_bench.py --steps 10 --warmup 3 --out /tmp/discriminator_bench.json
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.oracle_discriminator import forward as restated  # noqa: E402
from vtoonify_b200 import _lib, ops  # noqa: E402
from vtoonify_b200.vtoonify import ConditionalDiscriminator  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402

B, SIZE, STYLES = 8, 256, 3


def inputs(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((B, 3, SIZE, SIZE), generator=g).cuda(), torch.rand((B, 1), generator=g).cuda(),
            torch.randint(0, STYLES, (B,), generator=g).cuda())


class LibArm:
    def __init__(self, D, precision):
        self.D, self.precision = D, precision

    def params(self):
        return list(self.D.parameters())

    def forward(self, x, d, s):
        ops.set_precision(self.precision)
        return self.D(x, d, s)


class RestatedArm:
    def __init__(self, sd, kind):
        self.p = {k: v.cuda().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
        self.kind = kind

    def params(self):
        return [v for v in self.p.values() if v.is_floating_point()]

    def forward(self, x, d, s):
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = self.kind == "cudnn_tf32"
        if self.kind == "level_b":
            from vtoonify_b200.op import conv2d_gradfix, fused_leaky_relu, upfirdn2d
            return restated(self.p, x, d, s, conv2d=conv2d_gradfix.conv2d, upfirdn2d=upfirdn2d, flrelu=fused_leaky_relu)
        return restated(self.p, x, d, s)


def timed(fn):
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e[0].record()
    out = fn(e)
    e[2].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), out


def d_step(arm, seed):
    (xf, df, sf), (xr, dr, sr) = inputs(seed), inputs(seed + 1)
    for p in arm.params():
        p.grad = None

    def run(e):
        with torch.enable_grad():
            loss = F.softplus(-arm.forward(xr, dr, sr)).mean() + F.softplus(arm.forward(xf, df, sf)).mean()
            e[1].record()
            loss.backward()
    return timed(run)


def g_step(arm, seed):
    x, d, s = inputs(seed)
    x.requires_grad_()
    params = arm.params()
    for p in params:
        p.requires_grad_(False)

    def run(e):
        with torch.enable_grad():
            loss = F.softplus(-arm.forward(x, d, s)).mean()
            e[1].record()
            loss.backward()
    try:
        return timed(run)
    finally:
        for p in params:
            p.requires_grad_(True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("discriminator_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    D = ConditionalDiscriminator(SIZE, use_condition=True, style_num=STYLES)
    sd = det_state_dict(D, seed=0)
    D.load_state_dict(sd, strict=True)
    D.cuda()
    arms = {"lib_bf16x3": LibArm(D, "bf16x3"), "lib_tf32": LibArm(D, "tf32"), "cudnn_fp32": RestatedArm(sd, "cudnn_fp32"),
            "cudnn_tf32": RestatedArm(sd, "cudnn_tf32"), "level_b": RestatedArm(sd, "level_b")}
    res = {name: {"d_step": [], "g_step": []} for name in arms}
    peak = {}
    launches = {}
    for step in range(args.warmup + args.steps):
        for name, arm in arms.items():
            for kind, fn in (("d_step", d_step), ("g_step", g_step)):
                torch.cuda.reset_peak_memory_stats()
                n0 = _lib.launch_count()
                f, b, _ = fn(arm, 1000 * step + 7)
                if step >= args.warmup:
                    res[name][kind].append((f, b))
                    peak[f"{name}/{kind}"] = torch.cuda.max_memory_allocated() / 2 ** 30
                    if name.startswith("lib"):
                        launches[f"{name}/{kind}"] = _lib.launch_count() - n0
    ops.set_precision(ops.DEFAULT_PRECISION)
    summary = {}
    for name, kinds in res.items():
        for kind, v in kinds.items():
            fw = sorted(t[0] for t in v)[len(v) // 2]
            bw = sorted(t[1] for t in v)[len(v) // 2]
            tot = sorted(t[0] + t[1] for t in v)
            summary[f"{name}/{kind}"] = {"ms_median": tot[len(tot) // 2], "ms_min": tot[0], "fwd_ms_median": fw, "bwd_ms_median": bw,
                                         "peak_GiB": round(peak[f"{name}/{kind}"], 2), "launches": launches.get(f"{name}/{kind}")}
    # weight-gradient share of the library D step (bf16x3), in a separate profiled run
    from torch.profiler import ProfilerActivity, profile
    ops.set_precision("bf16x3")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        d_step(arms["lib_bf16x3"], 99)
    ops.set_precision(ops.DEFAULT_PRECISION)
    tot = wg = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if ev.key.startswith(("cudaLaunch", "cudaMemcpy", "cudaStream", "cudaDevice", "cudaEvent")):
            continue
        tot += t
        if "wgrad" in ev.key:
            wg += t
    out = {"gpu": gpu, "batch": B, "size": SIZE, "steps": args.steps, "results": summary,
           "wgrad_share_of_lib_d_step": round(wg / tot, 3) if tot else None}
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
