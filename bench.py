#!/usr/bin/env python
"""bench.py — frames/s of the VToonify per-frame synthesis hot path on H100 (BASELINE.json metric).

    python bench.py --gpus N --steps K --warmup W            # this framework (N>1: launched by torchrun)
    python bench.py --impl reference --gpus N --steps K ...  # the reference's CPU path (oracle port) on the host cores
    python bench.py --impl cudnn ...                         # the same graph on PyTorch/cuDNN CUDA kernels ("reference CUDA" row)
    python bench.py --config generator|vtoonify_t|video ...  # BASELINE configs[2] / [4] / [3]

Default (configs[1]): a "step" is one ``VToonify.forward`` (+ clamp) over one batch of 4 synthetic 576x1024 frames per GPU
(VToonify-D, deterministic random-init weights).
  N = 1   ``value`` = frames/s with the inputs resident in HBM; ``e2e`` = the same through ``FramePipeline`` with HOST buffers
          (pinned H2D of the fp32 inputs, D2H of the uint8 frames inside the timed region); ``e2e_u8`` = uint8 RGB frames on the
          wire in both directions with the face parsing (BiSeNet) computed on the device.
  N > 1   the reference's single-decoder layout (style_transfer.py:99-183): rank 0 owns the clip.  Every step rank 0 scatters one
          input batch per rank over NCCL, every rank synthesises its batch, the uint8 frames are gathered back to rank 0 — all
          inside the timed region, double-buffered (``ShardedFrameLoop``).  ``value``: the inputs start in rank 0's HBM and the
          frames end there; ``e2e``: they start and end in rank 0's pinned host memory.
Timing: CUDA events on the launching stream, barrier + synchronize on both sides, max over ranks.
--dump-outputs DIR (single GPU): after the timed steps, the last timed step's output is written to DIR/<name>.npy (float32; a fixed,
seeded sample of it when it is larger than the budget) so that two builds can be compared output for output on identical inputs.
"""
import argparse
import json
import math
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# BASELINE.md §2: algorithmic work per unit (FLOP = 2*MAC over every conv, bytes = fp32 ideal-fusion traffic)
CONFIGS = {
    "vtoonify_d": dict(kind="vtoonify", backbone="dualstylegan", H=576, W=1024, B=4, flop_per_px=6.97e6, bytes_per_px=28.3e3,
                       metric="frames/sec at 576x1024", unit="frames/s", name="BASELINE configs[1]"),
    "vtoonify_t": dict(kind="vtoonify", backbone="toonify", H=720, W=1280, B=2, flop_per_px=6.08e6, bytes_per_px=25.7e3,
                       metric="frames/sec at 720x1280 (VToonify-T)", unit="frames/s", name="BASELINE configs[4]"),
    "generator": dict(kind="generator", size=1024, B=8, flop_per_unit=148.5e9, bytes_per_unit=1.20e9,
                      metric="images/sec, StyleGAN2 Generator(1024) synthesis", unit="images/s", name="BASELINE configs[2]"),
    "video": dict(kind="vtoonify", backbone="dualstylegan", H=576, W=1024, B=4, flop_per_px=6.97e6, bytes_per_px=28.3e3,
                  frames=900, metric="frames/sec at 576x1024 (900-frame clip, rank-0 I/O)", unit="frames/s",
                  name="BASELINE configs[3]"),
}


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"],
                "bf16_tflops_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]), "source": "measured"}
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "source": "H100 SXM data sheet (dense, 700 W)"}


class ClockSampler(threading.Thread):
    """Samples SM clock / throttle reasons during the timed region (pynvml; nvidia-smi fallback)."""

    def __init__(self, index=0, period=0.2):
        super().__init__(daemon=True)
        self.index, self.period = index, period
        self.samples, self.reasons, self.max_mhz = [], set(), None
        self._halt = threading.Event()

    def run(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            h = pynvml.nvmlDeviceGetHandleByIndex(self.index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
            names = {"hw_slowdown": 0x8, "sw_power_cap": 0x4, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20,
                     "hw_power_brake": 0x80}
            while not self._halt.is_set():
                self.samples.append(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM))
                r = pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                for n, bit in names.items():
                    if r & bit:
                        self.reasons.add(n)
                time.sleep(self.period)
        except Exception as e:  # pragma: no cover
            self.reasons.add(f"sampler_error:{type(e).__name__}")

    def stop(self):
        self._halt.set()
        self.join(timeout=2)
        s = sorted(self.samples)
        return {"sm_mhz": (s[len(s) // 2] if s else None), "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                "samples": len(s)}


def usable_cores():
    """Host cores this process may really use: min(affinity, cgroup cpu.max quota); os.cpu_count() alone over-reports
    inside a quota-limited container and 128 oversubscribed threads are slower than 8."""
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:
        pass
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(per) + 0.999)))
    except Exception:
        pass
    return max(1, n)


def cpu_model():
    try:
        for line in open("/proc/cpuinfo"):
            if line.lower().startswith("model name"):
                return line.split(":", 1)[1].strip()
    except Exception:
        pass
    import platform
    return platform.processor() or "unknown"


# ----------------------------------------------------------------------------------------------------
# CPU legs (the only place bench.py executes oracle/): the reference's op_cpu path restated in oracle/vt_oracle.py
# ----------------------------------------------------------------------------------------------------
def _cpu_setup(cfg):
    import torch
    from oracle import vt_oracle as O
    from vtoonify_b200.weights import det_inputs, det_state_dict
    if cfg["kind"] == "generator":
        from vtoonify_b200.stylegan import Generator     # module tree only gives key names/shapes; no kernel is called
        g = Generator(cfg["size"], 512, 8)
        sd = det_state_dict(g, seed=3)
        noises = [sd[f"noises.noise_{i}"] for i in range(g.num_layers)]
        lat = torch.randn((1, g.n_latent, 512), generator=torch.Generator().manual_seed(7))
        return (lambda: O.generator_forward(sd, lat, noises)), None
    from vtoonify_b200.vtoonify import VToonify
    sd = det_state_dict(VToonify(backbone=cfg["backbone"]), seed=0)

    def make(h, w):
        x, s = det_inputs(1, h, w, seed=0)
        return lambda: O.vtoonify_forward(sd, x, s, 0.5, cfg["backbone"])
    return make(cfg["H"], cfg["W"]), make


def _pick_threads(make_small, threads=None):
    """the thread count (<= usable cores) that is actually fastest on a small frame"""
    import torch
    cores = usable_cores()
    if threads or make_small is None:
        return threads or cores
    cands = sorted({cores, min(cores, 64), min(cores, 32), min(cores, 16), min(cores, 8)}, reverse=True)
    small = make_small(144, 256)
    best = None
    for th in cands:
        torch.set_num_threads(th)
        small()                                               # warm the thread pool / primitive cache
        t0 = time.time(); small(); dt = time.time() - t0
        if best is None or dt < best[1]:
            best = (th, dt)
    return best[0]


def cpu_reference(cfg, steps, warmup, threads=None, budget_s=None):
    """Time the oracle port of the reference CPU path (model/stylegan/op_cpu + F.conv2d) on the host cores: every timed step is
    ONE full-size unit of the configuration (a 576x1024 frame for configs[1]; ~25 s on 16 cores), B = 1.

    ``budget_s`` (the reference arm): the warm-up frame is timed; only if ``steps`` full-size frames would not fit the budget on
    this host (slow or busy cores) the timed steps fall back to the largest frame of the same aspect that does, and the value is
    scaled by pixels - stated in ``sample``.  On the pool's 16-core hosts 20 full frames take ~8 min and fit."""
    import torch
    scale_note, px_scale = "", 1.0
    with torch.no_grad():
        full, make = _cpu_setup(cfg)
        threads = _pick_threads(make, threads)
        torch.set_num_threads(threads)
        if make is not None:
            make(72, 128)()                                   # thread pool / oneDNN primitive cache
        t_w = None
        for _ in range(warmup):
            t0 = time.time(); full(); t_w = time.time() - t0
        if budget_s is not None and t_w is not None and make is not None and steps * t_w > budget_s:
            for num, den in ((3, 4), (1, 2), (3, 8), (1, 4)):            # same aspect, multiples of 8 pixels
                h, w = cfg["H"] * num // den // 8 * 8, cfg["W"] * num // den // 8 * 8
                px_scale = (h * w) / float(cfg["H"] * cfg["W"])
                if steps * t_w * px_scale <= budget_s or (num, den) == (1, 4):
                    break
            full = make(h, w)
            scale_note = (f"; {steps} full-size frames would take {steps * t_w:.0f} s on this host (> {budget_s:.0f} s budget): timed on "
                          f"{h}x{w} frames ({px_scale:.3f} of the pixels) and scaled by pixels")
        t0 = time.time()
        for _ in range(steps):
            full()
        dt = (time.time() - t0) / max(1, steps) / px_scale
    ups = 1.0 / dt
    what = (f"Generator({cfg['size']}) image" if cfg["kind"] == "generator" else f"VToonify-{'D' if cfg['backbone'] == 'dualstylegan' else 'T'} "
            f"{cfg['H']}x{cfg['W']} frame")
    return ups, dt, {"kind": "port", "cores": threads, "value": ups, "unit": cfg["unit"], "cpu_model": cpu_model(),
                     "sample": f"oracle port of the reference op_cpu path, one full-size {what} per step (B=1), {dt:.2f} s/step, "
                               f"torch CPU fp32 {torch.__version__}, {threads} threads on {cpu_model()}{scale_note}"}


def workload_config(cfg, args, world):
    if cfg["kind"] == "generator":
        return {"workload": f"StyleGAN2 Generator({cfg['size']}, 512, 8, 2) synthesis from W+ latents, fixed noise, batch {args.batch} per "
                            f"GPU per step ({cfg['name']})", "batch_per_gpu": args.batch, "units_per_step": world * args.batch,
                "weights": "deterministic random-init (vtoonify_b200/weights.py)",
                "l2": "every activation of the 256^2..1024^2 levels exceeds the 50 MB L2; no flush needed"}
    H, W, B = args.height, args.width, args.batch
    return {"workload": f"VToonify-{'D' if cfg['backbone'] == 'dualstylegan' else 'T'} forward+clamp, "
                        f"{H}x{W} input frames -> {4 * H}x{4 * W}, batch {B} per GPU per step ({cfg['name']})",
            "backbone": cfg["backbone"], "batch_per_gpu": B, "frames_per_step": world * B,
            "weights": "deterministic random-init (vtoonify_b200/weights.py)",
            "l2": f"inputs ({B * 22 * H * W * 4 / 1e6:.0f} MB) and every activation exceed the 50 MB L2; no flush needed"}


def run_reference(args, cfg, rank, world):
    if rank != 0:
        return
    # one small-frame pass is the warm-up of the CPU arm (thread pool, primitive cache): repeating the 25 s frame W times would
    # only burn minutes; the K timed steps are full-size frames
    ups, dt, cb = cpu_reference(cfg, args.steps, 1 if args.warmup > 0 else 0, budget_s=args.ref_budget)
    conf = workload_config(cfg, args, world)       # the same workload description as the GPU arm's (the CPU runs it one unit at a time)
    line = {"impl": "reference", "metric": cfg["metric"], "value": ups, "unit": cfg["unit"], "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": dt * 1e3, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": conf,
            "cpu_baseline": cb,
            "e2e": {"value": ups, "unit": cfg["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    emit(json.dumps(line))


# ----------------------------------------------------------------------------------------------------
# "reference CUDA" row (BASELINE.md §3): the same graph on PyTorch's own CUDA kernels (cuDNN convolutions)
# ----------------------------------------------------------------------------------------------------
def run_cudnn(args, cfg, rank, world):
    """The oracle restatement executed on CUDA tensors = what the reference does on a GPU (F.conv2d / F.conv_transpose2d ->
    cuDNN, grouped-conv-free algebra, torch elementwise ops for blur / bias / activation).  None of this repo's kernels run."""
    if rank != 0:
        return
    import torch
    from oracle import vt_oracle as O
    from vtoonify_b200.weights import det_inputs, det_state_dict
    dev = torch.device("cuda", 0)
    res = {}
    # the reference's own CUDA kernels for upfirdn2d / fused_bias_act when oracle/_ref holds them (compiled unmodified from
    # /root/reference by oracle/build_ref.py); otherwise the oracle's pure-torch restatements run on the GPU
    from oracle import build_ref
    ref_ops = build_ref.load_ops()
    if ref_ops is not None:
        up_op, fused_op = ref_ops

        def upfirdn2d_ref(x, kernel, up=1, down=1, pad=(0, 0)):           # model/stylegan/op/upfirdn2d.py:89-125, 149-165
            up_x, up_y = (up, up) if isinstance(up, int) else up
            down_x, down_y = (down, down) if isinstance(down, int) else down
            if len(pad) == 2:
                pad = (pad[0], pad[1], pad[0], pad[1])
            _, C, H, W = x.shape
            out = up_op.upfirdn2d(x.reshape(-1, H, W, 1), kernel, up_x, up_y, down_x, down_y, pad[0], pad[1], pad[2], pad[3])
            return out.view(-1, C, out.shape[1], out.shape[2])

        def fused_lrelu_ref(x, bias=None, negative_slope=0.2, scale=2 ** 0.5):   # model/stylegan/op/fused_act.py:56-71
            empty = x.new_empty(0)
            return fused_op.fused_bias_act(x, empty if bias is None else bias, empty, 3, 0, negative_slope, scale)
        O.upfirdn2d, O.fused_leaky_relu = upfirdn2d_ref, fused_lrelu_ref
    with torch.no_grad():
        if cfg["kind"] == "generator":
            from vtoonify_b200.stylegan import Generator
            g = Generator(cfg["size"], 512, 8)
            sd = {k: v.to(dev) for k, v in det_state_dict(g, seed=3).items()}
            noises = [sd[f"noises.noise_{i}"] for i in range(g.num_layers)]
            lat = torch.randn((args.batch, g.n_latent, 512), generator=torch.Generator().manual_seed(7)).to(dev)
            step = lambda: O.generator_forward(sd, lat, noises)
            units = args.batch
        else:
            from vtoonify_b200.vtoonify import VToonify
            sd = {k: v.to(dev) for k, v in det_state_dict(VToonify(backbone=cfg["backbone"]), seed=0).items()}
            x, s = det_inputs(args.batch, args.height, args.width, seed=0)
            x, s = x.to(dev), s.to(dev)
            step = lambda: O.vtoonify_forward(sd, x, s, 0.5, cfg["backbone"]).clamp_(-1, 1)
            units = args.batch
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            for _ in range(max(1, args.warmup)):
                step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            res[tf32] = e0.elapsed_time(e1) / args.steps
    line = {"impl": "cudnn", "metric": cfg["metric"], "value": units / (res[True] * 1e-3), "unit": cfg["unit"], "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": res[True], "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "tf32 (torch default: cudnn.allow_tf32=True)", "data": "synthetic",
            "config": workload_config(cfg, args, 1),
            "fp32": {"value": units / (res[False] * 1e-3), "ms_per_step": res[False], "note": "cudnn.allow_tf32=False"},
            "custom_ops": ("the reference's own upfirdn2d / fused_bias_act CUDA kernels (oracle/_ref, compiled unmodified for sm_90a)"
                           if ref_ops is not None else "pure-torch restatements of upfirdn2d / fused_bias_act (oracle/_ref not built)"),
            "note": f"oracle restatement of the reference graph on torch {torch.__version__} CUDA kernels (cuDNN {torch.backends.cudnn.version()}); "
                    "test infrastructure timed as a baseline, none of this repo's kernels on the path"}
    emit(json.dumps(line))


# ----------------------------------------------------------------------------------------------------
def _roofline(prof, steps, ms, precision, peaks, cfg, units_per_rank_step, extra_layers=False):
    """Aggregate roofline of the dominant kernel (conv_tc_kernel) over its launches in the timed region of rank 0."""
    tc_ms = sum(a.elapsed_time(b) for a, b, *_ in prof)
    tc_flops = sum(p[2] for p in prof)
    tc_issued = sum(p[5] for p in prof)
    tc_bytes = sum(p[3] for p in prof)
    per = {}
    for a, b, f, nb, label, issued in prof:
        d = per.setdefault(label, [0.0, 0.0, 0, 0.0, 0.0])
        d[0] += a.elapsed_time(b); d[1] += f; d[2] += 1; d[3] += nb; d[4] += issued
    peak = peaks["bf16_tflops_sustained"]
    achieved = tc_flops / (tc_ms * 1e-3) / 1e12 if tc_ms > 0 else 0.0
    issued = tc_issued / (tc_ms * 1e-3) / 1e12 if tc_ms > 0 else 0.0

    def layer(k, v):
        t = v[0] * 1e-3
        return {"layer": k, "ms_per_step": v[0] / steps, "launches_per_step": v[2] / steps,
                "tflops_algorithmic": v[1] / t / 1e12, "tflops_issued_bf16": v[4] / t / 1e12,
                "frac_of_bf16_peak_algorithmic": v[1] / t / 1e12 / peak, "frac_of_bf16_peak_issued": v[4] / t / 1e12 / peak,
                "hbm_gbs_algorithmic": v[3] / t / 1e9, "frac_of_hbm_peak": v[3] / t / 1e9 / peaks["hbm_gbs"]}
    ordered = sorted(per.items(), key=lambda kv: -kv[1][0])
    top = [layer(k, v) for k, v in (ordered if extra_layers else ordered[:8])]
    products = {"bf16x3": 3, "tf32": 1, "fp32": 1}[precision]
    roof = {"bound": "tensor",
            "kernel": ("conv_tc_kernel (wgmma bf16, fp32 operands split into bf16 hi+lo, 3 products, implicit-GEMM conv)"
                       if precision == "bf16x3" else "conv_tc_kernel (wgmma tf32 implicit-GEMM conv)"),
            "achieved": achieved, "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak,
            "frac_algorithmic": achieved / peak, "frac_issued": issued / peak,
            "peak_note": f"{peaks['source']} dense bf16 throughput; "
                         f"achieved counts ALGORITHMIC conv flops (2*MAC); frac_issued counts the bf16 MMA flops actually issued "
                         f"({products} products per algorithmic product, x4 for the folded up-convolutions)",
            "launches": len(prof), "kernel_ms_per_step": tc_ms / steps, "share_of_step": tc_ms / ms if ms > 0 else None,
            "hbm": {"algorithmic_gbs": tc_bytes / (tc_ms * 1e-3) / 1e9 if tc_ms > 0 else 0.0, "peak_gbs": peaks["hbm_gbs"],
                    "frac": tc_bytes / (tc_ms * 1e-3) / 1e9 / peaks["hbm_gbs"] if tc_ms > 0 else 0.0,
                    "note": "algorithmic bytes (inputs + outputs + weights of every conv launch, fp32) / conv kernel time; per layer in top_layers"},
            "top_layers": top}
    if cfg["kind"] == "vtoonify":
        flop_unit = cfg["flop_per_px"] * cfg["H"] * cfg["W"]
        bytes_unit = cfg["bytes_per_px"] * cfg["H"] * cfg["W"]
    else:
        flop_unit, bytes_unit = cfg["flop_per_unit"], cfg["bytes_per_unit"]
    t = ms * 1e-3 / steps
    roof["whole_step"] = {"algorithmic_tflop_per_unit": flop_unit / 1e12,
                          "achieved_tflops": flop_unit * units_per_rank_step / t / 1e12,
                          "frac_of_bf16_peak": flop_unit * units_per_rank_step / t / 1e12 / peak,
                          "hbm_floor_gbs_needed": bytes_unit * units_per_rank_step / t / 1e9}
    return roof, per


def run_ours(args, cfg, rank, world, local_rank):
    import torch
    import torch.distributed as dist
    from vtoonify_b200 import _lib, ops
    from vtoonify_b200.frame_loop import FramePipeline, ShardedFrameLoop
    from vtoonify_b200.weights import det_inputs, det_state_dict

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    B = args.batch
    ops.set_precision(args.precision)
    peaks = load_peaks()
    is_gen = cfg["kind"] == "generator"
    video = args.config == "video"

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    with torch.no_grad():
        pnet = None
        if is_gen:
            from vtoonify_b200.stylegan import Generator
            model = Generator(cfg["size"], 512, 8).eval()
            model.load_state_dict(det_state_dict(model, seed=3), strict=True)
            model.to(dev)
            latent = torch.randn((B, model.n_latent, 512), generator=torch.Generator().manual_seed(7 + rank)).to(dev)
            step = lambda: model([latent], input_is_latent=True, randomize_noise=False)[0]
        else:
            from vtoonify_b200.vtoonify import VToonify
            H, W = args.height, args.width
            model = VToonify(backbone=cfg["backbone"]).eval()
            model.load_state_dict(det_state_dict(model, seed=0), strict=True)
            model.to(dev)
            n_in = world if rank == 0 else 1                     # rank 0 owns the clip: one distinct batch per rank and step
            hosts = [det_inputs(B, H, W, seed=rank + i)[0].pin_memory() for i in range(n_in)]
            style_host = det_inputs(B, H, W, seed=0)[1]
            x = hosts[0].to(dev)
            style = style_host.to(dev)
            step = lambda: model(x, style, d_s=0.5).clamp_(-1, 1)          # style_transfer.py:176-177
            if not args.no_u8:
                from vtoonify_b200.bisenet import BiSeNet
                pnet = BiSeNet(19).eval()
                pnet.load_state_dict(det_state_dict(pnet, seed=21), strict=True)
                pnet.to(dev)
            pipe = FramePipeline(model, style_host[:1], d_s=0.5, device=dev, parsing_net=pnet, copy=False, ring=3, graph=args.graph)

        prof = []
        sampler = None
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        scatter_b = gather_b = 0
        steps = args.steps
        if world == 1 or is_gen:
            # ---- device-resident inputs, no collective (N = 1; generator: independent replicas)
            for _ in range(args.warmup):
                step()
            barrier()
            sampler = ClockSampler(local_rank) if rank == 0 else None
            if sampler:
                sampler.start()
            ops.set_tc_profile(prof)
            n0 = _lib.launch_count()
            last = None
            e0.record()
            for _ in range(steps):
                last = step()
            e1.record()
            barrier()
            if args.dump_outputs and rank == 0 and last is not None:
                dump_outputs(args.dump_outputs, {"images" if is_gen else "frames": last})
        else:
            # ---- rank-0 clip: NCCL scatter -> forward -> NCCL gather of uint8 frames, inputs / results in rank 0's HBM
            dev_in = [h.to(dev) for h in hosts] if rank == 0 else None
            loop = ShardedFrameLoop(pipe.synthesize, (B, 22, H, W), torch.float32, (B, 4 * H, 4 * W, 3), torch.uint8, dev)
            stage = (lambda i: dev_in[i % world]) if rank == 0 else None
            sink = (lambda i, buf, ready: None) if rank == 0 else None
            loop.run(args.warmup * world, stage=stage, sink=sink)
            barrier()
            sampler = ClockSampler(local_rank) if rank == 0 else None
            if sampler:
                sampler.start()
            ops.set_tc_profile(prof)
            n0 = _lib.launch_count()
            loop.scatter_bytes = loop.gather_bytes = 0
            e0.record()
            loop.run(steps * world, stage=stage, sink=sink)
            e1.record()
            barrier()
            scatter_b, gather_b = loop.scatter_bytes, loop.gather_bytes
        launches = _lib.launch_count() - n0
        ops.set_tc_profile(None)
        ms = e0.elapsed_time(e1)
        clocks = sampler.stop() if sampler else None

        # ---- e2e through the public frame-loop API with host buffers
        e2e = e2e_u8 = None
        if not is_gen:
            def timed_pipeline(items_for, in_shape, in_dtype, fn):
                """returns (ms, h2d bytes/step, d2h bytes/step) of `steps` steps through host buffers"""
                if world == 1:
                    items = items_for(1)
                    for _ in pipe.run([items[0]] * max(1, min(2, args.warmup))):
                        pass
                    barrier()
                    pipe.h2d_bytes = pipe.d2h_bytes = 0
                    t0 = time.perf_counter()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in pipe.run([items[0]] * steps):
                        pass
                    b.record()
                    barrier()
                    return max(a.elapsed_time(b), (time.perf_counter() - t0) * 1e3), pipe.h2d_bytes // steps, pipe.d2h_bytes // steps
                items = items_for(world) if rank == 0 else None
                lp = ShardedFrameLoop(fn, in_shape, in_dtype, (B, 4 * H, 4 * W, 3), torch.uint8, dev)
                d2h = torch.cuda.Stream(dev)
                outs = [torch.empty((B, 4 * H, 4 * W, 3), dtype=torch.uint8).pin_memory() for _ in range(3 * world)] if rank == 0 else None
                cnt = {"h2d": 0, "d2h": 0}

                def stage(i):
                    cnt["h2d"] += items[i % world].numel() * items[i % world].element_size()
                    return items[i % world].to(dev, non_blocking=True)

                def sink(i, buf, ready):
                    with torch.cuda.stream(d2h):
                        ready()
                        outs[i % len(outs)].copy_(buf, non_blocking=True)
                        ev = torch.cuda.Event()
                        ev.record(d2h)
                    cnt["d2h"] += buf.numel()
                    return ev
                lp.run(max(1, min(2, args.warmup)) * world, stage=stage if rank == 0 else None, sink=sink if rank == 0 else None)
                barrier()
                cnt["h2d"] = cnt["d2h"] = 0
                t0 = time.perf_counter()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                lp.run(steps * world, stage=stage if rank == 0 else None, sink=sink if rank == 0 else None)
                d2h.synchronize()
                b.record()
                barrier()
                return max(a.elapsed_time(b), (time.perf_counter() - t0) * 1e3), cnt["h2d"] // steps, cnt["d2h"] // steps

            e2e = timed_pipeline(lambda n: hosts[:n], (B, 22, H, W), torch.float32, pipe.process)
            if pnet is not None:
                g = torch.Generator().manual_seed(99 + rank)
                frames_u8 = [torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8).pin_memory() for _ in range(world if rank == 0 else 1)]
                e2e_u8 = timed_pipeline(lambda n: frames_u8[:n], (B, H, W, 3), torch.uint8, pipe.process)

    vals = [ms, e2e[0] if e2e else 0.0, e2e_u8[0] if e2e_u8 else 0.0]
    t = torch.tensor(vals, device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, e2e_ms, e2e_u8_ms = float(t[0]), float(t[1]), float(t[2])
    if rank != 0:
        return
    units = world * B * steps
    ups = units / (ms * 1e-3)
    roofline, per = _roofline(prof, steps, ms, args.precision, peaks, cfg, B, extra_layers=is_gen)
    if args.dump_layers:
        with open(args.dump_layers, "w") as f:
            for k, v in sorted(per.items(), key=lambda kv: -kv[1][0]):
                f.write(f"{v[0] / steps:8.3f} ms  x{v[2] / steps:5.1f}  {v[1] / (v[0] * 1e-3) / 1e12:6.1f} TF/s alg  "
                        f"{v[4] / (v[0] * 1e-3) / 1e12:7.1f} TF/s issued  {v[3] / (v[0] * 1e-3) / 1e9:7.0f} GB/s alg  {k}\n")
    conf = workload_config(cfg, args, world)
    if world == 1 or is_gen:
        par = {"layout": f"{world} independent replica(s), no collective" if is_gen else "single GPU, inputs resident in HBM"}
    else:
        par = {"layout": f"rank-0 clip: per step NCCL scatter of {world} fp32 input batches from rank 0's HBM, forward on every rank, NCCL "
                         f"gather of the uint8 frames to rank 0, all inside the timed region (double-buffered, frame_loop.ShardedFrameLoop)",
               "nccl_bytes_per_step": {"scatter": scatter_b // steps, "gather": gather_b // steps}}
    line = {"metric": cfg["metric"], "value": ups, "unit": cfg["unit"], "n_gpus": world, "steps": steps,
            "warmup": args.warmup, "ms_per_step": ms / steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None,
            "dtype": {"tf32": "tf32", "bf16x3": "bf16x3 (fp32 operands split into bf16 hi+lo, 3 tensor-core products, fp32 accumulate)",
                      "fp32": "f32"}[args.precision], "data": "synthetic", "config": conf,
            "parallelism": par, "gpu_launches": int(launches), "clocks": clocks, "roofline": roofline}
    if e2e:
        line["e2e"] = {"value": units / (e2e_ms * 1e-3), "unit": cfg["unit"], "h2d_bytes_per_step": int(e2e[1]),
                       "d2h_bytes_per_step": int(e2e[2]), "ms_per_step": e2e_ms / steps,
                       "cuda_graph": bool(args.graph),
                       "api": ("vtoonify_b200.frame_loop.FramePipeline.run" if world == 1 else "vtoonify_b200.frame_loop.ShardedFrameLoop.run")
                              + " (pinned fp32 [B,22,H,W] inputs H2D on rank 0, clamp + uint8 BGR frames D2H on rank 0)"}
    if e2e_u8:
        line["e2e_u8"] = {"value": units / (e2e_u8_ms * 1e-3), "unit": cfg["unit"], "h2d_bytes_per_step": int(e2e_u8[1]),
                          "d2h_bytes_per_step": int(e2e_u8[2]), "ms_per_step": e2e_u8_ms / steps,
                          "api": "same loop with uint8 RGB frames on the wire and the BiSeNet face parsing (style_transfer.py:171-174) "
                                 "computed on every rank's device (more work per frame than `value`: the parsing network)"}
    if world == 1 and not args.no_cpu_baseline:
        _, _, cb = cpu_reference(cfg, 1, 0)
        line["cpu_baseline"] = cb
    emit(json.dumps(line))


def run_video(args, cfg, rank, world, local_rank):
    """configs[3]: a 900-frame 576x1024 clip (225 batches of 4) owned by rank 0 in pinned host memory as uint8 RGB; batches are
    dealt round-robin over the ranks (NCCL scatter), parsed + synthesised on the rank, the uint8 frames gathered to rank 0 and
    copied to pinned host memory.  The whole clip is the timed region."""
    import torch
    import torch.distributed as dist
    from vtoonify_b200 import _lib, ops
    from vtoonify_b200.bisenet import BiSeNet
    from vtoonify_b200.frame_loop import FramePipeline, ShardedFrameLoop
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_inputs, det_state_dict
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    ops.set_precision(args.precision)
    B, H, W = args.batch, args.height, args.width
    nb = (cfg["frames"] + B - 1) // B
    wire_u8 = args.wire == "u8"
    if world == 1:
        import datetime
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29533")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev, timeout=datetime.timedelta(seconds=600))
    with torch.no_grad():
        model = VToonify(backbone=cfg["backbone"]).eval()
        model.load_state_dict(det_state_dict(model, seed=0), strict=True)
        model.to(dev)
        pnet = BiSeNet(19).eval()
        pnet.load_state_dict(det_state_dict(pnet, seed=21), strict=True)
        pnet.to(dev)
        style = det_inputs(1, H, W, seed=0)[1]
        pipe = FramePipeline(model, style, d_s=0.5, device=dev, parsing_net=pnet, graph=args.graph)
        in_shape, in_dtype = ((B, H, W, 3), torch.uint8) if wire_u8 else ((B, 22, H, W), torch.float32)
        fn = pipe.process
        loop = ShardedFrameLoop(fn, in_shape, in_dtype, (B, 4 * H, 4 * W, 3), torch.uint8, dev)
        clip = outs = None
        if rank == 0:
            g = torch.Generator().manual_seed(5)
            n_distinct = 16                                    # the clip cycles over 16 distinct pinned batches (host memory bound)
            if wire_u8:
                clip = [torch.randint(0, 256, in_shape, generator=g, dtype=torch.uint8).pin_memory() for _ in range(n_distinct)]
            else:
                clip = [det_inputs(B, H, W, seed=i)[0].pin_memory() for i in range(n_distinct)]
            outs = [torch.empty((B, 4 * H, 4 * W, 3), dtype=torch.uint8).pin_memory() for _ in range(3 * world)]
        d2h = torch.cuda.Stream(dev)
        cnt = {"h2d": 0, "d2h": 0}

        def stage(i):
            t = clip[i % len(clip)]
            cnt["h2d"] += t.numel() * t.element_size()
            return t.to(dev, non_blocking=True)

        def sink(i, buf, ready):
            with torch.cuda.stream(d2h):
                ready()
                outs[i % len(outs)].copy_(buf, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(d2h)
            cnt["d2h"] += buf.numel()
            return ev
        st, sk = (stage, sink) if rank == 0 else (None, None)
        loop.run(max(1, args.warmup) * world, stage=st, sink=sk)
        torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
        cnt["h2d"] = cnt["d2h"] = 0
        loop.scatter_bytes = loop.gather_bytes = 0
        sampler = ClockSampler(local_rank) if rank == 0 else None
        if sampler:
            sampler.start()
        n0 = _lib.launch_count()
        t0 = time.perf_counter()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loop.run(nb, stage=st, sink=sk)
        d2h.synchronize()
        e1.record()
        torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
        ms = max(e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3)
        launches = _lib.launch_count() - n0
        clocks = sampler.stop() if sampler else None
    t = torch.tensor([ms], device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t[0])
    if rank != 0:
        return
    frames = nb * B
    rounds = (nb + world - 1) // world
    conf = workload_config(cfg, args, world)
    conf["workload"] = (f"{frames}-frame {H}x{W} clip ({nb} batches of {B}) in rank 0's pinned host memory as "
                        f"{'uint8 RGB frames (face parsing computed on the rank)' if wire_u8 else 'fp32 [B,22,H,W] network inputs'}, dealt round-robin over "
                        f"{world} GPU(s) by NCCL scatter, VToonify-D forward, uint8 BGR frames gathered to rank 0 and copied to pinned host memory "
                        f"({cfg['name']})")
    par = {"layout": f"round-robin frame batches over {world} rank(s); collectives: 1 scatter + 1 gather per round of {world} batches, overlapped",
           "nccl_bytes_per_step": {"scatter": loop.scatter_bytes // rounds, "gather": loop.gather_bytes // rounds}}
    line = {"metric": cfg["metric"], "value": frames / (ms * 1e-3), "unit": cfg["unit"], "n_gpus": world, "steps": rounds,
            "warmup": max(1, args.warmup), "ms_per_step": ms / rounds, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "bf16x3 (fp32 operands split into bf16 hi+lo, 3 tensor-core products, fp32 accumulate)",
            "data": "synthetic", "config": conf, "gpu_launches": int(launches), "clocks": clocks,
            "e2e": {"value": frames / (ms * 1e-3), "unit": cfg["unit"], "h2d_bytes_per_step": cnt["h2d"] // rounds,
                    "d2h_bytes_per_step": cnt["d2h"] // rounds, "note": "the whole clip is host-to-host: value == e2e"},
            "parallelism": par, "clip_seconds": ms * 1e-3}
    emit(json.dumps(line))


DUMP_BUDGET_FLOATS = 8 << 20   # 32 MB of float32 per dumped array


def dump_outputs(dirname, arrays):
    """arrays: name -> tensor.  Written as float32 .npy; an array larger than the budget is replaced by a fixed sample of its
    flattened elements (indices from a seeded generator, ascending), identical from run to run for the same shape."""
    import numpy as np
    import torch
    os.makedirs(dirname, exist_ok=True)
    for name, t in arrays.items():
        flat = t.detach().reshape(-1).float()
        if flat.numel() > DUMP_BUDGET_FLOATS:
            idx = torch.randint(0, flat.numel(), (DUMP_BUDGET_FLOATS,), generator=torch.Generator().manual_seed(0)).sort().values
            flat = flat[idx.to(flat.device)]
        np.save(os.path.join(dirname, name + ".npy"), flat.cpu().numpy().astype(np.float32))


_REAL_STDOUT = None


def emit(line):
    """Write the result line to the process's original stdout (fd 1 is pointed at stderr while the benchmark runs so that
    library chatter such as NCCL's version banner cannot end up next to the JSON line)."""
    if _REAL_STDOUT is None:
        print(line, flush=True)
    else:
        os.write(_REAL_STDOUT, (line + "\n").encode())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "cudnn"])
    ap.add_argument("--config", default="vtoonify_d", choices=sorted(CONFIGS),
                    help="vtoonify_d = BASELINE configs[1] (the metric's config, default); generator = configs[2]; video = configs[3]; "
                         "vtoonify_t = configs[4]")
    ap.add_argument("--backbone", default=None, choices=["dualstylegan", "toonify"], help="(legacy) overrides the config's backbone")
    ap.add_argument("--dump-layers", default=None, help="write the per-layer conv_tc timing table to this file")
    ap.add_argument("--precision", default="bf16x3", choices=["tf32", "bf16x3", "fp32"],
                    help="bf16x3 (default): split-operand tensor-core mode that meets the 1e-3 parity bar; tf32: faster, 3e-3 error")
    ap.add_argument("--height", type=int, default=None)
    ap.add_argument("--width", type=int, default=None)
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--wire", default="u8", choices=["u8", "f32"], help="--config video: what crosses PCIe / NVLink on the input side")
    ap.add_argument("--graph", action="store_true", help="end-to-end legs replay one captured CUDA graph per input geometry")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--ref-budget", type=float, default=660.0,
                    help="--impl reference: seconds the K timed CPU steps may take; full-size frames unless the host is too slow for that")
    ap.add_argument("--no-u8", action="store_true", help="skip the uint8-wire / on-device parsing end-to-end leg")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the last timed step's output to DIR/<name>.npy (float32, seeded sample when large); single GPU")
    args = ap.parse_args()
    cfg = dict(CONFIGS[args.config])
    if args.backbone:
        cfg["backbone"] = args.backbone
    if cfg["kind"] == "vtoonify":
        cfg["H"] = args.height = args.height or cfg["H"]
        cfg["W"] = args.width = args.width or cfg["W"]
    args.batch = args.batch or cfg["B"]
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    if args.dump_outputs and (args.impl != "ours" or args.config == "video" or int(os.environ.get("WORLD_SIZE", "1")) > 1):
        ap.error("--dump-outputs needs the single-GPU timed path of this implementation (not --config video)")

    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference(args, cfg, rank, world)
        return
    if args.impl == "cudnn":
        run_cudnn(args, cfg, rank, world)
        return
    if world > 1:
        import torch
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if os.environ.get("NCCL_DEBUG", "").upper() == "VERSION":
            os.environ["NCCL_DEBUG"] = "WARN"      # keep stdout to the single JSON line
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    try:
        if args.config == "video":
            run_video(args, cfg, rank, world, local_rank)
        else:
            run_ours(args, cfg, rank, world, local_rank)
    finally:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
