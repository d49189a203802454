"""The training scripts' geometric augmentation (train_vtoonify_d.py:262, train_vtoonify_t.py:206): random_apply_affine on
[8, 6, 1024, 1024] at p = 0.2, plus one zoom-out workload on the unfused side of the planner.

Workloads: a fixed list of transforms every arm uses: an untransformed batch (pad 6), the first seed whose batch-wide pad is near the
median of the training transforms (about 183 px), and seeds 1 and 2; then a 5.5x zoom-out on [8, 6, 512, 512].
Arms, alternated within each run:
- lib:   vtoonify_b200.simple_augment.random_apply_affine (the fused kernel, or the unfused route where the planner says 0);
- ref:   the statements of tests/oracle_augment.py in fp32 with the reference's own upfirdn2d CUDA op from oracle/_ref and torch's
         affine_grid / grid_sample: what the reference costs (skipped when oracle/_ref was not built);
- lvl_b: the same statements on vtoonify_b200.op.upfirdn2d.
Prints one JSON line per (run, workload, arm): ms per call from CUDA events, library launches per call, max_memory_allocated, and for
the library's fused route the bytes a single pass must move (read the input, write the output) over its time.

Then the whole torch.no_grad() data block of train_vtoonify_d.py:238-276 at batch 8 on the library's modules with det_state_dict
weights: the StyleGAN synthesis of x'' from a random w plus a direction, pSp on its 256^2 average pool (plus a fixed latent_avg, as
load_psp_standalone adds), zplus2wplus, the DualStyleGAN synthesis of y', the augmentation of cat(x'', y'), the two Downsamples,
BiSeNet at 512^2 and the mask pooling.  Two arms, alternated: the library augmentation and the reference-op one (the ref arm's
statements); both use the same fixed list of p = 0.2 transforms.  One JSON line per (run, arm): ms per block, the augmentation's
ms inside it (CUDA events around that statement) and its share, and max_memory_allocated.  Last, a line with the card name and
power limit from nvidia-smi in the same call.

    python tools/augment_bench.py --steps 20 --warmup 3 --runs 2
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


def ref_upfirdn2d():
    """the reference's upfirdn2d CUDA op behind its Python wrapper's signature, or None when oracle/_ref holds no build"""
    from oracle import build_ref
    ops = build_ref.load_ops()
    if ops is None:
        return None
    up_op = ops[0]

    def upfirdn2d(x, kernel, up=1, down=1, pad=(0, 0)):
        up_x, up_y = (up, up) if isinstance(up, int) else up
        down_x, down_y = (down, down) if isinstance(down, int) else down
        _, C, H, W = x.shape
        out = up_op.upfirdn2d(x.reshape(-1, H, W, 1), kernel, up_x, up_y, down_x, down_y, pad[0], pad[1], pad[2], pad[3])
        return out.view(-1, C, out.shape[1], out.shape[2])
    return upfirdn2d


def workloads():
    from vtoonify_b200 import simple_augment as A
    B, C, H, W = 8, 6, 1024, 1024

    def sampled(seed):
        torch.manual_seed(seed)
        return torch.inverse(A.sample_affine(0.2, B, H, W))

    median = next(s for s in range(200) if 160 <= max(int(v) for v in A.padding(sampled(s), H, W)) <= 210)
    out = [("identity", (B, C, H, W), torch.eye(3).repeat(B, 1, 1))]
    out += [(f"seed{s}", (B, C, H, W), sampled(s)) for s in (median, 1, 2)]
    z = torch.tensor([[5.5, 0.0, 0.3], [0.0, 5.5, -0.2], [0.0, 0.0, 1.0]]).repeat(B, 1, 1)
    out.append(("zoom5.5", (B, C, 512, 512), z))
    return out


def data_block(args, dev, arms):
    """train_vtoonify_d.py:238-276 (the `not fix_color` branch, before the iteration that starts colour fusion) at batch 8"""
    from argparse import Namespace

    import torch.nn.functional as F

    from vtoonify_b200 import simple_augment as A
    from vtoonify_b200.bisenet import BiSeNet
    from vtoonify_b200.psp import GradualStyleEncoder
    from vtoonify_b200.stylegan import Downsample
    from vtoonify_b200.vtoonify import VToonify
    from vtoonify_b200.weights import det_state_dict

    B = 8
    g_ema = VToonify(backbone="dualstylegan").eval()
    g_ema.load_state_dict(det_state_dict(g_ema, seed=0), strict=True)
    g_ema.to(dev)
    psp = GradualStyleEncoder(50, "ir_se", Namespace(input_nc=3, n_styles=18)).eval()
    psp.load_state_dict(det_state_dict(psp, seed=11), strict=True)
    psp.to(dev)
    parsing = BiSeNet(19).eval()
    parsing.load_state_dict(det_state_dict(parsing, seed=21), strict=True)
    parsing.to(dev)
    down = Downsample(kernel=[1, 3, 3, 1], factor=2).to(dev)
    g = torch.Generator().manual_seed(0)
    latent_avg = (0.1 * torch.randn(18, 512, generator=g)).to(dev)
    directions = (0.1 * torch.randn(32, 18, 512, generator=g)).to(dev)
    style = torch.randn(B, 18, 512, generator=g).to(dev)
    weight = [0.5] * 7 + [1] * 11
    Gs = []
    for seed in range(8):
        torch.manual_seed(seed)
        Gs.append(torch.inverse(A.sample_affine(0.2, B, 1024, 1024)))

    def block(aug, G, ev):
        noise_sample = torch.randn(B, 512, device=dev)
        wc = g_ema.stylegan().style(noise_sample).unsqueeze(1).repeat(1, 18, 1)
        wc[:, 3:7] += directions[torch.randint(0, directions.shape[0], (B,)), 3:7]
        xc, _ = g_ema.stylegan()([wc], input_is_latent=True, truncation=0.5, truncation_latent=0)
        xc = torch.clamp(xc, -1, 1)
        xl = psp(F.adaptive_avg_pool2d(xc, 256)) + latent_avg
        xl = g_ema.zplus2wplus(xl)
        xl = torch.cat((style[:, 0:7], xl[:, 7:18]), dim=1)
        xs, _ = g_ema.generator([wc], xl, input_is_latent=True, truncation=0.5, truncation_latent=0, use_res=True,
                                interp_weights=weight)
        xs = torch.clamp(xs, -1, 1)
        x = torch.cat((xc, xs), dim=1)
        ev[0].record()
        imgs = aug(x, G)
        ev[1].record()
        real_input1024 = imgs[:, 0:3]
        real_input512 = down(real_input1024)
        real_input256 = down(real_input512)
        mask512 = parsing(2 * real_input512)[0]
        mask256 = down(mask512)
        F.adaptive_avg_pool2d(mask512, 1024)
        return torch.cat((real_input256, mask256 / 16.0), dim=1), imgs[:, 3:]

    steps = max(args.steps // 2, 5)
    with torch.no_grad():
        for run in range(args.runs):
            for arm, aug in arms.items():
                torch.manual_seed(1000 + run)
                for i in range(args.warmup):
                    block(aug, Gs[i % len(Gs)], [torch.cuda.Event(enable_timing=True) for _ in range(2)])
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                evs = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in range(steps)]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(steps):
                    block(aug, Gs[i % len(Gs)], evs[i])
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / steps
                aug_ms = sum(a.elapsed_time(b) for a, b in evs) / steps
                print(json.dumps({"run": run, "workload": "data_block_b8", "arm": arm, "ms": round(ms, 2),
                                  "augment_ms": round(aug_ms, 2), "augment_share": round(aug_ms / ms, 4),
                                  "peak_mb": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augment_bench needs a CUDA device")
    from tests import oracle_augment as O
    from vtoonify_b200 import _lib
    from vtoonify_b200 import simple_augment as A
    from vtoonify_b200.op import upfirdn2d as lvl_b_upfirdn2d

    dev = torch.device("cuda", 0)
    ref_up = ref_upfirdn2d()
    arms = {"lib": lambda x, G: A.random_apply_affine(x, 0.2, G)[0],
            "lvl_b": lambda x, G: O.apply(x, G, upfirdn=lvl_b_upfirdn2d)}
    if ref_up is not None:
        arms["ref"] = lambda x, G: O.apply(x, G, upfirdn=ref_up)
    else:
        print(json.dumps({"note": "oracle/_ref not built: the ref arm is not measured"}))
    cases = workloads()
    with torch.no_grad():
        for run in range(args.runs):
            for name, shape, G in cases:
                x = torch.randn(shape, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
                B, C, H, W = shape
                pads = tuple(int(v) for v in A.padding(G, H, W))
                tile = A.plan(A.warp_coefficients(A.sampling_matrix(G, pads, H, W), pads, H, W), H, W)[0]
                for arm, fn in arms.items():
                    for _ in range(args.warmup):
                        fn(x, G)
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    base = torch.cuda.memory_allocated()
                    n0 = _lib.launch_count()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        fn(x, G)
                    e1.record()
                    torch.cuda.synchronize()
                    ms = e0.elapsed_time(e1) / args.steps
                    line = {"run": run, "workload": name, "shape": list(shape), "pads": list(pads), "tile": tile, "arm": arm,
                            "ms": round(ms, 4), "launches": (_lib.launch_count() - n0) / args.steps,
                            "peak_mb": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1),
                            "peak_over_input_mb": round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)}
                    if arm == "lib" and tile > 0:
                        nbytes = 2 * x.numel() * 4
                        line["analytic_gb"] = round(nbytes / 1e9, 4)
                        line["gb_per_s"] = round(nbytes / (ms * 1e-3) / 1e9, 1)
                    print(json.dumps(line), flush=True)
                del x
        torch.cuda.empty_cache()
        data_block(args, dev, {k: v for k, v in arms.items() if k in ("lib", "ref")})
    print(json.dumps({"card": card(), "torch": torch.__version__,
                      "note": "card name, power limit and max SM clock from nvidia-smi in the same call"}))


if __name__ == "__main__":
    main()
