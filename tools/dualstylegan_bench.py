"""The two DualStyleGAN teacher calls of VToonify-D training (train_vtoonify_d.py) at batch 8 on the 1024 model, next to the
Generator.forward call on the same latent that produces the training image x'' (train_vtoonify_d.py:125, 245):
   pretrain   g_ema.generator([ws_], style, input_is_latent=True, return_feat=True, truncation=0.5, truncation_latent=0,
              use_res=True, interp_weights=[d_s]*7 + [1]*11)                                   (:132, stops after 32²)
   full       g_ema.generator([wc], xl, input_is_latent=True, truncation=0.5, truncation_latent=0, use_res=True,
              interp_weights=[d_s]*7 + [1]*11)                                                 (:251, 1024² image)
   generator  g_ema.stylegan()([wc], input_is_latent=True, truncation=0.5, truncation_latent=0)
Every call gets a fresh random code pair, as in training (drawn before the timed window), and random noise.
   python tools/dualstylegan_bench.py [calls] [precision]      (on the GPU box)

ms per call from CUDA events around `calls` back-to-back calls after 3 warm-up calls; then, in a separate pass with per-launch
events, the conv_tc time per call and its share of the unprofiled call time.  The card's name, power limit and SM clocks are
read in the same run."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vtoonify_b200 import _lib, ops  # noqa: E402
from vtoonify_b200.dualstylegan import DualStyleGAN  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402

B, WARMUP, D_S = 8, 3, 0.5


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi not available"
    return q or torch.cuda.get_device_name()


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    prec = sys.argv[2] if len(sys.argv) > 2 else ops.DEFAULT_PRECISION
    if calls < 20:
        raise SystemExit("time at least 20 calls")
    ops.set_precision(prec)
    print(f"card: {card()}")
    m = DualStyleGAN(1024, 512, 8).eval()
    m.load_state_dict(det_state_dict(m, seed=5), strict=True)
    m.cuda()
    g = torch.Generator().manual_seed(0)
    n = WARMUP + 2 * calls
    pool = [(torch.randn((B, 18, 512), generator=g).cuda(), torch.randn((B, 18, 512), generator=g).cuda()) for _ in range(n)]
    kw = dict(input_is_latent=True, truncation=0.5, truncation_latent=0)
    weights = [D_S] * 7 + [1] * 11
    cases = {
        "pretrain": lambda w, s: m([w], s, return_feat=True, use_res=True, interp_weights=weights, **kw),
        "full": lambda w, s: m([w], s, use_res=True, interp_weights=weights, **kw),
        "generator": lambda w, s: m.generator([w], **kw),
    }
    result = {"card": card(), "precision": prec, "batch": B, "calls": calls}
    with torch.no_grad():
        for name, fn in cases.items():
            for w, s in pool[:WARMUP]:
                fn(w, s)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n0 = _lib.launch_count()
            e0.record()
            for w, s in pool[WARMUP:WARMUP + calls]:
                fn(w, s)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / calls
            launches = (_lib.launch_count() - n0) / calls
            prof = []
            ops.set_tc_profile(prof)
            try:
                for w, s in pool[WARMUP + calls:]:
                    fn(w, s)
                torch.cuda.synchronize()
            finally:
                ops.set_tc_profile(None)
            tc_ms = sum(a.elapsed_time(b) for a, b, *_ in prof) / calls
            result[name] = {"ms": round(ms, 3), "conv_tc_ms": round(tc_ms, 3), "conv_tc_share": round(tc_ms / ms, 3),
                            "launches": launches}
            print(f"{name:9s} B={B} [{prec}]: {ms:8.3f} ms/call  conv_tc {tc_ms:8.3f} ms ({100 * tc_ms / ms:4.1f} % of the call), "
                  f"{launches:.0f} launches/call")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
