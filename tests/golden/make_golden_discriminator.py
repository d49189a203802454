"""Generates tests/golden/discriminator_{cond,plain}.npz and state_dict_keys_discriminator{,_cond}.json: the UNMODIFIED reference
ConditionalDiscriminator (model/vtoonify.py:10-89) on CPU through its op_cpu path in float64, with the deterministic weights of
vtoonify_b200/weights.py (seed 0) and the seeded inputs of tests/oracle_discriminator.py.  Model: size 64, channel_multiplier 1
(a 256 -> 512 block and three 512 -> 512 blocks), batch 8 (two minibatch-stddev columns).  Loss: softplus(-out).mean().
Stored per case: the output, x.grad[:, :, ::4, ::4], every 1-D gradient in full, and for each weight gradient every WSTEP-th element
of the flattened tensor plus the whole tensor's L2 norm.  Run in the build container, like make_golden.py:

    python tests/golden/make_golden_discriminator.py
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, save  # noqa: E402
from model.vtoonify import ConditionalDiscriminator as RefD  # noqa: E402
from tests.oracle_discriminator import BATCH, CASES, CHANNEL_MULTIPLIER, SIZE, WSTEP, case_inputs, loss_fn  # noqa: E402
from vtoonify_b200.weights import det_state_dict  # noqa: E402


def golden_discriminator():
    for case, kw in CASES.items():
        m = RefD(SIZE, channel_multiplier=CHANNEL_MULTIPLIER, **kw)
        m.load_state_dict(det_state_dict(m, seed=0), strict=True)
        m = m.double()
        x, d, s = case_inputs(case)
        x = x.double().requires_grad_()
        out = m(x, d.double(), s) if kw["use_condition"] else m(x)
        loss = loss_fn(out)
        loss.backward()
        res = {"out": out.detach(), "x_grad_sub": x.grad[:, :, ::4, ::4]}
        for name, p in m.named_parameters():
            if p.dim() == 1:
                res["g:" + name] = p.grad
            else:
                res["gs:" + name] = p.grad.flatten()[::WSTEP]
                res["gn:" + name] = p.grad.norm()
        print(f"discriminator_{case}: loss {loss.item():.6f}, |x.grad| {x.grad.norm():.3e}")
        save(f"discriminator_{case}", **res)
    for name, kw in (("discriminator", {}), ("discriminator_cond", dict(use_condition=True, style_num=3))):
        sd = RefD(256, **kw).state_dict()
        path = os.path.join(HERE, f"state_dict_keys_{name}.json")
        with open(path, "w") as f:
            json.dump({k: list(v.shape) for k, v in sd.items()}, f, indent=0)
        print(f"{os.path.basename(path)}  {len(sd)} keys")


if __name__ == "__main__":
    torch.set_grad_enabled(True)        # make_golden switches it off at import
    golden_discriminator()
