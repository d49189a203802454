"""Writes tests/golden/smooth_*.npz from the unmodified reference smooth_parsing_map.py, run on the CPU in float32.

    python tests/golden/make_golden_smooth.py /path/to/reference

The only changes are shims of the environment: ``Tensor.cuda``, ``Tensor.to("cuda")`` and ``Module.to("cuda")`` stay on the CPU, and
``model.stylegan.op`` is the reference's own ``op_cpu`` (model/stylegan/op_cpu/readme.md).

``smooth_warp.npz``: the script's ``warp`` on seeded x [2, 22, 31, 37] and flows that mix zero flow, fractional samples, samples far
outside, samples exactly on the border and samples 1e-3 px outside it (in-bounds corner weight 0.999, well below the 0.9999
threshold).  No sample's in-bounds weight lies within 2e-4 of 1 without being 1: CPU and CUDA ``grid_sample`` need not round the
unnormalised coordinate alike, so a sample inside the threshold's band would not be a stable fixture.

``smooth_w2.npz`` (N = 6 frames of 64x72, window 2) and ``smooth_w5.npz`` (N = 5 frames of 64x64, window 5: every window is a boundary
window): the script's ``__main__`` through ``runpy`` with a ``cv2.VideoCapture`` stub serving seeded uint8 BGR frames, ``torch.load``
serving ``det_state_dict`` weights (RAFT's ``module.``-prefixed) and a parsing-network stub returning ``parsing_maps`` of a stored
low-resolution seed.  Stored: the frames, the seed and channels ``CHANNELS`` of ``parse``.
"""
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

N_CLASSES = 19
CHANNELS = (0, 7, 18)        # the stored channels of parse: the fusion treats every channel alike
CASES = {"w2": dict(N=6, h=64, w=72, window=2, seed=11), "w5": dict(N=5, h=64, w=64, window=5, seed=12)}


def frames_bgr(N, h, w, seed):
    """seeded smooth uint8 BGR frames [N, h, w, 3] that drift and rotate slightly from frame to frame"""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand((1, 3, h // 8 + 4, w // 8 + 4), generator=g), size=(h + 32, w + 32), mode="bicubic",
                         align_corners=False)
    base = base + 0.2 * F.interpolate(torch.rand((1, 3, h // 2 + 8, w // 2 + 8), generator=g), size=(h + 32, w + 32), mode="bilinear",
                                      align_corners=False)
    out = []
    for k in range(N):
        th = torch.tensor(0.02 * k)
        theta = torch.tensor([[torch.cos(th), -torch.sin(th), 0.03 * k], [torch.sin(th), torch.cos(th), -0.02 * k]])[None]
        grid = F.affine_grid(theta, (1, 3, h + 32, w + 32), align_corners=False)
        out.append(F.grid_sample(base, grid, mode="bilinear", padding_mode="border", align_corners=False)[0, :, 16:16 + h, 16:16 + w])
    x = torch.stack(out, 0)
    x = torch.round((x - x.min()) / (x.max() - x.min()) * 255.0)
    return x.permute(0, 2, 3, 1).to(torch.uint8).numpy()


def script_inputs(frames):
    """the script's ``Is``: ToTensor, Normalize(0.5, 0.5) of the RGB frames and the 2x bilinear up-sampling (lines 86-89, 122-128)"""
    rgb = torch.from_numpy(np.ascontiguousarray(frames[..., ::-1])).permute(0, 3, 1, 2).contiguous().float().div(255)
    return F.interpolate((rgb - 0.5) / 0.5, scale_factor=2, mode="bilinear", align_corners=False)


def parsing_seed(N, seed):
    g = torch.Generator().manual_seed(100 + seed)
    return 4.0 * torch.randn((N, N_CLASSES, 5, 6), generator=g)


def parsing_maps(seed, H, W):
    """the stub parsing network's output for every frame: the seed up-sampled to H x W, rounded to multiples of 1/64 (exact in float32)"""
    return torch.round(F.interpolate(seed, size=(H, W), mode="bilinear", align_corners=False) * 64.0) / 64.0


def warp_inputs():
    g = torch.Generator().manual_seed(5)
    B, C, H, W = 2, 22, 31, 37
    x = torch.randn((B, C, H, W), generator=g)
    flo = (torch.rand((B, 2, H, W), generator=g) - 0.5) * 12.0                  # fractional, partly outside
    flo[:, :, :4] = 0.0                                                           # zero flow
    flo[0, 0, 4:6] = 5000.0                                                       # far outside
    flo[1, 1, 4:6] = -3000.0
    xs = torch.arange(W, dtype=torch.float32).view(1, W)
    ys = torch.arange(H, dtype=torch.float32).view(H, 1)
    flo[:, 0, 6] = (W - 1) - xs                       # exactly on the right border, row 6
    flo[:, 1, 6] = 0.0
    flo[:, 0, 7] = -xs                                # exactly on the left border, row 7, with fractional y
    flo[:, 1, 7] = 0.25
    flo[:, 0, 8] = (W - 1) - xs + 1e-3                # 1e-3 px outside on the right and the left
    flo[:, 1, 8] = 0.0
    flo[:, 0, 9] = -xs - 1e-3
    flo[:, 1, 9] = 0.0
    flo[:, 1, 10] = (H - 1) - ys[10] + 1e-3           # 1e-3 px below the bottom border
    flo[:, 0, 10] = 0.0
    # no sample in the threshold's band: in float64, drop (to zero flow) any sample whose in-bounds weight is within 2e-4 of 1
    # without being 1
    px = xs.double() + flo[:, 0].double()
    py = ys.double() + flo[:, 1].double()
    x0, y0 = torch.floor(px), torch.floor(py)
    tx, ty = px - x0, py - y0
    m = torch.zeros_like(px)
    for dx, dy, wgt in ((0, 0, (1 - tx) * (1 - ty)), (1, 0, tx * (1 - ty)), (0, 1, (1 - tx) * ty), (1, 1, tx * ty)):
        ok = (x0 + dx >= 0) & (x0 + dx <= W - 1) & (y0 + dy >= 0) & (y0 + dy <= H - 1)
        m = m + torch.where(ok, wgt, torch.zeros_like(wgt))
    band = ((m - 1.0).abs() < 2e-4) & ((m - 1.0).abs() > 1e-9)
    band[:, :11] = False                               # the constructed rows are exact by construction
    flo[:, 0][band] = 0.0
    flo[:, 1][band] = 0.0
    return x.contiguous(), flo.contiguous()


class _VideoCapture:
    frames = None

    def __init__(self, path):
        self.k = 0

    def get(self, prop):
        return float(len(self.frames))

    def read(self):
        if self.k >= len(self.frames):
            return False, None
        self.k += 1
        return True, self.frames[self.k - 1].copy()

    def release(self):
        pass


class _ParsingStub(torch.nn.Module):
    """BiSeNet stand-in: returns (maps[i], ...) for the i-th call"""
    maps = None

    def __init__(self, n_classes=19):
        super().__init__()
        self.k = 0

    def load_state_dict(self, *a, **k):
        return None

    def forward(self, x):
        self.k += 1
        return (self.maps[self.k - 1:self.k],)


def _shim_cuda():
    def cpu_to(orig):
        def to(self, *a, **k):
            a = tuple("cpu" if (isinstance(v, str) and v.startswith("cuda")) or (isinstance(v, torch.device) and v.type == "cuda")
                      else v for v in a)
            if "device" in k and str(k["device"]).startswith("cuda"):
                k["device"] = "cpu"
            return orig(self, *a, **k)
        return to
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.Tensor.to = cpu_to(torch.Tensor.to)
    torch.nn.Module.to = cpu_to(torch.nn.Module.to)


def main(ref_root):
    sys.path.insert(0, ref_root)
    import model.stylegan.op_cpu as op_cpu
    sys.modules["model.stylegan.op"] = op_cpu
    _shim_cuda()
    from vtoonify_b200.weights import det_state_dict
    from model.raft.core.raft import RAFT
    from tests.golden.make_golden_raft import raft_args
    stub = types.ModuleType("model.bisenet.model")
    stub.BiSeNet = _ParsingStub
    sys.modules["model.bisenet.model"] = stub
    import cv2
    cv2.VideoCapture = _VideoCapture
    sys.argv = ["smooth_parsing_map.py"]
    script = runpy.run_path(os.path.join(ref_root, "smooth_parsing_map.py"), run_name="not_main")

    x, flo = warp_inputs()
    with torch.no_grad():
        out, mask = script["warp"](x, flo)
    assert torch.equal(mask, mask[:, :1].expand_as(mask))
    np.savez_compressed(os.path.join(HERE, "smooth_warp.npz"), x=x.numpy(), flo=flo.numpy(), out=out.numpy(), mask=mask[:, :1].numpy())
    print("warp", "mask mean", float(mask.mean()))

    torch.manual_seed(0)
    m = RAFT(raft_args()).eval()
    raft_sd = {"module." + k: v for k, v in det_state_dict(m, seed=0).items()}
    real_load = torch.load
    for name, c in CASES.items():
        frames = frames_bgr(c["N"], c["h"], c["w"], c["seed"])
        seed = parsing_seed(c["N"], c["seed"])
        _VideoCapture.frames = list(frames)
        _ParsingStub.maps = parsing_maps(seed, 2 * c["h"], 2 * c["w"])
        torch.load = lambda path, *a, **k: raft_sd if "raft" in str(path) else {}
        with tempfile.TemporaryDirectory() as tmp:
            sys.argv = ["smooth_parsing_map.py", "--window_size", str(c["window"]), "--video_path", os.path.join(tmp, "clip.mp4"),
                        "--output_path", tmp, "--raft_path", "raft-things.pth", "--faceparsing_path", "faceparsing.pth"]
            try:
                g = runpy.run_path(os.path.join(ref_root, "smooth_parsing_map.py"), run_name="__main__")
            finally:
                torch.load = real_load
            parse = np.load(os.path.join(tmp, "clip_parsingmap.npy"))
        assert torch.equal(g["Is"], script_inputs(frames)) and torch.equal(g["Ps"], _ParsingStub.maps)
        np.savez_compressed(os.path.join(HERE, f"smooth_{name}.npz"), frames=frames, seed=seed.numpy(), window=np.array(c["window"]),
                            channels=np.array(CHANNELS), parse=np.ascontiguousarray(parse[:, list(CHANNELS)]))
        print(name, "parse", parse.shape, "mean", float(parse.mean()))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
