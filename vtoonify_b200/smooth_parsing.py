"""Temporal smoothing of face-parsing maps (smooth_parsing_map.py) on the library.

``warp(x, flo)`` is a drop-in for the script's ``warp``: the same ``(output * mask, mask)``, the mask materialised at ``[B, C, H, W]``.

``smooth_parsing_maps(Is, Ps, raft_model, window=5, iters=20)`` is the script's whole smoothing loop (lines 143-167): it returns its
``parse`` ``[N, C, H/2, W/2]`` on ``Ps``'s device, given the script's ``Is`` (the 2x up-sampled frames in [-1, 1], ``[N, 3, H, W]``) and
``Ps`` (the parsing logits, ``[N, C, H, W]``), on the CPU or on the device.  ``raft_model`` is a ``vtoonify_b200.raft.RAFT``.

The loop streams (DESIGN.md section 12):
  * a device ring of the ``2 * window + 1`` frames of the current window holds each frame's image, its RAFT input
    ``(I + 1) * 255.0 / 2``, its parsing map and its ``fnet`` features; every frame is uploaded and encoded once, and device memory does
    not grow with ``N``;
  * slot ``k`` of output frame ``i`` reads frame ``slot_frames(N, window)[i][k]``, the reference's ``cat((Is[0:w], Is, Is[-w:]))``
    indexing, boundary windows included (a frame may fill two slots, or the centre's own frame a non-centre slot: those pairs run);
  * per output frame: ``cnet`` once on the centre, the RAFT iterations on the ``2 * window`` non-centre pairs as one batch, one fusion
    launch (warp, spatial weights, normalisation and the weighted sum; nothing ``[11, 22, H, W]``-sized is materialised) and one
    ``Downsample([1, 3, 3, 1], 2)`` launch.  The centre pair RAFT(I_i, I_i) of the script is skipped: the script overwrites both of
    its results.
The RAFT convolutions follow ``set_precision``; the warp and the fusion are fp32 in every mode.
"""
import torch

from . import ops
from ._lib import c_float, c_void_p, check, load
from .raft import MIN_SIZE, RAFT
from .stylegan import make_kernel

MAX_WINDOW = 31             # the fusion kernel's slot table holds 2 * 31 + 1 slots


def temporal_weights(window: int) -> torch.Tensor:
    """the script's ``wt`` (line 144), float32 on the CPU, ``[2 * window + 1]``"""
    return torch.exp(-(torch.arange(2 * window + 1).float() - window) ** 2 / (2 * ((window + 0.5) ** 2))).reshape(2 * window + 1)


def slot_frames(N: int, window: int):
    """for each output frame i, the frame index behind each of its ``2 * window + 1`` slots: ``Is_[i : i + 2w + 1]`` with
    ``Is_ = cat((Is[0:w], Is, Is[-w:]))`` (``Is[-0:]`` is all of ``Is``, as in Python)"""
    head = list(range(0, min(window, N)))
    tail = list(range(N))[-window:] if window else list(range(N))
    ext = head + list(range(N)) + tail
    return [ext[i:i + 2 * window + 1] for i in range(N)]


def _check_no_grad(name, *ts):
    if torch.is_grad_enabled():
        for t in ts:
            if t is not None and t.requires_grad:
                raise NotImplementedError(f"{name}: inputs that require grad are not supported (forward only; run under torch.no_grad())")


def warp(x: torch.Tensor, flo: torch.Tensor):
    """smooth_parsing_map.py:38-74 on planar fp32 CUDA tensors: x [B, C, H, W], flo [B, 2, H, W] -> (warped x * mask, mask)"""
    _check_no_grad("warp", x, flo)
    if x.dim() != 4 or flo.dim() != 4 or flo.shape[1] != 2 or flo.shape[0] != x.shape[0] or flo.shape[2:] != x.shape[2:]:
        raise ValueError(f"warp: x {tuple(x.shape)} must be [B, C, H, W] and flo {tuple(flo.shape)} [B, 2, H, W]")
    ops._req_cuda(x, flo)
    B, C, H, W = x.shape
    x, flo = x.contiguous(), flo.contiguous()
    out = torch.empty_like(x)
    mask = torch.empty_like(x)
    check(load().vt_flow_warp_f32(x.data_ptr(), flo.data_ptr(), out.data_ptr(), mask.data_ptr(), B, C, H, W, ops._stream()))
    return out, mask


def parsing_fuse(imgs, pars, flows, wt, out=None):
    """one centre of the window fusion (script lines 155-165 before ``down``): per-slot planar CUDA tensors imgs[k] [3, H, W],
    pars[k] [C, H, W], flows[k] [2, H, W] (``flows[window]`` is ignored and may be None), host weights wt [2 * window + 1] ->
    fused [C, H, W]"""
    n = len(imgs)
    if n % 2 != 1 or n > 2 * MAX_WINDOW + 1 or len(pars) != n or len(flows) != n or len(wt) != n:
        raise ValueError(f"parsing_fuse: need 2 * window + 1 <= {2 * MAX_WINDOW + 1} slots in every list")
    C, H, W = pars[0].shape
    for k in range(n):
        ok = tuple(imgs[k].shape) == (3, H, W) and tuple(pars[k].shape) == (C, H, W)
        ok = ok and (k == n // 2 or tuple(flows[k].shape) == (2, H, W))
        if not ok:
            raise ValueError(f"parsing_fuse: slot {k} must hold [3, {H}, {W}], [{C}, {H}, {W}] and [2, {H}, {W}] tensors")
        ops._req_cuda(imgs[k], pars[k], None if k == n // 2 else flows[k])
        if not (imgs[k].is_contiguous() and pars[k].is_contiguous() and (k == n // 2 or flows[k].is_contiguous())):
            raise ValueError(f"parsing_fuse: slot {k} tensors must be contiguous")
    if out is None:
        out = torch.empty((C, H, W), device=pars[0].device, dtype=torch.float32)
    ptrs = [(c_void_p * n)(*[None if t is None else t.data_ptr() for t in ts]) for ts in (imgs, pars, flows)]
    w = (c_float * n)(*[float(v) for v in wt])
    check(load().vt_parsing_fuse_f32(ptrs[0], ptrs[1], ptrs[2], w, n, out.data_ptr(), C, H, W, ops._stream()))
    return out


def _check_args(Is, Ps, raft_model, window, iters):
    if not isinstance(raft_model, RAFT):
        raise NotImplementedError("smooth_parsing_maps: raft_model must be a vtoonify_b200.raft.RAFT")
    raft_model._check_model()
    _check_no_grad("smooth_parsing_maps", Is, Ps)
    if int(window) != window or window < 0 or window > MAX_WINDOW:
        raise ValueError(f"smooth_parsing_maps: window must be an integer in 0..{MAX_WINDOW} (got {window})")
    if int(iters) < 1:
        raise ValueError("smooth_parsing_maps: iters must be at least 1")
    if Is.dim() != 4 or Is.shape[1] != 3 or Ps.dim() != 4 or Ps.shape[0] != Is.shape[0] or Ps.shape[2:] != Is.shape[2:]:
        raise ValueError(f"smooth_parsing_maps: Is {tuple(Is.shape)} must be [N, 3, H, W] and Ps {tuple(Ps.shape)} [N, C, H, W]")
    if Is.dtype != torch.float32 or Ps.dtype != torch.float32:
        raise ValueError(f"smooth_parsing_maps: Is and Ps must be float32 (got {Is.dtype}, {Ps.dtype})")
    N, _, H, W = Is.shape
    if N < max(window, 1):
        raise ValueError(f"smooth_parsing_maps: {N} frames are fewer than the window {window} (the script's RAFT batches would not match)")
    if H % 8 or W % 8 or H < MIN_SIZE or W < MIN_SIZE:
        raise ValueError(f"smooth_parsing_maps: H and W must be multiples of 8 and at least {MIN_SIZE} (got {H}x{W})")


def smooth_parsing_maps(Is: torch.Tensor, Ps: torch.Tensor, raft_model: RAFT, window: int = 5, iters: int = 20) -> torch.Tensor:
    """smooth_parsing_map.py:143-167: the temporally fused, down-sampled parsing maps [N, C, H/2, W/2] on ``Ps``'s device"""
    return _smooth(Is, Ps, raft_model, window, iters)


def _smooth(Is, Ps, raft_model, window, iters, flow_sink=None):
    """smooth_parsing_maps; ``flow_sink(i, up)`` (tests) receives output frame i's up-sampled flows [2 * window, 2, H, W]"""
    _check_args(Is, Ps, raft_model, window, iters)
    window, iters = int(window), int(iters)
    N, C, H, W = Ps.shape
    dev = Is.device if Is.is_cuda else (Ps.device if Ps.is_cuda else next(raft_model.parameters()).device)
    if dev.type != "cuda":
        raise ValueError("smooth_parsing_maps: the RAFT model (or Is / Ps) must be on a CUDA device")
    R = 2 * window + 1
    wt = temporal_weights(window).tolist()
    slots = slot_frames(N, window)
    kernel = make_kernel([1, 3, 3, 1]).to(dev)
    parse = torch.empty((N, C, H // 2, W // 2), device=Ps.device, dtype=torch.float32)
    with torch.no_grad():
        # the ring: frame f lives at position f % R (the frames one output reads span at most R consecutive indices)
        img = torch.empty((R, 3, H, W), device=dev, dtype=torch.float32)
        rin = torch.empty((R, 3, H, W), device=dev, dtype=torch.float32)
        par = torch.empty((R, C, H, W), device=dev, dtype=torch.float32)
        fmap = [None] * R
        loaded = -1                       # frames 0..loaded have been uploaded and encoded
        fused = torch.empty((C, H, W), device=dev, dtype=torch.float32)
        for i in range(N):
            fr = slots[i]
            for f in range(loaded + 1, max(fr) + 1):
                r = f % R
                img[r].copy_(Is[f])
                par[r].copy_(Ps[f])
                torch.add(img[r], 1, out=rin[r]).mul_(255.0).div_(2)        # the script's (I + 1) * 255.0 / 2
                if window:
                    fmap[r] = raft_model._features(raft_model._input_s2d(rin[r:r + 1]))
                loaded = f
            pos = [f % R for f in fr]
            c = pos[window]
            flows = [None] * R
            if window:
                nb = [pos[k] for k in range(R) if k != window]
                B = len(nb)
                f1 = fmap[c].expand(B, -1, -1, -1).contiguous()
                f2 = torch.cat([fmap[p] for p in nb], 0)
                net, x = raft_model._context(raft_model._input_s2d(rin[c:c + 1]))
                _, up = raft_model._iterate(f1, f2, net.expand(B, -1, -1, -1).contiguous(), x.expand(B, -1, -1, -1).contiguous(), iters)
                flows = [up[k if k < window else k - 1] if k != window else None for k in range(R)]
                if flow_sink is not None:
                    flow_sink(i, up)
            parsing_fuse([img[p] for p in pos], [par[p] for p in pos], flows, wt, out=fused)
            parse[i].copy_(ops.upfirdn2d_planar(fused[None], kernel, (1, 1), (2, 2), (1, 1, 1, 1))[0])
    return parse
