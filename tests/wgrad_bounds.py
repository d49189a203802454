"""Per-element error bars for results that are bilinear in two operands, ``y = f(u, v)`` (the weight gradient of a convolution,
and its input gradient, the transposed convolution), plus float64 references and a float32 emulation of the weight-gradient
kernel's arithmetic (csrc/conv_wgrad.cu) to calibrate the bars against.

With ``E = f(|u|, |v|)`` (the sum of absolute terms) and ``R = sqrt(f(u^2, v^2))`` (the root-sum-square of the terms), both in
float64, every element of a result is checked three ways:

* hard bar ``|y - y64| <= C_E * E``: a gross error in an element is caught whatever the size of the other elements;
* statistical bar ``|y - y64| <= C_R * R``: the bf16x3 split (hi*hi + lo*hi + hi*lo, fp32 accumulation) leaves about 2^-17 R,
  while dropping one of the cross products leaves about 2^-9 R;
* exact zeros: where ``E == 0`` (a tap wholly in the padding, a sample whose operand is zero, input rows no tap reaches) the
  result must be exactly 0.0.

C_E = 2^-14 and C_R = 2^-12 are calibrated in tests/test_wgrad_bounds.py: the float32 emulation of the kernel passes both bars
with at least 4x headroom at the largest K of the GPU suite, and the statistical bar rejects each mutation of that emulation."""
import torch

C_E = 2.0 ** -14
C_R = 2.0 ** -12


def bounds(f, u, v):
    """``(f(u, v), f(|u|, |v|), sqrt(f(u^2, v^2)))`` in float64 on the CPU"""
    u, v = u.detach().cpu().double(), v.detach().cpu().double()
    return f(u, v), f(u.abs(), v.abs()), f(u * u, v * v).clamp_min(0).sqrt()


def check(y, y64, E, R, what, c_E=C_E, c_R=C_R):
    """assert the three bars on every element; prints and returns the worst (hard, statistical) ratio err / bound"""
    y = y.detach().cpu().double()
    assert tuple(y.shape) == tuple(y64.shape), f"{what}: shape {tuple(y.shape)} vs {tuple(y64.shape)}"
    assert torch.isfinite(y).all(), f"{what}: {int((~torch.isfinite(y)).sum())} non-finite elements"
    err = (y - y64).abs()
    zero = E == 0
    nonzero_in_zero = int((y[zero] != 0).sum())
    live = ~zero
    hard = (err[live] / (c_E * E[live])).max().item() if live.any() else 0.0
    stat = (err[live] / (c_R * R[live])).max().item() if live.any() else 0.0
    print(f"{what}: worst err/bound hard {hard:.3g} (c_E {c_E:.3g}) statistical {stat:.3g} (c_R {c_R:.3g}); "
          f"{int(zero.sum())} exact zeros")
    assert nonzero_in_zero == 0, f"{what}: {nonzero_in_zero} elements with E == 0 are not exactly 0"
    assert hard <= 1.0, f"{what}: hard bar exceeded by {hard:.3g}x"
    assert stat <= 1.0, f"{what}: statistical bar exceeded by {stat:.3g}x"
    return hard, stat


# ---------------------------------------------------------------------------------------------------------------------------
# the weight-gradient reduction in float64
# ---------------------------------------------------------------------------------------------------------------------------
def _gather(s, ys, xs):
    """``s[:, :, ys][:, :, :, xs]`` with zeros wherever an index is outside ``s``"""
    Hs, Ws = s.shape[2], s.shape[3]
    vy, vx = (ys >= 0) & (ys < Hs), (xs >= 0) & (xs < Ws)
    g = s[:, :, ys.clamp(0, Hs - 1)][:, :, :, xs.clamp(0, Ws - 1)]
    return g * (vy[:, None] & vx[None, :]).to(s.dtype)


def shifted(s, dy, dx, stride, Ha, Wa):
    """``S[b, n, stride * i + dy, stride * j + dx]`` over the A grid (i < Ha, j < Wa), zero outside S"""
    return _gather(s, stride * torch.arange(Ha) + dy, stride * torch.arange(Wa) + dx)


def wgrad(a, s, taps, stride, per_sample):
    """``a`` [B, M, Ha, Wa], ``s`` [B, N, Hs, Ws] (NCHW) -> ``[nb * M, N, T]``:
    ``out[m, n, t] = sum over b, i, j of a[b, m, i, j] * s[b, n, stride * i + dy_t, stride * j + dx_t]`` (nb = B per sample)"""
    B, M, Ha, Wa = a.shape
    out = []
    for dy, dx in taps:
        sh = shifted(s, dy, dx, stride, Ha, Wa)
        if per_sample:
            out.append(torch.einsum("bmhw,bnhw->bmn", a, sh).reshape(B * M, -1))
        else:
            out.append(torch.einsum("bmhw,bnhw->mn", a, sh))
    return torch.stack(out, -1)


# ---------------------------------------------------------------------------------------------------------------------------
# the kernel's arithmetic in float32 (calibration only: the GPU tests compare with the float64 reference above)
# ---------------------------------------------------------------------------------------------------------------------------
KPIX = 32
MUTATIONS = ("hihi", "drop_lo_a", "shift_tap", "drop_last_step", "wrong_parity", "drop_sample")


def _split(x):
    hi = x.to(torch.bfloat16).float()
    return hi, (x - hi).to(torch.bfloat16).float()


def emulate_wgrad(a, s, taps, stride, per_sample, splits, box_w, mutation=None):
    """float32 emulation of conv_wgrad_kernel + conv_wgrad_reduce_kernel: operands split into bf16(x) and bf16(x - hi); the three
    products of each 32-pixel K step (a box of box_w x 32 / box_w pixels of the A grid) summed exactly and rounded to fp32 once;
    fp32 accumulation step by step within a split (steps sample-major in the shared form); splits added in split order.
    Stride 2 reads the parity view of S the tap lands on, as the kernel does.  ``mutation`` (one of MUTATIONS) breaks the
    emulation in one way, on tap 0 where it concerns a tap."""
    a, s = a.float(), s.float()
    B, M, Ha, Wa = a.shape
    bh = KPIX // box_w
    tx, ty = -(-Wa // box_w), -(-Ha // bh)
    tiles = tx * ty
    Hp, Wp = ty * bh, tx * box_w
    ap = torch.zeros((B, M, Hp, Wp))
    ap[:, :, :Ha, :Wa] = a

    def steps(x):
        """[B, C, Hp, Wp] -> [B, C, tiles, 32] in the kernel's order: tile index ty * tiles_x + tx, pixels x-fastest in a box"""
        C = x.shape[1]
        x = x.reshape(B, C, ty, bh, tx, box_w).permute(0, 1, 2, 4, 3, 5)
        return x.reshape(B, C, tiles, KPIX)

    a_hi, a_lo = _split(steps(ap))
    partial = []
    for t, (dy, dx) in enumerate(taps):
        view, vx, vy = s, dx, dy
        if stride == 2:
            px, py = dx & 1, dy & 1
            vx, vy = (dx - px) // 2, (dy - py) // 2
            if mutation == "wrong_parity" and t == 0:
                px ^= 1
            view = s[:, :, py::2, px::2]
        if mutation == "shift_tap" and t == 0:
            vx += 1
        s_hi, s_lo = _split(steps(shifted(view, vy, vx, 1, Hp, Wp)))
        terms = [(a_hi, s_hi), (a_lo, s_hi), (a_hi, s_lo)]
        if mutation == "hihi":
            terms = terms[:1]
        elif mutation == "drop_lo_a":
            terms = [terms[0], terms[2]]
        p = sum(torch.einsum("bmkp,bnkp->bkmn", u.double(), v.double()) for u, v in terms).float()   # [B, tiles, M, N]
        partial.append(p)
    p = torch.stack(partial, -1)                                     # [B, tiles, M, N, T]
    if per_sample:
        p = p.permute(1, 0, 2, 3, 4)                                 # [ksteps, nb, M, N, T]
    else:
        p = p.reshape(B * tiles, 1, *p.shape[2:])                    # k = b * tiles + tile
    ksteps = p.shape[0]
    skip = set()
    if mutation == "drop_last_step":
        skip.add(ksteps - 1)
    if mutation == "drop_sample":
        assert not per_sample and B > 1
        skip.update(range((B - 1) * tiles, B * tiles))
    out = None
    for sp in range(splits):
        acc = torch.zeros(p.shape[1:], dtype=torch.float32)
        for k in range(ksteps * sp // splits, ksteps * (sp + 1) // splits):
            if k not in skip:
                acc = acc + p[k]
        out = acc if out is None else out + acc
    nb = out.shape[0]
    return out.reshape(nb * M, *out.shape[2:])


# ---------------------------------------------------------------------------------------------------------------------------
# plan() of csrc/conv_wgrad.cu, restated
# ---------------------------------------------------------------------------------------------------------------------------
SPLIT_TARGET = 132
MIN_SPLIT_STEPS = 16


def plan(B, M, N, a_h, a_w, taps, per_sample):
    """the planner's choices for a descriptor: nw from N, box_w from a_w, the split count from the work-item count and K steps"""
    nw = 32 if N <= 64 else 64 if N <= 128 else 128
    box_w = 32 if a_w > 16 else 16 if a_w > 8 else 8
    tiles = -(-a_w // box_w) * -(-a_h // (KPIX // box_w))
    ksteps = tiles if per_sample else tiles * B
    m_tiles, n_tiles = -(-M // 64), -(-N // (2 * nw))
    items0 = taps * m_tiles * n_tiles * (B if per_sample else 1)
    want = -(-SPLIT_TARGET // items0) if items0 < SPLIT_TARGET else 1
    cap = ksteps // MIN_SPLIT_STEPS
    splits = max(1, min(want, cap)) if items0 < SPLIT_TARGET else 1
    return dict(nw=nw, box_w=box_w, ksteps=ksteps, m_tiles=m_tiles, n_tiles=n_tiles, items0=items0, splits=splits,
                capped=items0 < SPLIT_TARGET and cap < want)
