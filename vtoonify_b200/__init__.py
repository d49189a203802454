"""vtoonify_b200 — H100-native (sm_90a) implementation of VToonify's per-frame StyleGAN2 synthesis hot path.

Drop-in surface (same names / signatures / state_dict keys as the reference):
  vtoonify_b200.op            <-> model/stylegan/op   (upfirdn2d, fused_leaky_relu, FusedLeakyReLU, conv2d_gradfix)
  vtoonify_b200.stylegan      <-> model/stylegan/model.py (ModulatedConv2d, StyledConv, ToRGB, Generator, ...)
  vtoonify_b200.dualstylegan  <-> model/dualstylegan.py
  vtoonify_b200.vtoonify      <-> model/vtoonify.py (VToonify)
  vtoonify_b200.frame_loop    <-> style_transfer.py frame loop (synthetic frames, pinned double-buffered I/O, multi-GPU shards)

All compute is hand-written CUDA in vtoonify_b200/csrc behind the C-ABI of include/vtoonify_b200.h.
"""
from . import _lib  # noqa: F401
from .ops import get_precision, set_precision  # noqa: F401

__all__ = ["set_precision", "get_precision", "install_as_reference_ops"]


def install_as_reference_ops():
    """Make ``import model.stylegan.op`` (as done at model/stylegan/model.py:11) resolve to this package's ops,
    the non-invasive equivalent of the edit prescribed by model/stylegan/op_cpu/readme.md."""
    import sys
    from . import op
    sys.modules["model.stylegan.op"] = op
    sys.modules["model.stylegan.op.conv2d_gradfix"] = op.conv2d_gradfix
    return op
