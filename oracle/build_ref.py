"""oracle/build_ref.py — TEST / BASELINE INFRASTRUCTURE.  Compiles the reference's own two CUDA ops for sm_90a from the sources
where they lie (/root/reference/model/stylegan/op/{upfirdn2d,fused_bias_act}*.{cpp,cu}, unmodified, nothing is copied) into
oracle/_ref/ with torch.utils.cpp_extension (the same loader the reference uses at import: op/upfirdn2d.py:11-17,
op/fused_act.py:11-17).  The resulting .so files (git-ignored) give bench.py --impl cudnn the reference's real CUDA path for the
blur / activation ops.  No-op when the reference checkout is absent."""
import os
import sys

REF = "/root/reference/model/stylegan/op"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def build():
    if not os.path.isdir(REF):
        print("oracle/build_ref.py: reference checkout not present: using the prebuilt oracle/_ref if any")
        return False
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    os.makedirs(OUT, exist_ok=True)
    from torch.utils.cpp_extension import load
    for name, srcs in (("upfirdn2d", ["upfirdn2d.cpp", "upfirdn2d_kernel.cu"]), ("fused", ["fused_bias_act.cpp", "fused_bias_act_kernel.cu"])):
        bdir = os.path.join(OUT, name)
        os.makedirs(bdir, exist_ok=True)
        if os.path.exists(os.path.join(bdir, name + ".so")):
            continue
        load(name, sources=[os.path.join(REF, s) for s in srcs], build_directory=bdir, verbose=False, is_python_module=False)
    return True


def load_ops():
    """-> (upfirdn2d_op, fused) pybind modules of the reference, or None when they were not built"""
    import importlib.util
    mods = []
    for name in ("upfirdn2d", "fused"):
        so = os.path.join(OUT, name, name + ".so")
        if not os.path.exists(so):
            return None
        spec = importlib.util.spec_from_file_location(name, so)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        mods.append(m)
    return tuple(mods)


if __name__ == "__main__":
    sys.exit(0 if build() or True else 1)
