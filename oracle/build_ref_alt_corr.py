"""oracle/build_ref_alt_corr.py — TEST INFRASTRUCTURE.  Compiles RAFT's alt_cuda_corr from the reference's sources where they lie
(/root/reference/model/raft/alt_cuda_corr/correlation{.cpp,_kernel.cu}, unmodified, nothing is copied) for sm_90a into
oracle/_ref/alt_cuda_corr/ with torch.utils.cpp_extension.  The resulting .so (git-ignored) is the reference yardstick of the on-demand
correlation kernel (vt_raft_corr_ondemand_f32; tests/test_gpu_raft_ondemand.py).  No-op when the reference checkout is absent."""
import os
import sys

SRC = "/root/reference/model/raft/alt_cuda_corr"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "alt_cuda_corr")
NAME = "alt_cuda_corr"


def build():
    if not os.path.isdir(SRC):
        print("oracle/build_ref_alt_corr.py: reference checkout not present: using the prebuilt oracle/_ref if any")
        return False
    if os.path.exists(os.path.join(OUT, NAME + ".so")):
        return True
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    os.makedirs(OUT, exist_ok=True)
    from torch.utils.cpp_extension import load
    load(NAME, sources=[os.path.join(SRC, s) for s in ("correlation.cpp", "correlation_kernel.cu")], build_directory=OUT,
         verbose=False, is_python_module=False)
    return True


def load_alt_corr():
    """-> the reference's alt_cuda_corr pybind module (``forward(fmap1, fmap2, coords, radius)``), or None when it was not built"""
    import importlib.util
    so = os.path.join(OUT, NAME + ".so")
    if not os.path.exists(so):
        return None
    import torch  # noqa: F401  (the extension links against torch's libraries)
    spec = importlib.util.spec_from_file_location(NAME, so)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


if __name__ == "__main__":
    sys.exit(0 if build() or True else 1)
