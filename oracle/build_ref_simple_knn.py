"""oracle/build_ref_simple_knn.py -- TEST INFRASTRUCTURE: compile the UNMODIFIED reference simple_knn extension.

Recipe (no reference source is copied into this repo): torch's cpp_extension compiles the reference's own files where
they lie under <reference checkout>/submodules/simple-knn (ext.cpp, spatial.cu, simple_knn.cu) for sm_90a, with the
reference's default nvcc flags (so its squared distances contract to FMAs), into oracle/_ref/simple_knn_ref_C.so
(git-ignored), the way oracle/build_ref.py builds the rasterizer.  The module exports distCUDA2 (ext.cpp), which
tests/test_poisson_gpu.py and tests/perf_poisson.py compare and time next to simple_knn._C.distCUDA2.
"""
import importlib.util
import os
import sys

from oracle.build_ref import OUT, REF_ROOT

NAME = "simple_knn_ref_C"
REF = os.path.join(REF_ROOT, "submodules", "simple-knn")


def so_path():
    return os.path.join(OUT, NAME + ".so")


def build(force: bool = False):
    """Build if the reference tree is present; returns the .so path, or None (with a message) when there is none."""
    if os.path.exists(so_path()) and not force:
        return so_path()
    if not os.path.isdir(REF):
        print(f"[build_ref_simple_knn] no reference simple-knn at {REF} (set DGS_REFERENCE_ROOT): not built")
        return None
    os.makedirs(OUT, exist_ok=True)
    from torch.utils.cpp_extension import load
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    load(name=NAME, sources=[os.path.join(REF, f) for f in ("ext.cpp", "spatial.cu", "simple_knn.cu")],
         build_directory=OUT, is_python_module=False, verbose=False, extra_include_paths=[REF],
         extra_cflags=["-O3"], extra_cuda_cflags=["-O3", "-gencode", "arch=compute_90a,code=sm_90a",
                                                  "-Xcompiler", "-fno-gnu-unique"])
    return so_path() if os.path.exists(so_path()) else None


def load_module():
    """Import the prebuilt reference extension (needs torch imported first); None if absent."""
    p = so_path()
    if not os.path.exists(p):
        return None
    import torch  # noqa: F401  (the .so links against libtorch)
    if NAME in sys.modules:
        return sys.modules[NAME]
    spec = importlib.util.spec_from_file_location(NAME, p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[NAME] = mod
    return mod


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
