"""Builds libdgs_b200.so (the C-ABI shared library) in-tree with nvcc for sm_90a (H100).

    python open-diffusiongs_b200/csrc/build.py [--force] [--verbose]

Output: open-diffusiongs_b200/dgs_b200/lib/libdgs_b200.so (a build product, git-ignored).
No torch headers are involved: the library's boundary is plain C (include/dgs_b200.h).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
OUT_DIR = os.path.join(HERE, "..", "dgs_b200", "lib")
OUT = os.path.abspath(os.path.join(OUT_DIR, "libdgs_b200.so"))
SOURCES = ["core.cu", "raster.cu", "dit_glue.cu", "gemm_sm90.cu", "attention_sm90.cu", "attention_bwd_sm90.cu", "dit_api.cu", "diffusion_steps.cu", "lpips.cu", "ssim.cu", "geometry_loss.cu", "mesh.cu", "mesh_decimate.cu", "mesh_clean.cu", "mesh_remesh.cu", "mesh_color.cu", "mesh_render.cu", "knn.cu", "poisson.cu", "tsdf.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-O3"]
FILE_FLAGS = {  # their fp64 decisions round every product and sum, as their oracles do
    "mesh_clean.cu": ["-fmad=false"], "mesh_remesh.cu": ["-fmad=false"], "mesh_color.cu": ["-fmad=false"],
    "mesh_render.cu": ["-fmad=false"], "knn.cu": ["-fmad=false"], "poisson.cu": ["-fmad=false"],
    "tsdf.cu": ["-fmad=false"]}


def _stale(obj, deps):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    obj_dir = os.path.join(HERE, "build")
    os.makedirs(obj_dir, exist_ok=True)
    headers = [os.path.join(ROOT, "include", "dgs_b200.h")] + [
        os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".h", ".cuh"))]
    objs, procs = [], []
    for src in SOURCES:
        sp = os.path.join(HERE, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(obj_dir, src.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [sp] + headers):
            cmd = ["nvcc"] + NVCC_FLAGS + FILE_FLAGS.get(src, []) + ["-I", os.path.join(ROOT, "include"), "-I", HERE, "-c", sp, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            print(f"[dgs build] {src} FAILED:\n{out}")
        elif verbose and out.strip():
            print(out)
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or not os.path.exists(OUT):
        cmd = ["nvcc", "-shared", "-o", OUT] + objs + ["-lcudart", "-Xlinker", "--no-as-needed"]
        # cuTensorMapEncodeTiled & friends are resolved at run time through cudaGetDriverEntryPoint:
        # the library links only against libcudart so it also loads on a box without a driver.
        subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
