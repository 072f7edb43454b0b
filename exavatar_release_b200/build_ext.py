"""Builds libb200raster.so (the C-ABI library of include/b200raster.h) in-tree with nvcc for the H100 (sm_90a), and the
compiled torch binding of the public call on top of it (_b2r_torch.so).

The .so files are build products (git-ignored); nvcc cross-compiles the library without a GPU.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libb200raster.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]  # Hopper (H100); the only architecture the kernels are tuned for
NVCC_FLAGS = [
    *ARCH,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--shared",
]


# Per-file flags.  project.cu holds the DECISION path of the projection (near-plane cull, radius = ceil(3 sqrt(lambda)),
# tile rect, pixel centre): compiled without fma contraction its arithmetic is, operation for operation, the oracle's C
# expression order (SURVEY.md section 7.2 "bit-compatible discrete decisions"), so radii / rects / centres are identical
# bit for bit instead of "equal except when 3 sqrt(lambda) lands within an ulp of an integer".  The kernel is
# latency-bound; the ~100 extra FP instructions per Gaussian do not show in its duration.
# binning.cu: its scatter repeats the projection's tile region test for rects of more than 32 tiles (smaller ones replay
# a stored mask); the two must agree on every (splat, tile) pair or a list slot stays unfilled, so the unit is compiled
# with the same contraction setting (its kernels are integer sorts otherwise).
# skin.cu: the posed positions feed every human render and their recorded outputs; fma contraction would move them in the
# last bits, so the unit keeps every product and sum rounded on its own.
# geometry.cu: the nearest-vertex search evaluates dx*dx + dy*dy + dz*dz exactly as its torch restatement does (three
# rounded products, two rounded sums), so the argmin -- ties included -- is the restatement's, index for index.
# mesh_raster.cu: the face render's coverage test and depth pz are, operation for operation, the float32 restatement's
# (mesh_render.face_render_reference), so the per-pixel face is identical to it instead of "equal except at ulp ties".
# regularizers.cu: the arm window |fl(l_x - u_x)| < 0.01f and the fp32 distances that pick the 50 nearest upper-arm rows
# are the reference's expressions rounded operation by operation, so the selection (ties included) is the reference's.
# smplx_rig.cu: the subdivision midpoints are fl(fl(a + b) * 0.5f) like pytorch3d's SubdivideMeshes, and the rig's
# outputs feed every human render, so no product or sum is contracted.
# adam.cu: the step is bit-identical to torch.optim.Adam's foreach kernels, which fuse exactly where their SASS has an
# FFMA; the kernel writes those as __fmaf_rn and every other product and sum stays rounded on its own.
# scene_assets.cu: clamp_min's mask (x >= 0 with x = fl(fl(C0 sh) + 0.5) at degree 0) and the activations are torch's
# fp32 expressions rounded operation by operation, so the mask agrees with torch's at equality.
# human_assets.cu: every forward output is ExAvatar's fp32 torch expression rounded operation by operation (the mask
# multiplies, exp / tanh as torch's kernels call them), bit-identical to it.
PER_FILE_FLAGS = {"project.cu": ["--fmad=false"], "binning.cu": ["--fmad=false"], "skin.cu": ["--fmad=false"],
                  "geometry.cu": ["--fmad=false"], "mesh_raster.cu": ["--fmad=false"],
                  "regularizers.cu": ["--fmad=false"], "smplx_rig.cu": ["--fmad=false"], "adam.cu": ["--fmad=false"],
                  "scene_assets.cu": ["--fmad=false"], "human_assets.cu": ["--fmad=false"]}


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(PKG, "..", "include", "b200raster.h"),
                                                                  os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, ptxas_info: bool = False) -> str:
    """Builds libb200raster.so and the compiled torch binding of the public call (`build_torch_ext`) when either is
    missing or stale; force=True rebuilds both."""
    # B2R_LIB_OUT + B2R_NVCC_EXTRA: a tuning variant of the same library next to the product one (load it with B2R_LIB)
    global LIB
    variant = os.environ.get("B2R_LIB_OUT")
    if variant:
        LIB = os.path.abspath(variant)
        force = True
    if force or _stale():
        _build_lib(force, verbose, ptxas_info, variant)
    if not variant:  # the binding links the in-tree library only
        build_torch_ext(force, verbose)
    return LIB


def _build_lib(force: bool, verbose: bool, ptxas_info: bool, variant) -> None:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("B2R_NVCC_EXTRA", "").split()  # e.g. -DB2_DRAIN_UNROLL=8 for tuning experiments
    # one object per translation unit, compiled in parallel (no relocatable device code: kernels never call across
    # files), then one link -- a full rebuild takes as long as the slowest file instead of the sum
    from concurrent.futures import ThreadPoolExecutor
    objdir = os.path.join(PKG, "build") if not variant else os.path.join(os.path.dirname(LIB), "obj_" + os.path.basename(LIB))
    os.makedirs(objdir, exist_ok=True)
    flags = [f for f in NVCC_FLAGS if f != "--shared"]
    srcs = sources()
    objs = [os.path.join(objdir, os.path.basename(s)[:-3] + ".o") for s in srcs]
    hdr_t = max(os.path.getmtime(d) for d in glob.glob(os.path.join(CSRC, "*.cuh")) +
                [os.path.join(PKG, "..", "include", "b200raster.h"), os.path.abspath(__file__)])  # flags live in this file

    def compile_one(pair):
        src, obj = pair
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), hdr_t) and not extra:
            return
        cmd = [nvcc, *flags, *PER_FILE_FLAGS.get(os.path.basename(src), []), *extra,
               *(["-Xptxas", "-v"] if ptxas_info else []), "-c", "-o", obj, src]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        list(ex.map(compile_one, zip(srcs, objs)))
    cmd = [nvcc, *ARCH, "--shared", "-o", LIB, *objs]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)


TORCH_EXT = os.path.join(PKG, "_b2r_torch.so")
TORCH_SRC = os.path.join(PKG, "csrc_torch", "b2r_torch.cpp")


def build_torch_ext(force: bool = False, verbose: bool = False) -> str:
    """The compiled torch binding of the public call (csrc_torch/b2r_torch.cpp): host code only, g++ against the torch
    headers of this interpreter, linked to the in-tree libb200raster.so next to it (rpath $ORIGIN), which `build()`
    makes first.  Rebuilt when older than its source, the C ABI header, this file or the library."""
    lib = os.path.join(PKG, "libb200raster.so")
    deps = [TORCH_SRC, os.path.join(PKG, "..", "include", "b200raster.h"), os.path.abspath(__file__), lib]
    if not force and os.path.exists(TORCH_EXT) and os.path.getmtime(TORCH_EXT) > max(os.path.getmtime(d) for d in deps):
        return TORCH_EXT
    import sysconfig

    import torch
    from torch.utils.cpp_extension import include_paths, library_paths
    cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    incs = [*include_paths("cuda"), os.path.join(cuda_home, "include"), sysconfig.get_paths()["include"],
            os.path.join(PKG, "..", "include")]
    libdirs = [*library_paths("cuda"), os.path.join(cuda_home, "lib64"), PKG]
    cmd = [os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-shared", "-DTORCH_EXTENSION_NAME=_b2r_torch",
           "-DTORCH_API_INCLUDE_EXTENSION_H", f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
           *[f"-I{os.path.abspath(i)}" for i in dict.fromkeys(incs)], TORCH_SRC, "-o", TORCH_EXT,
           *[f"-L{os.path.abspath(d)}" for d in dict.fromkeys(libdirs)], "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda",
           "-ltorch", "-ltorch_python", "-lcudart", f"-l:{os.path.basename(lib)}", "-Wl,-rpath,$ORIGIN",
           *[f"-Wl,-rpath,{os.path.abspath(d)}" for d in library_paths("cuda")]]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return TORCH_EXT


if __name__ == "__main__":
    build(force=True, verbose=True, ptxas_info="--ptxas" in sys.argv)
