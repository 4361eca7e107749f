"""Build libgpsg_sm90.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python gps-gaussian_b200/build.py [--force] [--verbose]

Output: gps-gaussian_b200/lib/libgpsg_sm90.so (git-ignored build product).
build(defines=[...], out=path) compiles the same sources with extra -D macros (instrumented variants such as
GPSG_SORT_PHASES, see tools/sort_phases.py) into their own object directory and library.
raster_preprocess.cu is compiled with -fmad=false (see its header): the fp32 op order that decides
radii / tile rectangles must not be FMA-contracted.  rectify.cu likewise: its fp32 / fp64 op order is what makes
the rectified images and flow bit-identical to OpenCV.  mesh_render.cu likewise: its fp32 op order is the mesh oracle's.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libgpsg_sm90.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
          "--expt-relaxed-constexpr", "-Xptxas", "-v"]
SOURCES = {
    "gpsg_capi.cu": [],
    "raster_preprocess.cu": ["-fmad=false"],
    "raster_binning.cu": [],
    "raster_render.cu": [],
    "raster_backward.cu": [],
    "corr.cu": [],
    "corr_tc.cu": [],
    "sh.cu": [],
    "unproject.cu": [],
    "loss.cu": [],
    "point_splat.cu": [],
    "rectify.cu": ["-fmad=false"],
    "flow_head.cu": [],
    "gs_head.cu": [],
    "encoder_stem.cu": [],
    "encoder_down.cu": [],
    "decoder1.cu": [],
    "decoder23.cu": [],
    "update_block.cu": [],
    "mesh_render.cu": ["-fmad=false"],
    "jpeg_decode.cu": [],
    "jpeg_encode.cu": [],
}


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _deps(src):
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(os.path.dirname(HERE), "include", "gpsg.h"))
    return [src, os.path.abspath(__file__)] + hdrs


def _stale(dst, deps):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(name, extra, objdir, force, verbose):
    src = os.path.join(CSRC, name)
    obj = os.path.join(objdir, name.replace(".cu", ".o"))
    if not force and not _stale(obj, _deps(src)):
        return obj, ""
    cmd = [_nvcc()] + ARCH + COMMON + extra + ["-c", src, "-o", obj]
    p = subprocess.run(cmd, capture_output=True, text=True)
    log = " ".join(cmd) + "\n" + p.stdout + p.stderr
    if p.returncode != 0:
        raise RuntimeError(log)
    with open(obj + ".log", "w") as f:
        f.write(log)
    if verbose:
        print(log)
    return obj, log


def build(force=False, verbose=False, defines=(), out=None):
    objdir = os.path.join(OBJ, "_".join(defines)) if defines else OBJ
    lib = out or LIB
    flags = ["-D" + d for d in defines]
    os.makedirs(objdir, exist_ok=True)
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        res = list(ex.map(lambda kv: _compile(kv[0], kv[1] + flags, objdir, force, verbose), SOURCES.items()))
    objs = [r[0] for r in res]
    if force or _stale(lib, objs):
        cmd = [_nvcc()] + ARCH + ["-shared", "-o", lib] + objs + ["-Xcompiler", "-fvisibility=hidden", "-cudart",
                                                                  "static"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError(" ".join(cmd) + "\n" + p.stdout + p.stderr)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
