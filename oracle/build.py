"""Build the CPU oracle shared libraries and stage the original project (test infrastructure, not product).

    python oracle/build.py            # builds oracle/_build/liboracle_{f32,f64}.so, stages oracle/_ref/

The reference's rasterizer source (graphdeco-inria/diff-gaussian-rasterization) and
sampler source (princeton-vl/RAFT-Stereo/sampler) are not in the original project's tree, so
nothing of the reference compiles from its own sources (it is pure Python; see DESIGN.md "Oracle").  What
`oracle/_ref/` holds instead is the original project's tree itself, copied byte for byte from the checkout named by
GPSG_REFERENCE (default /root/reference) when one exists: the C3 harness (gps_gaussian_b200/harness.py, tests/test_c3_gpu.py,
bench.py's train_c3 block) runs the reference's own model and scripts from there against the drop-ins.  oracle/_ref/ is
git-ignored; where no checkout exists an earlier staging is kept and otherwise nothing is staged.
"""
import os
import shutil
import stat
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build")
REF_OUT = os.path.join(HERE, "_ref")
REFERENCE = os.environ.get("GPSG_REFERENCE", "/root/reference")
SRCS = ["gpsg_oracle.c", "corr_oracle.c", "taichi_splat_oracle.c"]


def _newer(dst, srcs):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(s) > t for s in srcs)


def stage_reference(force=False):
    """Copy the original project's tree to oracle/_ref (once). Returns the staged path, or None when neither the checkout
    nor an earlier staging exists."""
    marker = os.path.join(REF_OUT, "train_stage2.py")
    if os.path.isfile(os.path.join(REFERENCE, "train_stage2.py")) and (force or not os.path.exists(marker)):
        if os.path.isdir(REF_OUT):
            shutil.rmtree(REF_OUT)
        shutil.copytree(REFERENCE, REF_OUT, ignore=shutil.ignore_patterns(".git", "__pycache__", "*.pyc"))
        for d, _, files in os.walk(REF_OUT):            # a read-only checkout keeps its modes through copytree
            for p in [d] + [os.path.join(d, f) for f in files]:
                os.chmod(p, os.stat(p).st_mode | stat.S_IWUSR)
    return REF_OUT if os.path.exists(marker) else None


def build(force=False, verbose=False):
    stage_reference(force)
    os.makedirs(OUT, exist_ok=True)
    srcs = [os.path.join(HERE, s) for s in SRCS if os.path.exists(os.path.join(HERE, s))]
    outs = {}
    for tag, defs in (("f32", []), ("f64", ["-DORACLE_F64"])):
        dst = os.path.join(OUT, f"liboracle_{tag}.so")
        outs[tag] = dst
        if not force and not _newer(dst, srcs + [os.path.abspath(__file__)]):
            continue
        # -ffp-contract=off: no FMA contraction, so fp32 results follow the written op order
        cmd = ["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
               "-Wall", "-Wno-unused-function"] + defs + srcs + ["-lm", "-o", dst]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return outs


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
