"""Builds csrc/libtetranerf_b200.so for sm_90a (H100) with nvcc, in-tree next to the sources."""
from __future__ import annotations

import os
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = CSRC / "libtetranerf_b200.so"
SOURCES = ["tn_api.cu", "tn_build.cu", "tn_trace.cu", "tn_ops.cu", "tn_find.cu", "tn_render.cu", "tn_mlp_debug.cu", "tn_walk.cu", "tn_faces.cu", "tn_surface.cu", "tn_normals.cu", "tn_ray_grads.cu", "tn_vertex_grads.cu", "tn_refine.cu", "tn_smoothness.cu", "tn_background.cu", "tn_fold_guard.cu", "tn_coarsen.cu", "tn_flip.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-shared"]


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [HERE.parent / "include" / "tetranerf_b200.h"]
    return any(p.stat().st_mtime > t for p in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    for src in SOURCES:  # compile translation units in parallel, then link
        obj = CSRC / (src[:-3] + ".o")
        objs.append(str(obj))
        cmd = ["nvcc", *FLAGS[:-1], *os.environ.get("TN_EXTRA_NVCC_FLAGS", "").split(), "-c", str(CSRC / src), "-o", str(obj)]  # extra flags: experiments only
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose:
            print(out)
    subprocess.run(["nvcc", *ARCH, "-shared", "-o", str(LIB), *objs], check=True)
    return LIB


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
