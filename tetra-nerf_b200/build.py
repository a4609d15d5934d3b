"""Builds csrc/libtetranerf_b200.so for sm_90a (H100) with nvcc, in-tree next to the sources."""
from __future__ import annotations

import os
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = CSRC / "libtetranerf_b200.so"
SOURCES = ["tn_api.cu", "tn_build.cu", "tn_trace.cu", "tn_ops.cu", "tn_find.cu", "tn_render.cu", "tn_mlp_debug.cu", "tn_walk.cu", "tn_faces.cu"]
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


PYBIND_DIR = HERE / "tetranerf" / "utils" / "extension" / "_pybind"


def pybind_path() -> Path:
    import sysconfig

    return PYBIND_DIR / ("tetranerf_cpp_extension" + sysconfig.get_config_var("EXT_SUFFIX"))


def build_pybind(force: bool = False) -> Path:
    """The pybind11 module `tetranerf_cpp_extension` (csrc/py_binding.cpp, reference src/py_binding.cpp:433-449) over the C ABI:
    g++ against torch's headers, linked to libtetranerf_b200.so by a relative rpath; built in-tree next to the package."""
    import sysconfig

    import torch
    from torch.utils import cpp_extension as ce

    out = pybind_path()
    src = CSRC / "py_binding.cpp"
    hdr = HERE.parent / "include" / "tetranerf_b200.h"
    if not force and out.exists() and out.stat().st_mtime >= max(src.stat().st_mtime, hdr.stat().st_mtime):
        return out
    PYBIND_DIR.mkdir(parents=True, exist_ok=True)
    (PYBIND_DIR / "__init__.py").touch()
    tlib = Path(torch.__file__).resolve().parent / "lib"
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DTORCH_EXTENSION_NAME=tetranerf_cpp_extension", "-DTORCH_API_INCLUDE_EXTENSION_H",
           f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}", str(src), "-o", str(out)]
    for inc in ce.include_paths() + [sysconfig.get_paths()["include"], "/usr/local/cuda/include"]:
        cmd += ["-isystem", inc]
    cmd += [f"-L{CSRC}", "-ltetranerf_b200", f"-L{tlib}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
            "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath,$ORIGIN/../../../../csrc", f"-Wl,-rpath,{tlib}"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed on py_binding.cpp:\n" + r.stdout[-4000:])
    return out


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_pybind(force="--force" in sys.argv))
