"""In-tree build of the native code (sm_90a: H100).

  libgs_b200.so                      hand-written CUDA kernels + the C ABI of include/gs_b200.h
                                     (no libtorch dependency; links cudart statically)
  gaussian.cpython-*.so              torch/pybind11 shim == the reference's `gaussian` module
                                     surface (reference setup.py:33-52 builds the equivalent)

Both land next to this file, so the package imports from the source tree; objects go to
`build/` (git-ignored).  Usage:  python build.py [--force] [-v]
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CU_SOURCES = ["project.cu", "binning.cu", "blend.cu", "blend_sh.cu", "blend_sh_tc.cu", "render.cu", "optim.cu", "collective.cu", "loss.cu", "densify.cu",
              "densify_stats.cu", "blend_feat.cu", "mcmc.cu", "filter3d.cu", "surfel.cu", "blend_surfel.cu", "scores.cu"]
HEADERS = ["gs_common.cuh", "sh_common.cuh", "tc_common.cuh", "project.cuh", "internal.h", os.path.join(ROOT, "include", "gs_b200.h")]
LIB = os.path.join(HERE, "libgs_b200.so")
EXT = os.path.join(HERE, "gaussian" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build step failed:\n" + " ".join(cmd) + "\n" + r.stdout)
    if verbose and r.stdout.strip():
        print(r.stdout)


def build_lib(force=False, verbose=False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    hdrs = [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    objs, jobs = [], []
    for src in CU_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(o, [s] + hdrs):
            jobs.append([NVCC, "-c", s, "-o", o, "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"] + ARCH)
    with ThreadPoolExecutor(max_workers=4) as ex:
        list(ex.map(lambda c: _run(c, verbose), jobs))
    if force or jobs or _newer(LIB, objs):
        _run([NVCC, "-shared", "-o", LIB] + objs + ARCH + ["-cudart", "static", "-Xcompiler", "-fPIC"], verbose)
    return LIB


def build_ext(force=False, verbose=False) -> str:
    import torch
    from torch.utils import cpp_extension as ce

    lib = build_lib(force, verbose)
    src = os.path.join(CSRC, "bindings.cpp")
    if not (force or _newer(EXT, [src, lib, os.path.join(ROOT, "include", "gs_b200.h")])):
        return EXT
    inc = [f"-I{p}" for p in ce.include_paths("cuda")] + [f"-I{sysconfig.get_paths()['include']}"]
    libdirs = ce.library_paths("cuda")
    cmd = (["g++", "-shared", "-fPIC", "-O2", "-std=c++17", "-w", src, "-o", EXT,
            "-DTORCH_EXTENSION_NAME=gaussian", "-DTORCH_API_INCLUDE_EXTENSION_H",
            f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"] + inc +
           [f"-L{HERE}", "-lgs_b200", "-Wl,-rpath,$ORIGIN"] +
           [f"-L{d}" for d in libdirs] + [f"-Wl,-rpath,{d}" for d in libdirs] +
           ["-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"])
    _run(cmd, verbose)
    return EXT


def build_all(force=False, verbose=False):
    return build_lib(force, verbose), build_ext(force, verbose)


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
