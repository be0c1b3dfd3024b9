"""Build the UNMODIFIED reference CUDA extension into oracle/_ref/ (git-ignored).

TEST INFRASTRUCTURE ONLY.  Compiles <reference>/src/{gaussian.cu,bindings.cpp}
from where they lie (no source is copied into the repo) into
``oracle/_ref/gaussian_ref*.so``.  The only deviation from the reference's own
setup.py (setup.py:7-13) is build flags: ``-std=c++17`` instead of ``-std=c++14``
(torch >= 2.1 headers refuse C++14), an explicit sm_90a ``-gencode`` and the module
name ``gaussian_ref`` (``-DTORCH_EXTENSION_NAME``, so that it can be imported
next to our own ``gaussian`` module in one process).

The reference checkout is $GS_REFERENCE_DIR.  Tests and bench.py only load the built .so and the copied Python
files; nothing at test/bench time reads the sources.
The reference's pure-python files that the ``bench.py --impl reference`` arm and the drop-in tests
drive UNCHANGED (renderer.py, splatter.py, utils.py, train.py, visergui.py, transforms/) are copied next
to the .so at build time as build outputs (also git-ignored), never committed.
"""
import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("GS_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(HERE, "_ref")


def build(verbose: bool = False) -> str:
    """Returns the path of the built module, or '' when the reference is absent."""
    if not os.path.isdir(os.path.join(REF, "src")):
        return ""
    os.makedirs(OUT, exist_ok=True)
    suffix = sysconfig.get_config_var("EXT_SUFFIX")
    target = os.path.join(OUT, "gaussian_ref" + suffix)
    srcs = [os.path.join(REF, "src", "gaussian.cu"), os.path.join(REF, "src", "bindings.cpp")]
    if os.path.exists(target) and all(os.path.getmtime(target) >= os.path.getmtime(s) for s in srcs):
        _copy_glue()
        return target
    import torch
    from torch.utils import cpp_extension as ce

    inc = [f"-I{p}" for p in ce.include_paths("cuda")] + [f"-I{sysconfig.get_paths()['include']}"]
    # bindings.cpp includes "include/common.hpp" relative to its own directory: fine in place.
    common = ["-O3", "-std=c++17", "-DTORCH_EXTENSION_NAME=gaussian_ref",
              "-DTORCH_API_INCLUDE_EXTENSION_H", f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"]
    tmp = tempfile.mkdtemp(prefix="gs_ref_build_")   # private: a shared fixed path may belong to another user
    try:
        nvcc = os.path.join(ce.CUDA_HOME, "bin", "nvcc")
        o_cu = os.path.join(tmp, "gaussian.o")
        o_cpp = os.path.join(tmp, "bindings.o")
        cmds = [
            [nvcc, "-c", srcs[0], "-o", o_cu, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
             "--compiler-options", "-fPIC", "-w"] + common + inc,
            ["g++", "-c", srcs[1], "-o", o_cpp, "-fPIC", "-w"] + common + inc,
        ]
        procs = [subprocess.Popen(c, stdout=None if verbose else subprocess.DEVNULL) for c in cmds]
        codes = [p.wait() for p in procs]            # both finish before the directory is removed
        for code, c in zip(codes, cmds):
            if code != 0:
                raise RuntimeError("reference build failed: " + " ".join(c))
        libdirs = ce.library_paths("cuda")
        link = ["g++", "-shared", o_cu, o_cpp, "-o", target] + [f"-L{d}" for d in libdirs] + \
               [f"-Wl,-rpath,{d}" for d in libdirs] + \
               ["-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"]
        subprocess.check_call(link)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    _copy_glue()
    return target


def _copy_glue():
    for f in ("renderer.py", "splatter.py", "utils.py", "train.py", "visergui.py"):
        s = os.path.join(REF, f)
        if os.path.exists(s):
            shutil.copyfile(s, os.path.join(OUT, f))
    tdst = os.path.join(OUT, "transforms")
    if os.path.isdir(os.path.join(REF, "transforms")) and not os.path.isdir(tdst):
        shutil.copytree(os.path.join(REF, "transforms"), tdst)


if __name__ == "__main__":
    t = build(verbose=True)
    print("built:" if t else "reference sources not present; nothing built", t)
