"""In-tree build of the native pieces (no JIT cache: the .so files live in the source tree, so that a
copy of the built tree runs on another machine without compiling again).

    libblance_b200.so   nvcc, sm_90a (H100) only: the CUDA kernels + the C ABI (include/blance_b200.h)
    _host*.so           g++: the C++ host mirror of blance's api.go (pybind11 face), linked
                        against libblance_b200.so

Rebuilds only when a source is newer than its output."""
import glob
import os
import subprocess
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
INCLUDE = os.path.join(ROOT, "include")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
              "-fmad=false",           # the score of plan.go:634-689 is never fused
              "-Xcompiler", "-fPIC", "-shared", "-cudart", "static"]


def _newer(srcs, out):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(s) > t for s in srcs)


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s" % (" ".join(cmd), r.stdout))
    return r.stdout


def lib_path():
    return os.path.join(LIBDIR, "libblance_b200.so")


def host_module_path():
    return os.path.join(HERE, "_host" + sysconfig.get_config_var("EXT_SUFFIX"))


def build_cuda_lib(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = [os.path.join(CSRC, "c_abi.cu")]
    deps = srcs + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(INCLUDE, "blance_b200.h")]
    out = lib_path()
    if force or _newer(deps, out):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-I" + INCLUDE, "-I" + CSRC] + srcs + ["-o", out]
        log = _run(cmd)
        if verbose:
            print(log)
    return out


def build_host_module(force=False):
    import pybind11
    out = host_module_path()
    srcs = [os.path.join(CSRC, "host_api.cpp"), os.path.join(CSRC, "py_module.cpp")]
    deps = srcs + [os.path.join(CSRC, "host_api.hpp"), os.path.join(INCLUDE, "blance_b200.h"), lib_path()]
    if force or _newer(deps, out):
        cxx = os.environ.get("CXX", "g++")
        cmd = [cxx, "-O2", "-std=c++17", "-pthread", "-fPIC", "-shared", "-fvisibility=hidden",
               "-I" + INCLUDE, "-I" + CSRC, "-I" + sysconfig.get_paths()["include"], "-I" + pybind11.get_include()] + srcs + \
              ["-L" + LIBDIR, "-lblance_b200", "-Wl,-rpath,$ORIGIN/lib", "-o", out]
        _run(cmd)
    return out


def build_all(force=False, verbose=False):
    build_cuda_lib(force, verbose)
    build_host_module(force)


if __name__ == "__main__":
    import sys
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(lib_path())
    print(host_module_path())
