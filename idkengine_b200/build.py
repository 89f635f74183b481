"""Build helpers: compile the in-tree native libraries.

  libidkpt.so   -- the product: CUDA kernels for sm_90a (H100) + the C ABI (include/idkpt.h)
  libidkhost.so -- host-side mirror of the engine's C# BVH builder (no CUDA)

The oracle (oracle/) has its own recipe, oracle/build.py: it is test infrastructure and
is deliberately not built or referenced from this package.
"""
import os
import subprocess
import shutil

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_DIR = os.path.dirname(PKG_DIR)
INCLUDE_DIR = os.path.join(REPO_DIR, "include")

CSRC_DIR = os.path.join(PKG_DIR, "csrc")
HOST_DIR = os.path.join(PKG_DIR, "host_mirror")
LIBIDKPT = os.path.join(CSRC_DIR, "libidkpt.so")
LIBIDKHOST = os.path.join(HOST_DIR, "libidkhost.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    # Parity contract (DESIGN.md "Float semantics"): no FMA contraction, IEEE div/sqrt.
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-fvisibility=hidden",
    "-shared",
]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _sources(d, exts):
    out = []
    for root, _, files in os.walk(d):
        for f in sorted(files):
            if f.endswith(exts):
                out.append(os.path.join(root, f))
    return out


def find_nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: the CUDA toolkit is required to build libidkpt")
    return nvcc


def build_host(force=False, verbose=False):
    srcs = _sources(HOST_DIR, (".cpp",))
    deps = srcs + _sources(INCLUDE_DIR, (".h",))
    if not force and _newer(LIBIDKHOST, deps):
        return LIBIDKHOST
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-pthread",
           "-fvisibility=hidden", "-I", INCLUDE_DIR, "-o", LIBIDKHOST] + srcs
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    return LIBIDKHOST


def build_cuda(force=False, verbose=False, extra_flags=()):
    srcs = _sources(CSRC_DIR, (".cu",))
    deps = srcs + _sources(CSRC_DIR, (".cuh", ".h")) + _sources(INCLUDE_DIR, (".h",))
    if not force and _newer(LIBIDKPT, deps):
        return LIBIDKPT
    cmd = [find_nvcc()] + NVCC_FLAGS + list(extra_flags) + ["-I", INCLUDE_DIR, "-I", CSRC_DIR, "-o", LIBIDKPT] + srcs
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    return LIBIDKPT


def build_all(force=False, verbose=False):
    return build_host(force, verbose), build_cuda(force, verbose)


if __name__ == "__main__":
    import sys
    print(build_all(force="--force" in sys.argv, verbose=True))
