"""Build recipe for the oracle (TEST INFRASTRUCTURE ONLY -- see oracle/oracle.cpp header).

    python oracle/build.py        ->  oracle/liboracle.so

One library holds the whole checker: oracle/liboracle.cpp includes oracle.cpp and every pass oracle (oracle_*.cpp), and
tests/oracle_lib.py loads the result. The library is rebuilt when any oracle source or public header is newer than it.

The reference itself (C# + GLSL) cannot be compiled in this image (no dotnet/mono, no GL, no glslang), so there is
no oracle/_ref: the oracle is a CPU restatement ("port") and parity is unpinned by the reference (DESIGN.md).
"""
import glob
import os
import subprocess

ORACLE_DIR = os.path.dirname(os.path.abspath(__file__))
LIBORACLE = os.path.join(ORACLE_DIR, "liboracle.so")


def build(force=False, verbose=False):
    src = os.path.join(ORACLE_DIR, "liboracle.cpp")
    deps = [f for pattern in ("*.cpp", "*.inc") for f in glob.glob(os.path.join(ORACLE_DIR, pattern))] + \
        glob.glob(os.path.join(ORACLE_DIR, "..", "include", "*.h"))
    if not force and os.path.exists(LIBORACLE) and all(os.path.getmtime(d) <= os.path.getmtime(LIBORACLE) for d in deps):
        return LIBORACLE
    tmp = "%s.%d.tmp" % (LIBORACLE, os.getpid())
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
           "-fvisibility=hidden", "-o", tmp, src]
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    os.replace(tmp, LIBORACLE)    # a process that loads the library meanwhile sees the old file or the new one, never half of one
    return LIBORACLE


if __name__ == "__main__":
    print(build(force=True, verbose=True))
