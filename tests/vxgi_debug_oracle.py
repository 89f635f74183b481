"""ctypes wrapper of the grid-visualisation oracle (oracle/oracle_vxgi_debug.cpp -> oracle/liboracle_vxgi_debug.so), which
tests/test_vxgi_debug*.py use. The library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_lib as ol

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_vxgi_debug.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_vxgi_debug.so")

_lib = None


def build(force=False):
    deps = [SRC] + [os.path.join(ORACLE_DIR, f) for f in ("oracle.cpp", "oracle_vxgi.inc", "oracle_post.inc")] + \
        [os.path.join(REPO, "include", f) for f in ("idkpt.h", "idkvx.h", "idk_gpu_types.h")]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    tmp = LIB + ".%d.tmp" % os.getpid()
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                    "-fvisibility=hidden", "-o", tmp, SRC], check=True)
    os.replace(tmp, LIB)
    return LIB


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        vp = ctypes.c_void_p
        L.oracle_vx_debug_render.restype = ctypes.c_int32
        L.oracle_vx_debug_render.argtypes = [vp, vp, vp, vp, ctypes.c_float, ctypes.c_float, ctypes.c_int32, ctypes.c_int32, vp,
                                             ctypes.POINTER(ctypes.c_uint64), ctypes.c_int32]
        _lib = L
    return _lib


def debug_render(ci, raw_chain, frame, step_multiplier, cone_angle, width, height, sky=None, threads=None):
    """Voxelizer.DebugRender on the CPU. raw_chain: the grid's rgba16f levels back to back (uint16 or float16); sky:
    capi.sky_desc(...) result or None (black). Returns (image float32 [h, w, 4], cone samples)."""
    raw = np.ascontiguousarray(np.asarray(raw_chain).view(np.uint16).reshape(-1))
    fr = np.ascontiguousarray(frame)
    out = np.zeros((height, width, 4), np.float32)
    steps = ctypes.c_uint64()
    rc = lib().oracle_vx_debug_render(ctypes.addressof(ci), raw.ctypes.data, ctypes.addressof(sky) if sky is not None else None,
                                      fr.ctypes.data, float(step_multiplier), float(cone_angle), width, height, out.ctypes.data,
                                      ctypes.byref(steps), threads or ol.default_threads())
    assert rc == 0, rc
    return out, steps.value
