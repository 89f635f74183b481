"""ctypes wrapper of the sky oracle (oracle/oracle_sky.cpp -> oracle/liboracle_sky.so), which tests/test_sky*.py use. The
library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_sky.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_sky.so")

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
        vp, i32, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint64
        L.oracle_sky_atmosphere.restype = i32
        L.oracle_sky_atmosphere.argtypes = [ctypes.POINTER(capi.IdkPtAtmosphereSettings), i32, vp, i32]
        L.oracle_sky_equirect.restype = i32
        L.oracle_sky_equirect.argtypes = [vp, i32, i32, vp, i32]
        L.oracle_sky_directions.restype = None
        L.oracle_sky_directions.argtypes = [i32, vp]
        L.oracle_det_atan2.restype = None
        L.oracle_det_atan2.argtypes = [vp, vp, u64, vp]
        L.oracle_det_asin.restype = None
        L.oracle_det_asin.argtypes = [vp, u64, vp]
        _lib = L
    return _lib


def atmosphere(settings, n, threads=None):
    """idkpt_sky_atmosphere on the CPU: faces float32 [6, n, n, 4]."""
    faces = np.zeros((6, n, n, 4), np.float32)
    assert lib().oracle_sky_atmosphere(ctypes.byref(settings), n, faces.ctypes.data, threads or ol.default_threads()) == 0
    return faces


def equirect(rgb, threads=None):
    """idkpt_sky_equirectangular on the CPU: rgb float32 [h, w, 3] -> faces float32 [6, w // 4, w // 4, 4]."""
    img = np.ascontiguousarray(rgb, np.float32)
    h, w = img.shape[:2]
    faces = np.zeros((6, w // 4, w // 4, 4), np.float32)
    assert lib().oracle_sky_equirect(img.ctypes.data, w, h, faces.ctypes.data, threads or ol.default_threads()) == 0
    return faces


def directions(n):
    """The fp32 texel directions of both kernels, float32 [6, n, n, 3]."""
    d = np.zeros((6, n, n, 3), np.float32)
    lib().oracle_sky_directions(n, d.ctypes.data)
    return d


def det_atan2(y, x):
    y, x = np.ascontiguousarray(y, np.float32), np.ascontiguousarray(x, np.float32)
    out = np.zeros(y.shape, np.float32)
    lib().oracle_det_atan2(y.ctypes.data, x.ctypes.data, y.size, out.ctypes.data)
    return out


def det_asin(x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(x.shape, np.float32)
    lib().oracle_det_asin(x.ctypes.data, x.size, out.ctypes.data)
    return out
