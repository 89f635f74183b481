"""ctypes wrapper of the SSR / TAA oracle (oracle/oracle_ssr_taa.cpp -> oracle/liboracle_ssr_taa.so), which tests/test_ssr_taa*.py
use. The library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

from idkengine_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_ssr_taa.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_ssr_taa.so")

_lib = None


def build(force=False):
    deps = [SRC] + [os.path.join(ORACLE_DIR, f) for f in ("oracle_deferred.cpp", "oracle_point_shadows.cpp", "oracle.cpp", "oracle_vxgi.inc",
                                                          "oracle_post.inc")] + \
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
        vp, i32 = ctypes.c_void_p, ctypes.c_int32
        L.oracle_ssr.restype = i32
        L.oracle_ssr.argtypes = [vp, ctypes.POINTER(capi.IdkPtSsrSettings), ctypes.POINTER(capi.IdkPtSkyDesc), vp, vp, vp, vp, vp, i32, i32, vp, vp]
        L.oracle_taa_resolve.restype = i32
        L.oracle_taa_resolve.argtypes = [ctypes.POINTER(capi.IdkPtTaaSettings), vp, vp, vp, i32, i32, vp, i32, i32, vp]
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def ssr(frame, settings, sky, depth, normal_rg, albedo, metallic_roughness, src):
    """SSR.Compute + Merge Textures: G-buffer arrays, src rgba32f [H, W, 4], sky = capi.sky_desc(...) ->
    (merged float32 [H, W, 4], ssr float16 [H, W, 4])."""
    d, n, a, mr, s = _f32(depth), _f32(normal_rg), _f32(albedo), _f32(metallic_roughness), _f32(src)
    h, w = d.shape
    fr = np.ascontiguousarray(frame)
    out = np.zeros((h, w, 4), np.float16)
    merged = np.zeros((h, w, 4), np.float32)
    rc = lib().oracle_ssr(fr.ctypes.data, ctypes.byref(settings), ctypes.byref(sky), d.ctypes.data, n.ctypes.data, a.ctypes.data,
                          mr.ctypes.data, s.ctypes.data, w, h, out.ctypes.data, merged.ctypes.data)
    assert rc == 0, rc
    return merged, out


def taa_resolve(settings, color, depth, velocity, history):
    """One TaaResolve.Compute step: render-size color rgba32f [h, w, 4], depth [h, w], velocity [h, w, 2]; history float16
    [H, W, 4] (the previous step's output, zeros at the start) -> float16 [H, W, 4]."""
    c, d, v = _f32(color), _f32(depth), _f32(velocity)
    hist = np.ascontiguousarray(history, np.float16)
    rh, rw = d.shape
    H, W = hist.shape[:2]
    out = np.zeros((H, W, 4), np.float16)
    rc = lib().oracle_taa_resolve(ctypes.byref(settings), c.ctypes.data, d.ctypes.data, v.ctypes.data, rw, rh, hist.ctypes.data, W, H,
                                  out.ctypes.data)
    assert rc == 0, rc
    return out
