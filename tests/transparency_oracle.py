"""ctypes wrapper of the transparency oracle (oracle/oracle_transparency.cpp -> oracle/liboracle_transparency.so), which
tests/test_transparency*.py use. The library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_transparency.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_transparency.so")
LAYERS = 10

_lib = None


def build(force=False):
    deps = [SRC] + [os.path.join(ORACLE_DIR, f) for f in ("oracle_deferred.cpp", "oracle_point_shadows.cpp", "oracle.cpp",
                                                           "oracle_vxgi.inc", "oracle_post.inc")] + \
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
        L.oracle_transparency.restype = i32
        L.oracle_transparency.argtypes = [ctypes.POINTER(capi.IdkPtSceneDesc), ctypes.POINTER(capi.IdkPtSkyDesc), vp, i32, i32,
                                          vp, vp, vp, i32, vp, vp, vp, vp, i32, i32, vp, i32, vp, vp, vp, vp, i32]
        _lib = L
    return _lib


def transparency(scene, frame, depth, color, shadow_mode=0, shadows=None, maps=(), jitter=None, sky=None, voxels=None,
                 bound=True, threads=None, layer_colors=False):
    """idkpt_transparency on the CPU. depth float32 [H, W]; color rgba32f [H, W, 4] (not modified); shadows (GpuPointShadow)
    with one uint16 [6, N, N] map each (ShadowMode 1); sky: capi.sky_desc(...) result or None (black); voxels: (IdkVxCreateInfo,
    concatenated rgba16f levels uint16, IdkVxConeSettings) for IsVXGI. Returns (composited float32 [H, W, 4], layers
    [H, W, LAYERS] structured (depth, tri, xf), kept counts int32 [H, W]); with layer_colors=True
    also the kept layers' premultiplied rgba16f colours, float32 [H, W, LAYERS, 4] (zero past the count)."""
    d, keep = capi.scene_desc(scene)
    fr = np.ascontiguousarray(frame)
    dep = np.ascontiguousarray(depth, np.float32)
    h, w = dep.shape
    out = np.array(color, np.float32, copy=True, order="C")
    assert out.shape == (h, w, 4)
    sh = np.ascontiguousarray(shadows if shadows is not None else np.zeros(0, gt.GpuPointShadow), gt.GpuPointShadow).reshape(-1)
    sizes = np.array([m.shape[1] for m in maps] or [0], np.int32)
    texels = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(m, np.uint16).ravel() for m in maps]) if maps else np.zeros(1, np.uint16))
    jit = None if jitter is None else np.ascontiguousarray(jitter, np.float32)
    sky_keep = sky
    sky_struct = sky[0] if isinstance(sky, tuple) else sky
    layers = np.zeros((h, w, LAYERS), [("depth", np.float32), ("tri", np.uint32), ("xf", np.uint32)])
    counts = np.zeros((h, w), np.int32)
    lc = np.zeros((h, w, LAYERS, 4), np.float32) if layer_colors else None
    ci, levels, cone = voxels if voxels is not None else (None, None, None)
    lv = None if levels is None else np.ascontiguousarray(levels, np.uint16)
    rc = lib().oracle_transparency(ctypes.byref(d), ctypes.byref(sky_struct) if sky_struct is not None else None, fr.ctypes.data,
                                   shadow_mode, int(voxels is not None), sh.ctypes.data if len(sh) else None, sizes.ctypes.data,
                                   texels.ctypes.data, len(sh), ctypes.addressof(ci) if ci is not None else None,
                                   lv.ctypes.data if lv is not None else None, ctypes.addressof(cone) if cone is not None else None,
                                   dep.ctypes.data, w, h, jit.ctypes.data if jit is not None else None, int(bound), out.ctypes.data,
                                   layers.ctypes.data, counts.ctypes.data,
                                   lc.ctypes.data if lc is not None else None, threads or ol.default_threads())
    assert rc == 0, rc
    del keep, sky_keep
    return (out, layers, counts, lc) if layer_colors else (out, layers, counts)
