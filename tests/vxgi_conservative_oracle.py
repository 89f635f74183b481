"""ctypes wrapper of the conservative-rasterisation oracle (oracle/oracle_vxgi_conservative.cpp ->
oracle/liboracle_vxgi_conservative.so), which tests/test_vxgi_conservative*.py and scripts/time_vxgi_conservative.py use. The
library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt, vxgi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_vxgi_conservative.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_vxgi_conservative.so")

_lib = None


def build(force=False):
    deps = [SRC] + [os.path.join(ORACLE_DIR, f) for f in ("oracle_point_shadows.cpp", "oracle.cpp", "oracle_vxgi.inc", "oracle_post.inc")] + \
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
        P = ctypes.POINTER
        vp, i32, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint64
        L.oracle_vx_voxelize_conservative.restype = i32
        L.oracle_vx_voxelize_conservative.argtypes = [P(capi.IdkPtSceneDesc), P(vxgi.IdkVxCreateInfo), vp, u64, P(u64), i32]
        L.oracle_vx_voxelize_conservative_shadow_maps.restype = i32
        L.oracle_vx_voxelize_conservative_shadow_maps.argtypes = [P(capi.IdkPtSceneDesc), P(vxgi.IdkVxCreateInfo), vp, vp, vp, i32,
                                                                  vp, u64, P(u64), i32]
        _lib = L
    return _lib


def _split(raw, ci):
    levels, off = [], 0
    for (w, h, d) in vxgi.level_sizes(ci):
        k = w * h * d * 4
        levels.append(raw[off:off + k].view(np.float16).reshape(d, h, w, 4))
        off += k
    return levels


def vx_voxelize(scene, ci, threads=None):
    """oracle_lib.vx_voxelize under the conservative rule (point-shadowed lights by shadow rays). Returns (list of float16
    [d, h, w, 4] arrays per level, concatenated raw uint16 chain, fragment count)."""
    total = sum(w * h * d for w, h, d in vxgi.level_sizes(ci))
    raw = np.zeros(total * 4, np.uint16)
    d, keep = capi.scene_desc(scene)
    frags = ctypes.c_uint64()
    n = lib().oracle_vx_voxelize_conservative(ctypes.byref(d), ctypes.byref(ci), raw.ctypes.data, total, ctypes.byref(frags),
                                              threads or ol.default_threads())
    assert n == len(vxgi.level_sizes(ci)), n
    return _split(raw, ci), raw, frags.value


def vx_voxelize_shadow_maps(scene, ci, shadows, maps, threads=None):
    """point_shadow_oracle.vx_voxelize_shadow_maps under the conservative rule: point-shadowed lights use the PCF lookup into
    `maps` (one uint16 [6, N, N] array per GpuPointShadow record). Returns (levels, raw chain, fragment count)."""
    sh = np.ascontiguousarray(shadows, gt.GpuPointShadow)
    assert len(sh) == len(maps) >= 1
    sizes = np.array([m.shape[1] for m in maps], np.int32)
    texels = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(m, np.uint16).ravel() for m in maps]))
    total = sum(w * h * d for w, h, d in vxgi.level_sizes(ci))
    raw = np.zeros(total * 4, np.uint16)
    d, keep = capi.scene_desc(scene)
    frags = ctypes.c_uint64()
    n = lib().oracle_vx_voxelize_conservative_shadow_maps(ctypes.byref(d), ctypes.byref(ci), sh.ctypes.data, sizes.ctypes.data,
                                                          texels.ctypes.data, len(sh), raw.ctypes.data, total, ctypes.byref(frags),
                                                          threads or ol.default_threads())
    assert n == len(vxgi.level_sizes(ci)), n
    return _split(raw, ci), raw, frags.value
