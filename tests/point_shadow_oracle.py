"""ctypes wrapper of the point-shadow oracle (oracle/oracle_point_shadows.cpp -> oracle/liboracle_point_shadows.so), which
tests/test_point_shadows*.py use. The library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt, vxgi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_point_shadows.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_point_shadows.so")

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
        vp, i32, u32, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint32, ctypes.c_uint64
        L.oracle_point_shadow_render.restype = None
        L.oracle_point_shadow_render.argtypes = [ctypes.POINTER(capi.IdkPtSceneDesc), vp, i32, u32, vp]
        L.oracle_point_shadow_visibility.restype = None
        L.oracle_point_shadow_visibility.argtypes = [vp, i32, vp, vp, u64, vp]
        L.oracle_vx_voxelize_shadow_maps.restype = i32
        L.oracle_vx_voxelize_shadow_maps.argtypes = [ctypes.POINTER(capi.IdkPtSceneDesc), ctypes.POINTER(vxgi.IdkVxCreateInfo), vp, vp, vp, i32,
                                                     vp, u64, ctypes.POINTER(u64), i32]
        _lib = L
    return _lib


def _shadow(shadow):
    return np.ascontiguousarray(np.asarray(shadow, gt.GpuPointShadow).reshape(1))


def point_shadow_render(scene, shadow, size, face_mask=0x3F, inout=None):
    """One shadow's cube map, uint16 [6, size, size]; faces outside face_mask keep `inout`'s texels (default: 65535, a freshly
    cleared map)."""
    out = np.full((6, size, size), 65535, np.uint16) if inout is None else np.ascontiguousarray(inout, np.uint16).copy()
    d, keep = capi.scene_desc(scene)
    sh = _shadow(shadow)
    lib().oracle_point_shadow_render(ctypes.byref(d), sh.ctypes.data, size, face_mask, out.ctypes.data)
    return out


def point_shadow_visibility(shadow, cube_map, light_to_sample):
    """Visibility() for directions [M, 3] into a uint16 [6, N, N] map."""
    sh = _shadow(shadow)
    m = np.ascontiguousarray(cube_map, np.uint16)
    v = np.ascontiguousarray(light_to_sample, np.float32).reshape(-1, 3)
    out = np.zeros(len(v), np.float32)
    lib().oracle_point_shadow_visibility(sh.ctypes.data, m.shape[1], m.ctypes.data, v.ctypes.data, len(v), out.ctypes.data)
    return out


def vx_voxelize_shadow_maps(scene, ci, shadows, maps, threads=None):
    """Like oracle_lib.vx_voxelize, but point-shadowed lights use the PCF lookup into `maps` (one uint16 [6, N, N] array per
    GpuPointShadow record) instead of shadow rays. Returns (levels, raw chain, fragment count)."""
    sh = np.ascontiguousarray(shadows, gt.GpuPointShadow)
    assert len(sh) == len(maps) >= 1
    sizes = np.array([m.shape[1] for m in maps], np.int32)
    texels = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(m, np.uint16).ravel() for m in maps]))
    level_sizes = vxgi.level_sizes(ci)
    total = sum(w * h * d for w, h, d in level_sizes)
    raw = np.zeros(total * 4, np.uint16)
    d, keep = capi.scene_desc(scene)
    frags = ctypes.c_uint64()
    n = lib().oracle_vx_voxelize_shadow_maps(ctypes.byref(d), ctypes.byref(ci), sh.ctypes.data, sizes.ctypes.data, texels.ctypes.data,
                                             len(sh), raw.ctypes.data, total, ctypes.byref(frags), threads or ol.default_threads())
    assert n == len(level_sizes), n
    levels, off = [], 0
    for (w, h, dd) in level_sizes:
        k = w * h * dd * 4
        levels.append(raw[off:off + k].view(np.float16).reshape(dd, h, w, 4))
        off += k
    return levels, raw, frags.value
