"""ctypes wrapper of the volumetric lighting oracle (oracle/oracle_volumetric.cpp -> oracle/liboracle_volumetric.so), which
tests/test_volumetric*.py use. The library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

from idkengine_b200 import capi, gpu_types as gt

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_volumetric.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_volumetric.so")

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
        vp, i32, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint64
        L.oracle_volumetric_lighting.restype = i32
        L.oracle_volumetric_lighting.argtypes = [vp, u64, vp, ctypes.POINTER(capi.IdkPtVolumetricSettings), vp, vp, vp, i32, vp, i32, i32,
                                                 i32, i32, vp, vp, vp, vp]
        L.oracle_volumetric_upscale.restype = None
        L.oracle_volumetric_upscale.argtypes = [vp, vp, i32, i32, vp, vp, i32, i32, i32, i32, vp]
        L.oracle_cube_nearest.restype = None
        L.oracle_cube_nearest.argtypes = [vp, i32, vp, u64, vp]
        _lib = L
    return _lib


def render_size(width, height, scale):
    """VolumetricLighting.SetSize: (Vector2i)((Vector2)PresentationResolution * ResolutionScale), truncated in float32."""
    s = np.float32(scale)
    return int(np.float32(width) * s), int(np.float32(height) * s)


def volumetric_lighting(lights, frame, settings, shadows, maps, depth, width, height, jitter=None):
    """VolumetricLighting.Compute: shadows (GpuPointShadow, LightIndex into `lights`) with one uint16 [6, N, N] map each, the
    G-buffer depth float32 [Hg, Wg]. Returns (uint16 [H, W, 4] result, uint16 [h, w, 4] render-size image, float32 [h, w]
    render-size depth)."""
    lt = np.ascontiguousarray(lights, gt.GpuLight)
    sh = np.ascontiguousarray(shadows, gt.GpuPointShadow).reshape(-1)
    assert len(sh) == len(maps)
    sizes = np.array([m.shape[1] for m in maps], np.int32)
    texels = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(m, np.uint16).ravel() for m in maps]) if maps else np.zeros(1, np.uint16))
    d = np.ascontiguousarray(depth, np.float32)
    fr = np.ascontiguousarray(frame)
    w, h = render_size(width, height, settings.ResolutionScale)
    out = np.zeros((height, width, 4), np.uint16)
    march = np.zeros((max(h, 1), max(w, 1), 4), np.uint16)
    mdepth = np.zeros((max(h, 1), max(w, 1)), np.float32)
    jit = None if jitter is None else np.ascontiguousarray(jitter, np.float32)
    rc = lib().oracle_volumetric_lighting(lt.ctypes.data if len(lt) else None, len(lt), fr.ctypes.data, ctypes.byref(settings),
                                          sh.ctypes.data if len(sh) else None, sizes.ctypes.data, texels.ctypes.data, len(sh),
                                          d.ctypes.data, d.shape[1], d.shape[0], width, height, jit.ctypes.data if jit is not None else None,
                                          out.ctypes.data, march.ctypes.data, mdepth.ctypes.data)
    assert rc == 0, rc
    return out, march, mdepth


def volumetric_upscale(frame, depth, march, march_depth, width, height):
    """The upscale dispatch alone: render-size uint16 [h, w, 4] rgba16f and float32 [h, w] depth -> uint16 [H, W, 4]."""
    d = np.ascontiguousarray(depth, np.float32)
    m = np.ascontiguousarray(march, np.uint16)
    md = np.ascontiguousarray(march_depth, np.float32)
    fr = np.ascontiguousarray(frame)
    out = np.zeros((height, width, 4), np.uint16)
    lib().oracle_volumetric_upscale(fr.ctypes.data, d.ctypes.data, d.shape[1], d.shape[0], m.ctypes.data, md.ctypes.data, m.shape[1], m.shape[0],
                                    width, height, out.ctypes.data)
    return out


def cube_nearest(cube_map, dirs):
    """The volumetric pass's texture(samplerCube, dir).r (NEAREST) for directions [M, 3] into a uint16 [6, N, N] map."""
    m = np.ascontiguousarray(cube_map, np.uint16)
    d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
    out = np.zeros(len(d), np.float32)
    lib().oracle_cube_nearest(m.ctypes.data, m.shape[1], d.ctypes.data, len(d), out.ctypes.data)
    return out
