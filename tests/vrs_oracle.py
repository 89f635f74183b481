"""ctypes wrapper of the variable-rate deferred lighting oracle (oracle/oracle_vrs.cpp -> oracle/liboracle_vrs.so), which
tests/test_vrs*.py use. The library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

from idkengine_b200 import capi, gpu_types as gt

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_vrs.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_vrs.so")

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


_DEFERRED_ARGS = None


def lib():
    global _lib, _DEFERRED_ARGS
    if _lib is None:
        L = ctypes.CDLL(build())
        vp, i32, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint64
        _DEFERRED_ARGS = [vp, u64, vp, i32, vp, vp, vp, i32, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, i32]
        L.oracle_shading_rate.restype = i32
        L.oracle_shading_rate.argtypes = [vp, ctypes.POINTER(capi.IdkPtShadingRateSettings), vp, vp, i32, i32, vp, vp]
        L.oracle_deferred_lighting_vrs.restype = i32
        L.oracle_deferred_lighting_vrs.argtypes = _DEFERRED_ARGS + [vp, vp]
        L.oracle_deferred_samples.restype = i32
        L.oracle_deferred_samples.argtypes = _DEFERRED_ARGS + [vp, vp, u64, vp]
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def tiles_of(w, h):
    return (h + capi.VRS_TILE - 1) // capi.VRS_TILE, (w + capi.VRS_TILE - 1) // capi.VRS_TILE


def shading_rate(frame, settings, color, velocity, debug=False):
    """LightingShadingRateClassifier.Compute: color rgba32f [h, w, 4], velocity [h, w, 2] -> uint8 rates [ceil(h/16), ceil(w/16)],
    and with debug=True (DebugMode 2..4) also the float32 debug image: (rates, debug)."""
    c, v = _f32(color), _f32(velocity)
    h, w = v.shape[:2]
    fr = np.ascontiguousarray(frame)
    rates = np.zeros(tiles_of(w, h), np.uint8)
    dbg = np.zeros(tiles_of(w, h), np.float32) if debug else None
    rc = lib().oracle_shading_rate(fr.ctypes.data, ctypes.byref(settings), c.ctypes.data, v.ctypes.data, w, h, rates.ctypes.data,
                                   dbg.ctypes.data if debug else None)
    assert rc == 0, rc
    return (rates, dbg) if debug else rates


def _deferred_args(lights, frame, shadow_mode, shadows, maps, gbuffer, jitter, ssao, indirect, rt):
    """oracle_deferred_lighting's arguments, and the arrays to keep alive while they are used."""
    lt = np.ascontiguousarray(lights, gt.GpuLight)
    sh = np.ascontiguousarray(shadows, gt.GpuPointShadow).reshape(-1)
    assert len(sh) == len(maps)
    sizes = np.array([m.shape[1] for m in maps] or [0], np.int32)
    texels = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(m, np.uint16).ravel() for m in maps]) if maps else np.zeros(1, np.uint16))
    d, n, a, mr, e = [_f32(x) for x in gbuffer]
    h, w = d.shape
    fr = np.ascontiguousarray(frame)
    jit = None if jitter is None else _f32(jitter)
    ao = None if ssao is None else np.ascontiguousarray(ssao, np.uint8)
    gi = None if indirect is None else _f32(indirect)
    rts = [_f32(x) for x in (rt or [])]
    rt_ptrs = (ctypes.c_void_p * max(len(rts), 1))(*[x.ctypes.data for x in rts])
    keep = (lt, sh, sizes, texels, d, n, a, mr, e, fr, jit, ao, gi, rts, rt_ptrs)
    args = [lt.ctypes.data if len(lt) else None, len(lt), fr.ctypes.data, shadow_mode, sh.ctypes.data if len(sh) else None,
            sizes.ctypes.data, texels.ctypes.data, len(sh), d.ctypes.data, n.ctypes.data, a.ctypes.data, mr.ctypes.data, e.ctypes.data,
            w, h, jit.ctypes.data if jit is not None else None, ao.ctypes.data if ao is not None else None,
            gi.ctypes.data if gi is not None else None, rt_ptrs, len(rts)]
    return args, keep, (h, w)


def deferred_lighting_vrs(lights, frame, shadow_mode, shadows, maps, gbuffer, rates, jitter=None, ssao=None, indirect=None, rt=None):
    """The deferred lighting draw under a rate image (uint8 [ceil(H/16), ceil(W/16)] palette indices); the other arguments as
    deferred_oracle.deferred_lighting. -> float32 [H, W, 4]."""
    args, keep, (h, w) = _deferred_args(lights, frame, shadow_mode, shadows, maps, gbuffer, jitter, ssao, indirect, rt)
    r = np.ascontiguousarray(rates, np.uint8)
    assert r.shape == tiles_of(w, h)
    out = np.zeros((h, w, 4), np.float32)
    rc = lib().oracle_deferred_lighting_vrs(*args, r.ctypes.data, out.ctypes.data)
    assert rc == 0, rc
    del keep
    return out


def deferred_samples(lights, frame, shadow_mode, shadows, maps, gbuffer, img_coords, uvs, jitter=None, ssao=None, indirect=None, rt=None):
    """The fragment shader at samples: img_coords int [M, 2] (x, y), uvs float32 [M, 2] -> float32 [M, 4]."""
    args, keep, _ = _deferred_args(lights, frame, shadow_mode, shadows, maps, gbuffer, jitter, ssao, indirect, rt)
    ic = np.ascontiguousarray(img_coords, np.int32).reshape(-1, 2)
    uv = _f32(uvs).reshape(-1, 2)
    out = np.zeros((len(ic), 4), np.float32)
    rc = lib().oracle_deferred_samples(*args, ic.ctypes.data, uv.ctypes.data, len(ic), out.ctypes.data)
    assert rc == 0, rc
    del keep
    return out
