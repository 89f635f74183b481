"""ctypes wrapper of the point-shadow oracle (oracle/oracle_point_shadows.cpp in oracle/liboracle.so), which
tests/test_point_shadows*.py use."""
import ctypes

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt, vxgi
from oracle_lib import lib


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
    sh, sizes, texels = ol.pack_shadow_maps(shadows, maps)
    assert len(sh) == len(maps) >= 1
    level_sizes = vxgi.level_sizes(ci)
    total = sum(w * h * d for w, h, d in level_sizes)
    raw = np.zeros(total * 4, np.uint16)
    d, keep = capi.scene_desc(scene)
    frags = ctypes.c_uint64()
    n = lib().oracle_vx_voxelize_shadow_maps(ctypes.byref(d), ctypes.byref(ci), sh.ctypes.data, sizes.ctypes.data, texels.ctypes.data,
                                             len(sh), raw.ctypes.data, total, ctypes.byref(frags), threads or ol.default_threads())
    assert n == len(level_sizes), n
    return ol.split_levels(raw, ci), raw, frags.value
