"""ctypes wrapper of the conservative-rasterisation oracle (oracle/oracle_vxgi_conservative.cpp in oracle/liboracle.so), which
tests/test_vxgi_conservative*.py and scripts/time_vxgi_conservative.py use."""
import ctypes

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi, vxgi
from oracle_lib import lib


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
    return ol.split_levels(raw, ci), raw, frags.value


def vx_voxelize_shadow_maps(scene, ci, shadows, maps, threads=None):
    """point_shadow_oracle.vx_voxelize_shadow_maps under the conservative rule: point-shadowed lights use the PCF lookup into
    `maps` (one uint16 [6, N, N] array per GpuPointShadow record). Returns (levels, raw chain, fragment count)."""
    sh, sizes, texels = ol.pack_shadow_maps(shadows, maps)
    assert len(sh) == len(maps) >= 1
    total = sum(w * h * d for w, h, d in vxgi.level_sizes(ci))
    raw = np.zeros(total * 4, np.uint16)
    d, keep = capi.scene_desc(scene)
    frags = ctypes.c_uint64()
    n = lib().oracle_vx_voxelize_conservative_shadow_maps(ctypes.byref(d), ctypes.byref(ci), sh.ctypes.data, sizes.ctypes.data,
                                                          texels.ctypes.data, len(sh), raw.ctypes.data, total, ctypes.byref(frags),
                                                          threads or ol.default_threads())
    assert n == len(vxgi.level_sizes(ci)), n
    return ol.split_levels(raw, ci), raw, frags.value
