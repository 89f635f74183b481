"""ctypes wrapper of the transparency oracle (oracle/oracle_transparency.cpp in oracle/liboracle.so), which
tests/test_transparency*.py use."""
import ctypes

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt
from oracle_lib import lib

LAYERS = 10


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
    sh, sizes, texels = ol.pack_shadow_maps(shadows if shadows is not None else np.zeros(0, gt.GpuPointShadow), maps)
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
