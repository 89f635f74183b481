"""ctypes wrapper of the SSR / TAA oracle (oracle/oracle_ssr_taa.cpp in oracle/liboracle.so), which tests/test_ssr_taa*.py
use."""
import ctypes

import numpy as np

from oracle_lib import _f32, lib


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
