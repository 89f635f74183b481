"""ctypes wrapper of the variable-rate deferred lighting oracle (oracle/oracle_vrs.cpp in oracle/liboracle.so), which
tests/test_vrs*.py use."""
import ctypes

import numpy as np

from deferred_oracle import deferred_args
from idkengine_b200 import capi
from oracle_lib import _f32, lib


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


def deferred_lighting_vrs(lights, frame, shadow_mode, shadows, maps, gbuffer, rates, jitter=None, ssao=None, indirect=None, rt=None):
    """The deferred lighting draw under a rate image (uint8 [ceil(H/16), ceil(W/16)] palette indices); the other arguments as
    deferred_oracle.deferred_lighting. -> float32 [H, W, 4]."""
    args, keep, (h, w) = deferred_args(lights, frame, shadow_mode, shadows, maps, gbuffer, jitter, ssao, indirect, rt)
    r = np.ascontiguousarray(rates, np.uint8)
    assert r.shape == tiles_of(w, h)
    out = np.zeros((h, w, 4), np.float32)
    rc = lib().oracle_deferred_lighting_vrs(*args, r.ctypes.data, out.ctypes.data)
    assert rc == 0, rc
    del keep
    return out


def deferred_samples(lights, frame, shadow_mode, shadows, maps, gbuffer, img_coords, uvs, jitter=None, ssao=None, indirect=None, rt=None):
    """The fragment shader at samples: img_coords int [M, 2] (x, y), uvs float32 [M, 2] -> float32 [M, 4]."""
    args, keep, _ = deferred_args(lights, frame, shadow_mode, shadows, maps, gbuffer, jitter, ssao, indirect, rt)
    ic = np.ascontiguousarray(img_coords, np.int32).reshape(-1, 2)
    uv = _f32(uvs).reshape(-1, 2)
    out = np.zeros((len(ic), 4), np.float32)
    rc = lib().oracle_deferred_samples(*args, ic.ctypes.data, uv.ctypes.data, len(ic), out.ctypes.data)
    assert rc == 0, rc
    del keep
    return out
