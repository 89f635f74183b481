"""ctypes wrapper of the variable-rate light-sphere and skybox oracle (oracle/oracle_lights_skybox_vrs.cpp), which
tests/test_lights_skybox_vrs*.py use."""
import ctypes

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi


def tiles_of(w, h):
    return (h + capi.VRS_TILE - 1) // capi.VRS_TILE, (w + capi.VRS_TILE - 1) // capi.VRS_TILE


def lights_and_skybox_vrs(scene, frame, gbuffer, color, rates, jitter=None, sky=None, threads=None):
    """idkpt_lights_and_skybox_vrs on the CPU over copies of gbuffer and color, under rates (uint8 [ceil(H/16), ceil(W/16)]
    palette indices); the other arguments and the result as lights_skybox_oracle.lights_and_skybox."""
    d, keep = capi.scene_desc(scene)
    fr = np.ascontiguousarray(frame)
    g = [np.array(a, np.float32, copy=True, order="C") for a in gbuffer]
    col = np.array(color, np.float32, copy=True, order="C")
    h, w = g[0].shape
    r = np.ascontiguousarray(rates, np.uint8)
    assert r.shape == tiles_of(w, h), (r.shape, tiles_of(w, h))
    winner = np.zeros((h, w), np.int32)
    jit = None if jitter is None else np.ascontiguousarray(jitter, np.float32)
    sd = None if sky is None else capi.sky_desc(sky)
    rc = ol.lib().oracle_lights_skybox_vrs(ctypes.byref(d), ctypes.byref(sd) if sd is not None else None, fr.ctypes.data, w, h,
                                          jit.ctypes.data if jit is not None else None, g[0].ctypes.data, g[1].ctypes.data,
                                          g[4].ctypes.data, g[5].ctypes.data, col.ctypes.data, winner.ctypes.data, r.ctypes.data,
                                          threads or ol.default_threads())
    assert rc == 0, rc
    del keep
    return tuple(g), col, winner


def fragment_of(rates, w, h):
    """Per pixel (x0, y0, cw, ch) of its coarse fragment: int [h, w, 4]."""
    cwh = np.array([[1, 1], [2, 1], [2, 2], [4, 2], [4, 4]])[np.repeat(np.repeat(np.asarray(rates), 16, 0), 16, 1)[:h, :w]]
    x, y = np.meshgrid(np.arange(w), np.arange(h))
    return np.stack([x - x % cwh[..., 0], y - y % cwh[..., 1], cwh[..., 0], cwh[..., 1]], -1)
