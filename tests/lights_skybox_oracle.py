"""ctypes wrapper of the light-sphere and skybox oracle (oracle/oracle_lights_skybox.cpp in oracle/liboracle.so), which
tests/test_lights_skybox*.py use."""
import ctypes

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi
from oracle_lib import lib

SPHERE_VERTICES, SPHERE_TRIANGLES = 169, 264
SKY = -2       # winner codes besides light * SPHERE_TRIANGLES + triangle
UNTOUCHED = -1

def sphere_mesh():
    """(vertices float32 [169, 3], indices uint32 [264, 3]) of the unit sphere."""
    v = np.zeros((SPHERE_VERTICES, 3), np.float32)
    i = np.zeros((SPHERE_TRIANGLES, 3), np.uint32)
    lib().oracle_sphere_mesh(v.ctypes.data, i.ctypes.data)
    return v, i


def lights_and_skybox(scene, frame, gbuffer, color, jitter=None, sky=None, threads=None):
    """idkpt_lights_and_skybox on the CPU over copies of gbuffer (the six planes of GBuffer) and color (the lit image [h, w, 4]):
    -> (gbuffer planes, color, winner int32 [h, w]) with winner = light * 264 + triangle, SKY or UNTOUCHED. sky: a constant
    colour (3-tuple) or cube-map faces [6, N, N, 4]; None = black."""
    d, keep = capi.scene_desc(scene)
    fr = np.ascontiguousarray(frame)
    g = [np.array(a, np.float32, copy=True, order="C") for a in gbuffer]
    col = np.array(color, np.float32, copy=True, order="C")
    h, w = g[0].shape
    winner = np.zeros((h, w), np.int32)
    jit = None if jitter is None else np.ascontiguousarray(jitter, np.float32)
    sd = None if sky is None else capi.sky_desc(sky)
    rc = lib().oracle_lights_skybox(ctypes.byref(d), ctypes.byref(sd) if sd is not None else None, fr.ctypes.data, w, h,
                                    jit.ctypes.data if jit is not None else None, g[0].ctypes.data, g[1].ctypes.data,
                                    g[4].ctypes.data, g[5].ctypes.data, col.ctypes.data, winner.ctypes.data,
                                    threads or ol.default_threads())
    assert rc == 0, rc
    del keep
    return tuple(g), col, winner
