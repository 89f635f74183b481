"""ctypes wrapper of the G-buffer pass oracle (oracle/oracle_gbuffer.cpp in oracle/liboracle.so), which tests/test_gbuffer*.py
use."""
import ctypes

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi
from oracle_lib import lib

CHANNELS = (1, 2, 3, 2, 3, 2)   # depth, normal_rg, albedo, metallic_roughness, emissive, velocity_rg
STORE_R11G11 = 0                # oracle_gbuffer_store kinds
STORE_B10 = 1
STORE_RG8 = 2
STORE_RG16F = 3

def gbuffer(scene, frame, width, height, jitter=None, prev_positions=None, threads=None):
    """idkpt_gbuffer on the CPU -> (depth [h, w], normal_rg [h, w, 2], albedo [h, w, 3], metallic_roughness [h, w, 2],
    emissive [h, w, 3], velocity_rg [h, w, 2]), float32."""
    d, keep = capi.scene_desc(scene)
    fr = np.ascontiguousarray(frame)
    jit = None if jitter is None else np.ascontiguousarray(jitter, np.float32)
    prev = None if prev_positions is None else np.ascontiguousarray(prev_positions, np.float32)
    out = [np.zeros((height, width) if c == 1 else (height, width, c), np.float32) for c in CHANNELS]
    rc = lib().oracle_gbuffer(ctypes.byref(d), fr.ctypes.data, width, height, jit.ctypes.data if jit is not None else None,
                              prev.ctypes.data if prev is not None else None, *[a.ctypes.data for a in out],
                              threads or ol.default_threads())
    assert rc == 0, rc
    del keep
    return tuple(out)


def store(kind, values):
    """One attachment conversion (STORE_*) of float32 values, returned as float32."""
    v = np.ascontiguousarray(values, np.float32)
    out = np.zeros_like(v)
    lib().oracle_gbuffer_store(kind, v.ctypes.data, v.size, out.ctypes.data)
    return out
