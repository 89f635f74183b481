"""ctypes wrapper of the grid-visualisation oracle (oracle/oracle_vxgi_debug.cpp in oracle/liboracle.so), which
tests/test_vxgi_debug*.py use."""
import ctypes

import numpy as np

import oracle_lib as ol
from oracle_lib import lib


def debug_render(ci, raw_chain, frame, step_multiplier, cone_angle, width, height, sky=None, threads=None):
    """Voxelizer.DebugRender on the CPU. raw_chain: the grid's rgba16f levels back to back (uint16 or float16); sky:
    capi.sky_desc(...) result or None (black). Returns (image float32 [h, w, 4], cone samples)."""
    raw = np.ascontiguousarray(np.asarray(raw_chain).view(np.uint16).reshape(-1))
    fr = np.ascontiguousarray(frame)
    out = np.zeros((height, width, 4), np.float32)
    steps = ctypes.c_uint64()
    rc = lib().oracle_vx_debug_render(ctypes.addressof(ci), raw.ctypes.data, ctypes.addressof(sky) if sky is not None else None,
                                      fr.ctypes.data, float(step_multiplier), float(cone_angle), width, height, out.ctypes.data,
                                      ctypes.byref(steps), threads or ol.default_threads())
    assert rc == 0, rc
    return out, steps.value
