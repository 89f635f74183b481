"""ctypes wrapper of the sky oracle (oracle/oracle_sky.cpp in oracle/liboracle.so), which tests/test_sky*.py use."""
import ctypes

import numpy as np

import oracle_lib as ol
from oracle_lib import lib


def atmosphere(settings, n, threads=None):
    """idkpt_sky_atmosphere on the CPU: faces float32 [6, n, n, 4]."""
    faces = np.zeros((6, n, n, 4), np.float32)
    assert lib().oracle_sky_atmosphere(ctypes.byref(settings), n, faces.ctypes.data, threads or ol.default_threads()) == 0
    return faces


def equirect(rgb, threads=None):
    """idkpt_sky_equirectangular on the CPU: rgb float32 [h, w, 3] -> faces float32 [6, w // 4, w // 4, 4]."""
    img = np.ascontiguousarray(rgb, np.float32)
    h, w = img.shape[:2]
    faces = np.zeros((6, w // 4, w // 4, 4), np.float32)
    assert lib().oracle_sky_equirect(img.ctypes.data, w, h, faces.ctypes.data, threads or ol.default_threads()) == 0
    return faces


def directions(n):
    """The fp32 texel directions of both kernels, float32 [6, n, n, 3]."""
    d = np.zeros((6, n, n, 3), np.float32)
    lib().oracle_sky_directions(n, d.ctypes.data)
    return d


def det_atan2(y, x):
    y, x = np.ascontiguousarray(y, np.float32), np.ascontiguousarray(x, np.float32)
    out = np.zeros(y.shape, np.float32)
    lib().oracle_det_atan2(y.ctypes.data, x.ctypes.data, y.size, out.ctypes.data)
    return out


def det_asin(x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(x.shape, np.float32)
    lib().oracle_det_asin(x.ctypes.data, x.size, out.ctypes.data)
    return out
