"""ctypes wrapper of the variable-rate light-sphere and skybox oracle (oracle/oracle_lights_skybox_vrs.cpp), which
tests/test_lights_skybox_vrs*.py use. The oracle is the root of its own library, liboracle_lights_skybox_vrs.so, built here
with oracle/build.py's compiler flags; the export's signature is declared here, beside the wrapper."""
import ctypes
import glob
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi

ORACLE_DIR = os.path.join(ol.REPO, "oracle")
SOURCE = os.path.join(ORACLE_DIR, "oracle_lights_skybox_vrs.cpp")

# name -> (restype, argtypes) of the exports this module declares
SIGNATURES = {
    "oracle_lights_skybox_vrs": (ctypes.c_int32, [ctypes.POINTER(capi.IdkPtSceneDesc), ctypes.POINTER(capi.IdkPtSkyDesc)] +
                                 [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32] + [ctypes.c_void_p] * 8 + [ctypes.c_int32]),
}

_fn = None


def build():
    """The library beside liboracle.so (or, where the tree is read-only, in the temporary directory), rebuilt when an oracle
    source or public header is newer than it."""
    out_dir = ORACLE_DIR if os.access(ORACLE_DIR, os.W_OK) else tempfile.gettempdir()
    target = os.path.join(out_dir, "liboracle_lights_skybox_vrs.so")
    deps = [f for pattern in ("*.cpp", "*.inc") for f in glob.glob(os.path.join(ORACLE_DIR, pattern))] + \
        glob.glob(os.path.join(ol.REPO, "include", "*.h"))
    if os.path.exists(target) and all(os.path.getmtime(d) <= os.path.getmtime(target) for d in deps):
        return target
    tmp = "%s.%d.tmp" % (target, os.getpid())
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                    "-fvisibility=hidden", "-I", ORACLE_DIR, "-o", tmp, SOURCE], check=True)
    os.replace(tmp, target)    # a process that loads the library meanwhile sees the old file or the new one, never half of one
    return target


def _oracle():
    global _fn
    if _fn is None:
        fn = ctypes.CDLL(build()).oracle_lights_skybox_vrs
        fn.restype, fn.argtypes = SIGNATURES["oracle_lights_skybox_vrs"]
        _fn = fn
    return _fn


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
    rc = _oracle()(ctypes.byref(d), ctypes.byref(sd) if sd is not None else None, fr.ctypes.data, w, h,
                   jit.ctypes.data if jit is not None else None, g[0].ctypes.data, g[1].ctypes.data, g[4].ctypes.data,
                   g[5].ctypes.data, col.ctypes.data, winner.ctypes.data, r.ctypes.data, threads or ol.default_threads())
    assert rc == 0, rc
    del keep
    return tuple(g), col, winner


def fragment_of(rates, w, h):
    """Per pixel (x0, y0, cw, ch) of its coarse fragment: int [h, w, 4]."""
    cwh = np.array([[1, 1], [2, 1], [2, 2], [4, 2], [4, 4]])[np.repeat(np.repeat(np.asarray(rates), 16, 0), 16, 1)[:h, :w]]
    x, y = np.meshgrid(np.arange(w), np.arange(h))
    return np.stack([x - x % cwh[..., 0], y - y % cwh[..., 1], cwh[..., 0], cwh[..., 1]], -1)
