"""ctypes wrapper of the G-buffer pass oracle (oracle/oracle_gbuffer.cpp -> oracle/liboracle_gbuffer.so), which
tests/test_gbuffer*.py use. The library is compiled on first use with the flags of oracle/build.py."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, "oracle")
SRC = os.path.join(ORACLE_DIR, "oracle_gbuffer.cpp")
LIB = os.path.join(ORACLE_DIR, "liboracle_gbuffer.so")

CHANNELS = (1, 2, 3, 2, 3, 2)   # depth, normal_rg, albedo, metallic_roughness, emissive, velocity_rg
STORE_R11G11 = 0                # oracle_gbuffer_store kinds
STORE_B10 = 1
STORE_RG8 = 2
STORE_RG16F = 3

_lib = None


def build(force=False):
    deps = [SRC] + [os.path.join(ORACLE_DIR, f) for f in ("oracle.cpp", "oracle_vxgi.inc", "oracle_post.inc")] + \
        [os.path.join(REPO, "include", f) for f in ("idkpt.h", "idkvx.h", "idk_gpu_types.h")]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    tmp = LIB + ".%d.tmp" % os.getpid()
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                    "-fvisibility=hidden", "-o", tmp, SRC], check=True)
    os.replace(tmp, LIB)
    return LIB


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        vp, i32, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint64
        L.oracle_gbuffer.restype = i32
        L.oracle_gbuffer.argtypes = [ctypes.POINTER(capi.IdkPtSceneDesc), vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32]
        L.oracle_gbuffer_store.restype = None
        L.oracle_gbuffer_store.argtypes = [i32, vp, u64, vp]
        _lib = L
    return _lib


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
