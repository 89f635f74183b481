"""ctypes wrapper of the C#-semantics TLAS collision oracle (tests/cpp/collision_tlas_oracle.cpp), the checker of
idkpt_collide_spheres_tlas. The library is compiled once per process, with the oracle's flags, into a temporary directory that
is removed at exit."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt

SOURCE = os.path.join(ol.REPO, "tests", "cpp", "collision_tlas_oracle.cpp")

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="collision_tlas_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libcollision_tlas_oracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                        "-fvisibility=hidden", "-o", so, SOURCE], check=True)
        L = ctypes.CDLL(so)
        vp = ctypes.c_void_p
        L.oracle_collide_spheres_walk.restype = ctypes.c_int32
        L.oracle_collide_spheres_walk.argtypes = [ctypes.POINTER(capi.IdkPtSceneDesc), vp, ctypes.c_uint64, vp, vp, vp, vp,
                                                  ctypes.c_int32, ctypes.c_int32]
        _lib = L
    return _lib


def collide_spheres(scene, spheres, settings, threads=None, use_tlas=True):
    """C#-semantics SceneVsMovingSphereCollisionRoutine per sphere over the walk BVH.CpuUseTlas picks. use_tlas=True:
    TLAS.Intersect(Box) over scene.tlas_nodes (idkpt_collide_spheres_tlas); False: every instance in index order, the same
    restated routine as collision_oracle.collide_spheres. Returns (IdkPtSphereCollision records, first winner [n, 2] =
    (global BLAS triangle, instance index) or -1, its distance or FLT_MAX)."""
    if use_tlas:
        assert scene.use_tlas and len(scene.tlas_nodes) == 2 * len(scene.blas_instances) - 1
    d, keep = capi.scene_desc(scene)
    spheres = np.ascontiguousarray(spheres, gt.IdkPtMovingSphere)
    st = np.array(tuple(settings), gt.IdkPtCollisionSettings)
    out = np.zeros(len(spheres), gt.IdkPtSphereCollision)
    first = np.zeros((len(spheres), 2), np.int32)
    dist = np.zeros(len(spheres), np.float32)
    lib().oracle_collide_spheres_walk(ctypes.byref(d), spheres.ctypes.data, len(spheres), st.ctypes.data, out.ctypes.data,
                                      first.ctypes.data, dist.ctypes.data, threads or ol.default_threads(), int(use_tlas))
    return out, first, dist
