"""ctypes wrapper of the C#-semantics collision oracle (oracle/oracle_collision.cpp), the checker of idkpt_collide_spheres and
idkpt_collide_spheres_tlas, and the collision tests' inputs: moving spheres and the scenes that pin the TLAS walk's visit
order."""
import ctypes

import numpy as np

import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt, host, scenes


def collide_spheres(scene, spheres, settings, threads=None, use_tlas=False):
    """C#-semantics SceneVsMovingSphereCollisionRoutine per sphere over the walk BVH.CpuUseTlas picks. use_tlas=False: every
    instance in index order (idkpt_collide_spheres); True: TLAS.Intersect(Box) over scene.tlas_nodes
    (idkpt_collide_spheres_tlas). settings: (TestSteps, RecursiveSteps, EpsilonNormalOffset, Response). Returns
    (IdkPtSphereCollision records, first winner [n, 2] = (global BLAS triangle, instance index) or -1, its distance or
    FLT_MAX)."""
    if use_tlas:
        assert scene.use_tlas and len(scene.tlas_nodes) == 2 * len(scene.blas_instances) - 1
    d, keep = capi.scene_desc(scene)
    spheres = np.ascontiguousarray(spheres, gt.IdkPtMovingSphere)
    st = np.array(tuple(settings), gt.IdkPtCollisionSettings)
    out = np.zeros(len(spheres), gt.IdkPtSphereCollision)
    first = np.zeros((len(spheres), 2), np.int32)
    dist = np.zeros(len(spheres), np.float32)
    ol.lib().oracle_collide_spheres(ctypes.byref(d), spheres.ctypes.data, len(spheres), st.ctypes.data, out.ctypes.data,
                                    first.ctypes.data, dist.ctypes.data, threads or ol.default_threads(), int(use_tlas))
    del keep
    return out, first, dist


def spheres(prev, dest, radius, vel=None):
    s = np.zeros(len(prev), gt.IdkPtMovingSphere)
    s["PrevPosition"], s["Position"], s["Radius"] = prev, dest, radius
    s["Velocity"] = 0.0 if vel is None else vel
    return s


def random_spheres(scene, n, seed, step=0.5, radius=(0.02, 0.5)):
    """Spheres over the scene's bounds: a random start, a destination up to `step` away, radii in `radius`."""
    p = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1)
    lo, hi = p.min(0), p.max(0)
    if scene.mesh_transforms is not None and len(scene.blas_instances) > 1:   # instanced scenes: the instances' world bounds
        t = scene.mesh_transforms["ModelMatrix"][:, :, 3]
        lo, hi = np.minimum(lo, t.min(0) - 1.0), np.maximum(hi, t.max(0) + 1.0)
    rng = np.random.default_rng(seed)
    prev = rng.uniform(lo, hi, (n, 3))
    dest = prev + rng.uniform(-step, step, (n, 3))
    vel = rng.uniform(-3.0, 3.0, (n, 3))
    return spheres(prev.astype(np.float32), dest.astype(np.float32), rng.uniform(*radius, n).astype(np.float32), vel.astype(np.float32))


def with_tlas(sc):
    sc.build_tlas()
    return sc


def dfs_leaf_order(tlas):
    """Instance ids in the order a left-first depth-first walk of every TLAS node reaches its leaves."""
    order, stack = [], [0]
    while stack:
        w = int(tlas["IsLeafAndChildOrInstanceId"][stack.pop()])
        if w >> 31:
            order.append(w & 0x7FFFFFFF)
        else:
            stack += [w + 1, w]
    return order


def stacked_quads(heights):
    """One horizontal 4 x 4 quad per height, each its own model and instance (instance i at heights[i]), and the scene's TLAS."""
    meshes, mats = scenes._materials([dict(color=(0.6, 0.6, 0.6))])
    models = []
    for y in heights:
        a = scenes._Assembler()
        a.add(scenes.quad([-2, y, -2], [-2, y, 2], [2, y, 2], [2, y, -2]), 0)
        models.append(a.model(meshes, mats, name=f"quad{y}"))
    return host.Scene().add(*models, threads=1).build_tlas()


def visit_order_case():
    """Stacked quads and, between each pair of neighbouring quads whose depth-first TLAS leaf order is not their index order, a
    resting sphere exactly half-way: the two quads tie. Returns (scene, spheres, [(depth-first first, lower index)] per sphere)."""
    heights = [float(h) for h in (5, 2, 7, 0, 3, 6, 1, 4)]
    sc = stacked_quads(heights)
    rank = {inst: k for k, inst in enumerate(dfs_leaf_order(sc.tlas_nodes))}
    assert sorted(rank) == list(range(len(heights)))
    by_height = sorted(range(len(heights)), key=lambda i: heights[i])
    centres, want = [], []
    for lo, hi in zip(by_height, by_height[1:]):
        if (rank[lo] < rank[hi]) != (lo < hi):
            centres.append([0.7, (heights[lo] + heights[hi]) / 2, -0.3])
            want.append((lo if rank[lo] < rank[hi] else hi, min(lo, hi)))
    c = np.array(centres, np.float32)
    return sc, spheres(c, c, 0.75), want
