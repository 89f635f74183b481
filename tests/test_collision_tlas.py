"""oracle_collide_spheres_tlas, the checker of idkpt_collide_spheres_tlas: SceneVsMovingSphereCollisionRoutine over the walk
BVH.Intersect(in Box) takes with CpuUseTlas == true (TLAS.Intersect(Box)), against the linear walk of oracle_collide_spheres.
The TLAS oracle restates the routine with the walk as a parameter; with the linear walk it must equal oracle_collide_spheres.
The two walks test the same triangles with the same arithmetic; they differ only in which instances they reach and in what
order, so the winner of a test step can differ only between candidates at the same distance."""
import numpy as np
import pytest

import collision_oracle as co
import collision_tlas_oracle as cto
from idkengine_b200 import host, scenes
from idkengine_b200.pathtracer import CAMERA_COLLISION, LIGHT_COLLISION
from test_collision_gpu import random_spheres, spheres

PRESETS = pytest.mark.parametrize("settings", [LIGHT_COLLISION, CAMERA_COLLISION], ids=["lights", "camera"])


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


CROSS = {
    "closed_box": lambda: scenes.closed_box(subdiv=4, threads=1)[0],
    "instance_grid": lambda: scenes.instance_grid(3, threads=1)[0],
    "atrium": lambda: scenes.atrium(target_tris=20000, threads=1)[0],
}


@PRESETS
@pytest.mark.parametrize("name", list(CROSS))
def test_restated_routine_with_the_linear_walk_equals_the_linear_oracle(name, settings):
    """The TLAS oracle's routine, run with the linear walk, is byte-equal to oracle_collide_spheres: only the walk differs."""
    sc = CROSS[name]()
    s = random_spheres(sc, 2048, seed=23 + len(name))
    lin = co.collide_spheres(sc, s, settings)
    again = cto.collide_spheres(sc, s, settings, use_tlas=False)
    for a, b in zip(lin, again):
        assert a.tobytes() == b.tobytes()
    assert (lin[0]["Hits"] > 0).sum() >= 16


SINGLE = {
    "closed_box": lambda: with_tlas(scenes.closed_box(subdiv=4, threads=1)[0]),
    "open_floor": lambda: with_tlas(scenes.open_floor(threads=1)[0]),
    "atrium": lambda: with_tlas(scenes.atrium(target_tris=20000, threads=1)[0]),
}


@PRESETS
@pytest.mark.parametrize("name", list(SINGLE))
def test_single_instance_tlas_equals_the_linear_walk(name, settings):
    """With one instance the TLAS root is that instance's leaf: both walks visit the same BLAS, so every byte agrees."""
    sc = SINGLE[name]()
    assert len(sc.tlas_nodes) == 1 and sc.tlas_nodes["IsLeafAndChildOrInstanceId"][0] == 0x80000000
    s = random_spheres(sc, 2048, seed=len(name))
    lin = co.collide_spheres(sc, s, settings)
    tl = cto.collide_spheres(sc, s, settings)
    for a, b in zip(lin, tl):
        assert a.tobytes() == b.tobytes()
    assert (lin[0]["Hits"] > 0).sum() >= 16


INSTANCED = {
    "instance_grid": lambda: scenes.instance_grid(3, threads=1)[0],
    "grid_4096": lambda: with_tlas(scenes._instanced(scenes._grid_matrices(4096))),
}


@PRESETS
@pytest.mark.parametrize("name", list(INSTANCED))
def test_instanced_first_winner_agrees_up_to_ties(name, settings):
    """The first recursive step's winner is the linear walk's, or a different candidate at exactly the same distance."""
    sc = INSTANCED[name]()
    s = random_spheres(sc, 4096, seed=17 + len(name))
    _, lf, ld = co.collide_spheres(sc, s, settings)
    out, tf, td = cto.collide_spheres(sc, s, settings)
    same = (lf == tf).all(1)
    assert (ld[~same].view(np.uint32) == td[~same].view(np.uint32)).all(), np.flatnonzero(~same)[:8]
    assert ((lf[:, 0] >= 0) == (tf[:, 0] >= 0)).all()
    assert (out["Hits"] > 0).sum() >= 16


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


@PRESETS
def test_ties_go_to_the_depth_first_instance(settings):
    sc, s, want = visit_order_case()
    assert len(want) >= 2, want
    _, lf, ld = co.collide_spheres(sc, s, settings)
    _, tf, td = cto.collide_spheres(sc, s, settings)
    assert (ld == 0.5).all() and (td == 0.5).all()
    assert tf[:, 1].tolist() == [w[0] for w in want]      # the TLAS walk: the leaf it reaches first
    assert lf[:, 1].tolist() == [w[1] for w in want]      # the linear walk: the lower instance index
    assert (tf[:, 1] != lf[:, 1]).all()
