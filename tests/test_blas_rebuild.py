"""host.Scene.rebuild_blases (BVH.BlasesBuild(first, count) over the Scene's arrays) and host.blas_global_sah
(BLAS.ComputeGlobalSAH): the host mirror that the device rebuild (idkpt_blas_rebuild, idkpt_blas_sah) is compared against."""
import copy

import numpy as np
import pytest

import oracle_lib as ol
from idkengine_b200 import host, scenes


def room_crate_ball():
    """multi_blas's models reordered so that the refittable crate sits between the pre-split room and ball."""
    room, ball, crate = scenes.multi_blas_models()
    scene = host.Scene().add(room, crate, ball, threads=1)
    scene.add_light((-1.0, 2.5, 1.0), (30.0, 28.0, 20.0), 0.3)
    return scene


def hall_crate_ball():
    """A pre-split BLAS first: two of the room's walls with a small sphere inside, so that the large quads split. Each rebuild
    pre-splits its already duplicated triangles again, so its triangle count grows and every later offset moves."""
    room, ball, crate = scenes.multi_blas_models()
    a = scenes._Assembler()
    a.add(scenes.quad([-3, 0, -3], [-3, 0, 3], [3, 0, 3], [3, 0, -3]), 0)
    a.add(scenes.quad([-3, 0, -3], [3, 0, -3], [3, 4, -3], [-3, 4, -3]), 0)
    a.add(scenes.uv_sphere([0, 1, 0], 0.5, 12, 16), 0)
    hall = a.model(room.meshes[:1], room.materials[:1], name="hall")
    scene = host.Scene().add(hall, crate, ball, threads=1)
    scene.add_light((-1.0, 2.5, 1.0), (30.0, 28.0, 20.0), 0.3)
    return scene


def blas_vertex_range(scene, b):
    d = scene.blas_descs[b]
    t = scene.blas_triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]]
    idx = np.concatenate([t["X"], t["Y"], t["Z"]])
    return int(idx.min()), int(idx.max()) + 1


def deform(scene, b, amount=0.3):
    """Moves the vertices of BLAS b: a twist about y, growing with the height, in float32."""
    v0, v1 = blas_vertex_range(scene, b)
    p = scene.positions[v0:v1]
    x, y, z = p["x"].astype(np.float64), p["y"].astype(np.float64), p["z"].astype(np.float64)
    a = amount * (y - y.min())
    p["x"] = (np.cos(a) * x - np.sin(a) * z).astype(np.float32)
    p["z"] = (np.sin(a) * x + np.cos(a) * z).astype(np.float32)
    scene.positions[v0:v1] = p


def check_rebuilt(before, after, first, count):
    """`after` is `before` with BLASes [first, first + count) rebuilt from after.positions."""
    nd = len(before.blas_descs)
    for b in range(nd):
        o, n = before.blas_descs[b], after.blas_descs[b]
        new_nodes = after.blas_nodes[n["NodeOffset"]:n["NodeOffset"] + n["NodeCount"]]
        new_tris = after.blas_triangles[n["TriangleOffset"]:n["TriangleOffset"] + n["TriangleCount"]]
        if first <= b < first + count:
            src = before.blas_triangles[o["TriangleOffset"]:o["TriangleOffset"] + o["TriangleCount"]]
            want = host.build_blas(after.positions, src, presplit=not o["IsRefittable"], threads=1)
            assert new_nodes.tobytes() == want["nodes"].tobytes()
            assert new_tris.tobytes() == want["triangles"].tobytes()
            assert n["RequiredStackSize"] == want["required_stack_size"]
            for f in ("IsRefittable", "LeafIndicesOffset", "LeafIndicesCount", "ParentIndicesOffset", "ParentIndicesCount"):
                assert n[f] == o[f]
        else:
            assert new_nodes.tobytes() == before.blas_nodes[o["NodeOffset"]:o["NodeOffset"] + o["NodeCount"]].tobytes()
            assert new_tris.tobytes() == before.blas_triangles[o["TriangleOffset"]:o["TriangleOffset"] + o["TriangleCount"]].tobytes()
            assert n.tobytes() == o.tobytes() if b < first else (n["NodeCount"], n["TriangleCount"]) == (o["NodeCount"], o["TriangleCount"])
        assert n["NodeOffset"] == (0 if b == 0 else after.blas_descs[b - 1]["NodeOffset"] + after.blas_descs[b - 1]["NodeCount"])
        assert n["TriangleOffset"] == (0 if b == 0 else after.blas_descs[b - 1]["TriangleOffset"] + after.blas_descs[b - 1]["TriangleCount"])
    last = after.blas_descs[-1]
    assert last["NodeOffset"] + last["NodeCount"] == len(after.blas_nodes)
    assert last["TriangleOffset"] + last["TriangleCount"] == len(after.blas_triangles)
    assert after.blas_stack_size == max(1, int(after.blas_descs["RequiredStackSize"].max()))


def random_rays(n=4000, seed=8, half=3.5):
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    return ol.make_rays(rng.uniform(-half, half, (n, 3)).astype(np.float32) + np.float32([0, 1.5, 0]),
                        (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32))


def test_refittable_blas_in_the_middle():
    before = room_crate_ball()
    assert list(before.blas_descs["IsRefittable"]) == [0, 1, 0]
    deform(before, 1)
    after = copy.deepcopy(before)
    after.rebuild_blases(1, 1, threads=2)
    check_rebuilt(before, after, 1, 1)
    assert after.blas_nodes[before.blas_descs[1]["NodeOffset"]:].tobytes() != before.blas_nodes[before.blas_descs[1]["NodeOffset"]:].tobytes()
    assert len(after.blas_triangles) == len(before.blas_triangles)     # no pre-splitting: the same triangles, reordered


def test_pre_split_blas_first_changes_the_triangle_count():
    before = hall_crate_ball()
    deform(before, 0, amount=0.2)
    after = copy.deepcopy(before)
    after.rebuild_blases(0, 1, threads=2)
    check_rebuilt(before, after, 0, 1)
    # pre-split again from the already duplicated list: more triangles, and every later offset moved
    assert after.blas_descs[0]["TriangleCount"] > before.blas_descs[0]["TriangleCount"]
    assert after.blas_descs[1]["TriangleOffset"] != before.blas_descs[1]["TriangleOffset"]


def test_every_blas_at_once_and_zero_count():
    before = room_crate_ball()
    deform(before, 1)
    deform(before, 2, amount=0.1)
    after = copy.deepcopy(before)
    after.rebuild_blases(0, 3, threads=2)
    check_rebuilt(before, after, 0, 3)
    same = copy.deepcopy(after)
    same.rebuild_blases(2, 0)
    for f in ("blas_nodes", "blas_triangles", "blas_descs"):
        assert getattr(same, f).tobytes() == getattr(after, f).tobytes()


@pytest.mark.parametrize("first,count", [(0, 1), (1, 1), (0, 3)])
def test_traced_rays_equal_brute_force_after_a_rebuild(first, count):
    scene = room_crate_ball()
    for b in range(first, first + count):     # a BLAS whose vertices moved must be rebuilt (or refitted) before tracing
        deform(scene, b, amount=0.05 if b != 1 else 0.3)
    scene.rebuild_blases(first, count, threads=2)
    rays = random_rays()
    a, b = ol.trace_rays(scene, rays), ol.brute_force(scene, rays)
    assert np.array_equal(a["T"], b["T"])
    assert (a["T"] < 1e30).sum() > 1000


@pytest.mark.parametrize("make", [lambda: scenes.multi_blas(threads=1)[0], lambda: scenes.cornell_1k(threads=1)[0],
                                  lambda: scenes.instance_grid(threads=1)[0], lambda: scenes.closed_box(subdiv=3, threads=1)[0],
                                  room_crate_ball], ids=["multi_blas", "cornell_1k", "instance_grid", "closed_box", "room_crate_ball"])
def test_global_sah_equals_the_builds_sah(make):
    scene = make()
    assert len(scene.build_info) == len(scene.blas_descs)
    for d, info in zip(scene.blas_descs, scene.build_info):
        nodes = scene.blas_nodes[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]]
        assert np.float64(host.blas_global_sah(nodes)).tobytes() == np.float64(info["sah"]).tobytes()


def test_global_sah_follows_the_triangle_cost_and_refit():
    scene = room_crate_ball()
    d = scene.blas_descs[1]
    nodes = scene.blas_nodes[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]]
    s = host.default_build_settings()
    s.TriangleCost = 2.5
    built = host.build_blas(scene.positions, scene.blas_triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]],
                            presplit=False, threads=1, settings=s)
    assert host.blas_global_sah(built["nodes"], 2.5) == built["sah"]
    assert host.blas_global_sah(nodes, 2.5) > host.blas_global_sah(nodes)
    sah_built = host.blas_global_sah(nodes)
    deform(scene, 1, amount=0.8)
    ol.blas_refit(scene, 1)
    refitted = scene.blas_nodes[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]]
    sah_refit = host.blas_global_sah(refitted)
    scene.rebuild_blases(1, 1, threads=1)
    d = scene.blas_descs[1]
    rebuilt = host.blas_global_sah(scene.blas_nodes[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]])
    assert sah_refit > rebuilt and sah_refit != sah_built
    assert scene.build_info[1]["sah"] == rebuilt
