"""Scope table 8f.2: skinning + BLAS refit + TLAS re-upload (ModelManager.Update, ModelManager.cs:236-261)."""
import copy

import numpy as np
import pytest

import oracle_lib as ol
from idkengine_b200 import capi, scenes
from idkengine_b200 import gpu_types as gt
from raster_lib import skinning_setup


def test_oracle_refit_bounds_triangles(multi_blas):
    """BLAS.Refit restatement: after moving vertices every leaf box is the exact bound of its triangles, every interior
    box the union of its children, and rays through the refitted tree still agree with brute force."""
    scene = copy.deepcopy(multi_blas[0])
    u, jm, cmd = skinning_setup(scene, 2)
    before = scene.blas_nodes.copy()
    ol.skin_vertices(u, jm, scene.positions, scene.vertices, cmd[0])
    ol.blas_refit(scene, 2)
    d = scene.blas_descs[2]
    nodes = scene.blas_nodes[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]]
    assert not np.array_equal(nodes["Min"], before[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]]["Min"])
    other = np.ones(len(scene.blas_nodes), bool)
    other[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]] = False
    assert np.array_equal(scene.blas_nodes[other], before[other])          # other BLASes untouched
    assert np.array_equal(nodes["TriStartOrChild"], before[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]]["TriStartOrChild"])
    P = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1)
    for i in range(1, len(nodes)):
        nd = nodes[i]
        if nd["TriCount"] > 0:
            t = scene.blas_triangles[d["TriangleOffset"] + nd["TriStartOrChild"]:d["TriangleOffset"] + nd["TriStartOrChild"] + nd["TriCount"]]
            pts = P[np.concatenate([t["X"], t["Y"], t["Z"]])]
            assert np.array_equal(nd["Min"], pts.min(0)) and np.array_equal(nd["Max"], pts.max(0))
        else:
            l, r = nodes[nd["TriStartOrChild"]], nodes[nd["TriStartOrChild"] + 1]
            assert np.array_equal(nd["Min"], np.minimum(l["Min"], r["Min"])) and np.array_equal(nd["Max"], np.maximum(l["Max"], r["Max"]))
    rng = np.random.default_rng(8)
    rays = np.zeros(4000, gt.IdkPtRay)
    rays["Origin"] = rng.uniform(-2.5, 2.5, (4000, 3)).astype(np.float32)
    dd = rng.normal(size=(4000, 3))
    rays["Direction"] = (dd / np.linalg.norm(dd, axis=1, keepdims=True)).astype(np.float32)
    rays["TMax"] = np.float32(3.4028235e38)
    a, b = ol.trace_rays(scene, rays), ol.brute_force(scene, rays)
    assert np.array_equal(a["T"], b["T"])


def test_skinning_identity_round_trip(multi_blas):
    """Identity joint matrices leave positions bit-identical and normals within the 11/10-bit requantisation step."""
    scene = copy.deepcopy(multi_blas[0])
    u, jm, cmd = skinning_setup(scene, 1)
    jm[:] = 0
    jm[:, 0, 0] = jm[:, 1, 1] = jm[:, 2, 2] = 1
    pos0, vtx0 = scene.positions.copy(), scene.vertices.copy()
    ol.skin_vertices(u, jm, scene.positions, scene.vertices, cmd[0])
    v0, n = int(cmd["OutputVertexOffset"][0]), int(cmd["VertexCount"][0])
    for c in "xyz":
        assert np.allclose(scene.positions[c], pos0[c], rtol=0, atol=1e-6)
    r0, r1 = vtx0["Normal"][v0:v0 + n] & 2047, scene.vertices["Normal"][v0:v0 + n] & 2047
    assert np.abs(r0.astype(np.int64) - r1.astype(np.int64)).max() <= 2


@pytest.mark.gpu
def test_skin_refit_tlas_bit_exact():
    from idkengine_b200.pathtracer import PathTracer
    scene, cam = scenes.multi_blas(threads=1)
    scene.build_tlas()
    expect = copy.deepcopy(scene)
    u, jm, cmd = skinning_setup(scene, 2)
    ol.skin_vertices(u, jm, expect.positions, expect.vertices, cmd[0])
    ol.blas_refit(expect, 2)
    expect.build_tlas()
    w, h = 128, 96
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.Gpu.DoTraceLights = 1
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(frame)
        pt.Compute()
        still = pt.Result.copy()
        pt.SetSkinningData(u)
        ms_skin = pt.SkinVertices(jm, cmd)
        assert pt.AccumulatedSamples == 0
        ms_refit = pt.BlasRefit(2, 1)
        assert ms_skin > 0 and ms_refit > 0
        pos = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(scene.positions))
        vtx = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(scene.vertices))
        nodes = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, len(scene.blas_nodes))
        assert pos.tobytes() == expect.positions.tobytes()
        assert vtx.tobytes() == expect.vertices.tobytes()
        assert nodes.tobytes() == expect.blas_nodes.tobytes()
        # host TLAS build from the read-back boxes (the reference builds its TLAS on the CPU, BVH.cs:278-298), then re-upload
        scene.blas_nodes, scene.positions, scene.vertices = nodes, pos, vtx
        scene.build_tlas()
        assert scene.tlas_nodes.tobytes() == expect.tlas_nodes.tobytes()
        pt.UpdateRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, scene.tlas_nodes)
        assert pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(scene.tlas_nodes)).tobytes() == expect.tlas_nodes.tobytes()
        pt.Compute()
        pt.Compute()
        moved = pt.Result.copy()
        # refit of every BLAS is idempotent
        pt.BlasRefit(0, 3)
        assert pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, len(scene.blas_nodes)).tobytes()[32 * scene.blas_descs[2]["NodeOffset"]:] == \
            expect.blas_nodes.tobytes()[32 * scene.blas_descs[2]["NodeOffset"]:]
        with pytest.raises(RuntimeError):
            pt.BlasRefit(2, 5)
        bad = cmd.copy()
        bad["JointMatricesOffset"] = 7
        with pytest.raises(RuntimeError):
            pt.SkinVertices(jm, bad)
    res = np.zeros((h, w, 4), np.float32)
    o = ol.path_trace(expect, frame, s, w, h, sky=(0.6, 0.7, 0.9), result=res)
    o = ol.path_trace(expect, frame, s, w, h, sky=(0.6, 0.7, 0.9), accumulated=o.accumulated, result=res)
    assert np.array_equal(moved.view(np.uint32), res.view(np.uint32))
    assert not np.array_equal(moved, still)


@pytest.mark.gpu
@pytest.mark.parametrize("grid,radius", [(3, 15), (2, 2), (4, 7)])
def test_device_tlas_build_equals_host_build(grid, radius):
    """idkpt_tlas_build (BVH.TlasBuild + TLAS.Build PLOC on the device, no read-back) == the host mirror's TLAS.Build on the same
    roots and transforms, node for node, including after instances moved (transform update) -- then rendering through it."""
    from idkengine_b200.pathtracer import PathTracer
    scene, cam = scenes.instance_grid(grid, threads=1)
    scene.build_tlas(search_radius=radius)
    want = scene.tlas_nodes.copy()
    n = len(scene.blas_instances)
    w, h = 96, 64
    s = capi.default_settings()
    s.RayDepth = 4
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(frame)
        ms = pt.TlasBuild(radius)
        got = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * n - 1)
        assert ms > 0 and got.tobytes() == want.tobytes()
        # move a third of the instances, rebuild on both sides
        moved = scene.mesh_transforms.copy()
        for k in range(0, len(moved), 3):
            moved["ModelMatrix"][k][:, 3] += np.array([0.7, 0.15 * (k % 4), -0.5], np.float32)
            m = np.eye(4); m[:3, :] = moved["ModelMatrix"][k]
            moved["InvModelMatrix"][k] = np.linalg.inv(m)[:3, :].astype(np.float32)
        pt.UpdateRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, 0, moved)
        pt.TlasBuild(radius)
        scene.mesh_transforms = moved
        scene.build_tlas(search_radius=radius)
        got2 = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * n - 1)
        assert got2.tobytes() == scene.tlas_nodes.tobytes() and got2.tobytes() != want.tobytes()
        pt.Compute()
        img = pt.Result
    res = np.zeros((h, w, 4), np.float32)
    ol.path_trace(scene, frame, s, w, h, sky=(0.6, 0.7, 0.9), result=res)
    assert np.array_equal(img.view(np.uint32), res.view(np.uint32))
