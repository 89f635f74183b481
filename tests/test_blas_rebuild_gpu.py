"""idkpt_blas_rebuild (PathTracer.RebuildBlases: BVH.BlasesBuild(first, count) on the device scene in place) and idkpt_blas_sah
(PathTracer.BlasSah: BLAS.ComputeGlobalSAH of the device trees). Each case compares against host.Scene.rebuild_blases applied
to a copy of the scene with the positions read back from the device. Every comparison is exact."""
import copy

import numpy as np
import pytest

import gbuffer_oracle as go
import oracle_lib as ol
import transparency_oracle as to
from idkengine_b200 import capi, host, scenes, vxgi
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, assert_bits, skinning_setup
from test_blas_rebuild import hall_crate_ball, random_rays, room_crate_ball

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_NO_SCENE = -1, -4
W, H = 96, 64
SKY = (0.6, 0.7, 0.9)
CAM = dict(position=(0.0, 1.6, 5.0), view_dir=(0.0, -0.1, -1.0), fov_y_deg=60.0)


def settings():
    s = capi.default_settings()
    s.Gpu.DoTraceLights = 1
    return s


def read_scene(pt, scene):
    """The device's BLAS arrays, positions and vertices as a Scene (the host's CPU copy refreshed through idkpt_read_range)."""
    out = copy.deepcopy(scene)
    descs = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_DESCS, 0, len(scene.blas_descs))
    last = descs[-1]
    out.blas_descs = descs
    out.blas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, int(last["NodeOffset"] + last["NodeCount"]))
    out.blas_triangles = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_TRIANGLES, 0, int(last["TriangleOffset"] + last["TriangleCount"]))
    out.positions = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(scene.positions))
    out.vertices = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(scene.vertices))
    out.blas_stack_size = max(1, int(descs["RequiredStackSize"].max()))
    if scene.use_tlas:
        out.tlas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(scene.tlas_nodes))
    return out


def mirror(pt, scene, first, count):
    """host.Scene.rebuild_blases of `scene` over the device's current positions, then the host TLAS build."""
    m = copy.deepcopy(scene)
    m.positions = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(scene.positions))
    m.vertices = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(scene.vertices))
    m.rebuild_blases(first, count, threads=ol.default_threads())
    if scene.use_tlas:
        m.build_tlas()
    return m


def assert_scene(pt, want):
    got = read_scene(pt, want)
    for f in ("blas_descs", "blas_nodes", "blas_triangles", "tlas_nodes"):
        assert getattr(got, f).tobytes() == getattr(want, f).tobytes(), f
    return got


def assert_hits(got, want):
    for k in ("T", "BaryX", "BaryY", "TriangleId", "MeshTransformId", "NodePairFetches", "TriangleTests"):
        assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(want[k]).tobytes(), k


def assert_traces(pt, want, rays=None):
    rays = random_rays() if rays is None else rays
    for trace, oracle in ((pt.TraceRays, ol.trace_rays), (pt.TraceRaysAny, ol.trace_rays_any)):
        got, _ = trace(rays, trace_lights=True)
        assert_hits(got, oracle(want, rays, trace_lights=True))
        assert (got["T"] < 1e30).sum() > len(rays) // 10


def assert_image(pt, want, frame, s):
    pt.ResetAccumulation()
    pt.Compute()
    pt.Compute()
    res = np.zeros((H, W, 4), np.float32)
    o = ol.path_trace(want, frame, s, W, H, sky=SKY, result=res)
    ol.path_trace(want, frame, s, W, H, sky=SKY, accumulated=o.accumulated, result=res)
    assert np.array_equal(pt.Result.view(np.uint32), res.view(np.uint32))


def opened(scene, s=None):
    pt = PathTracer(W, H, s or settings())
    pt.SetScene(scene)
    pt.SetSky(SKY)
    frame = scenes.camera_frame(CAM, W, H)
    pt.SetFrame(frame)
    return pt, frame


@pytest.mark.parametrize("make,blas", [(room_crate_ball, 1), (hall_crate_ball, 0)], ids=["refittable_middle", "pre_split_first"])
def test_skinned_blas_rebuilt(make, blas):
    scene = make()
    scene.build_tlas()
    u, jm, cmd = skinning_setup(scene, blas)
    s = settings()
    pt, frame = opened(scene, s)
    with pt:
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        ms = pt.RebuildBlases(blas, 1)
        assert ms > 0 and pt.AccumulatedSamples == 0
        pt.TlasBuild()
        want = mirror(pt, scene, blas, 1)
        got = assert_scene(pt, want)
        if blas == 0:     # pre-split again: more triangles, and every later offset moved
            assert want.blas_descs[0]["TriangleCount"] > scene.blas_descs[0]["TriangleCount"]
            assert got.blas_descs[1]["TriangleOffset"] != scene.blas_descs[1]["TriangleOffset"]
        assert_traces(pt, want)
        assert_image(pt, want, frame, s)


def test_every_blas_then_refit():
    scene = room_crate_ball()
    scene.build_tlas()
    u, jm, cmd = skinning_setup(scene, 1)
    jm2 = skinning_setup(scene, 1, seed=9)[1]
    s = settings()
    pt, frame = opened(scene, s)
    with pt:
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.RebuildBlases(0, len(scene.blas_descs))      # Application.cs:163
        pt.TlasBuild()
        want = mirror(pt, scene, 0, len(scene.blas_descs))
        assert_scene(pt, want)
        assert_image(pt, want, frame, s)
        pt.SkinVertices(jm2, cmd)                        # a refit of the rebuilt tree
        pt.BlasRefit(1, 1)
        pt.TlasBuild()
        want.positions = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(scene.positions))
        want.vertices = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(scene.vertices))
        ol.blas_refit(want, 1)
        want.build_tlas()
        assert_scene(pt, want)
        assert_traces(pt, want)


def test_raster_frame_after_a_rebuild():
    scene = room_crate_ball()
    scene.materials["AlphaCutoff"][::3] = 2.0          # blended surfaces for the transparency pass
    scene.materials["BaseColorFactor"][::3] = (scene.materials["BaseColorFactor"][::3] & 0x00FFFFFF) | (0x80 << 24)
    u, jm, cmd = skinning_setup(scene, 1)
    frame = scenes.camera_frame(CAM, W, H)
    with PathTracer(W, H) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        kept = pt.PrevPositionsDevicePtr()
        pt.RebuildBlases(1, 1)
        want = mirror(pt, scene, 1, 1)
        assert_scene(pt, want)
        assert pt.PrevPositionsDevicePtr() == kept
        got = pt.GBuffer(frame, W, H, jitter=JITTER, prev_positions="kept")
        color = np.random.default_rng(4).uniform(0, 1, (H, W, 4)).astype(np.float32)
        arr = color.copy()
        pt.Transparency(frame, got[0], settings=capi.IdkPtTransparencySettings(0, 0), jitter=JITTER, color=arr)
    # the kept previous positions are still the ones the skin overwrote, i.e. the positions the scene was set with
    for a, b in zip(got, go.gbuffer(want, frame, W, H, jitter=JITTER, prev_positions=np.stack([scene.positions[c] for c in "xyz"], 1))):
        assert_bits(a, b)
    ref = to.transparency(want, frame, got[0], color, jitter=JITTER, sky=None)[0]
    assert np.array_equal(arr.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("conservative", [False, True])
def test_bound_voxeliser_after_a_pre_split_rebuild(conservative):
    scene = hall_crate_ball()
    u, jm, cmd = skinning_setup(scene, 0)
    lo, hi = (-3.2, -1.2, -3.2), (3.2, 4.2, 3.2)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(64, lo, hi) as bound, vxgi.Voxelizer(64, lo, hi) as owned:
        pt.SetScene(scene)
        bound.SetSceneFrom(pt)
        bound.IsConservativeRasterization = owned.IsConservativeRasterization = conservative
        bound.Render()
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.RebuildBlases(0, 1)
        want = mirror(pt, scene, 0, 1)
        assert len(want.blas_triangles) > len(scene.blas_triangles)
        owned.SetScene(want)
        sb, so = bound.Render(), owned.Render()
        assert sb.Fragments == so.Fragments > 0
        for l in range(len(bound.sizes)):
            assert np.array_equal(bound.ReadLevel(l).view(np.uint16), owned.ReadLevel(l).view(np.uint16))


def coincident_model(n):
    """n copies of one triangle, refittable: the tree built over them is a chain that needs no traversal stack. Skinning
    spreads the copies apart, and the rebuilt tree then needs one."""
    p = np.array([[0, 1, 0], [0.5, 1, 0], [0, 1.5, 0]] * n, np.float32)
    return host.Model(p, np.arange(3 * n, dtype=np.uint32).reshape(-1, 3), refittable=True, name="coincident")


def test_rebuild_raises_the_stack_size():
    room, ball, crate = scenes.multi_blas_models()
    scene = host.Scene().add(room, coincident_model(512), threads=1)
    scene.build_tlas()
    u, jm, cmd = skinning_setup(scene, 1)
    s = settings()
    pt, frame = opened(scene, s)
    with pt:
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.RebuildBlases(1, 1)
        pt.TlasBuild()
        want = mirror(pt, scene, 1, 1)
        assert want.blas_stack_size > scene.blas_stack_size
        assert_scene(pt, want)
        assert_traces(pt, want)
        assert_image(pt, want, frame, s)


def test_rejections_leave_everything():
    scene = room_crate_ball()
    scene.build_tlas()
    pt, frame = opened(scene)
    with pt:
        with pytest.raises(IdkPtError, match=f"failed \\({ERR_NO_SCENE}\\)"):
            with PathTracer(16, 16) as empty:
                empty.RebuildBlases(0, 1)
        pt.Compute()
        image = pt.Result.copy()
        before = read_scene(pt, scene)
        bad_nan = host.default_build_settings()
        bad_nan.SplitFactor = float("nan")
        bad_stop = host.default_build_settings()
        bad_stop.StopSplittingThreshold = 0
        for args in [(2, 2, None), (4, 0, None), (0, 1, bad_nan), (0, 1, bad_stop)]:
            with pytest.raises(IdkPtError, match=f"failed \\({ERR_INVALID_ARGUMENT}\\)"):
                pt.RebuildBlases(*args)
        pt.RebuildBlases(1, 0)
        after = read_scene(pt, scene)
        for f in ("blas_descs", "blas_nodes", "blas_triangles", "tlas_nodes"):
            assert getattr(after, f).tobytes() == getattr(before, f).tobytes(), f
        assert pt.AccumulatedSamples == 1
        assert np.array_equal(pt.Result.view(np.uint32), image.view(np.uint32))
        # a layout with a hole before the last BLAS (set through SetScene) is refused for a range before it
        shifted = copy.deepcopy(scene)
        d = shifted.blas_descs
        pad = np.zeros(2, shifted.blas_nodes.dtype)
        o = int(d[2]["NodeOffset"])
        shifted.blas_nodes = np.concatenate([shifted.blas_nodes[:o], pad, shifted.blas_nodes[o:]])
        d["NodeOffset"][2] += 2
        pt.SetScene(shifted)
        with pytest.raises(IdkPtError, match=f"failed \\({ERR_INVALID_ARGUMENT}\\)"):
            pt.RebuildBlases(1, 1)
        pt.RebuildBlases(2, 1)                            # the first desc of the range may start anywhere
        assert read_scene(pt, shifted).blas_descs[2]["NodeOffset"] == o


def test_rebuild_between_queued_samples():
    scene = room_crate_ball()
    scene.build_tlas()
    u, jm, cmd = skinning_setup(scene, 1)
    s = settings()
    images = []
    for asynchronous in (False, True):
        pt, frame = opened(scene, s)
        with pt:
            pt.SetSkinningData(u)
            (pt.ComputeAsync if asynchronous else pt.Compute)()
            pt.SkinVertices(jm, cmd)
            pt.RebuildBlases(1, 1)
            pt.TlasBuild()
            for _ in range(2):
                (pt.ComputeAsync if asynchronous else pt.Compute)()
            pt.Sync()
            images.append(pt.Result.copy())
    assert np.array_equal(images[0].view(np.uint32), images[1].view(np.uint32))


def test_blas_sah():
    scene = room_crate_ball()
    scene.build_tlas()
    u, jm, cmd = skinning_setup(scene, 1)
    nd = len(scene.blas_descs)

    def host_sah(sc, cost=None):
        return np.array([host.blas_global_sah(sc.blas_nodes[d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]], cost) for d in sc.blas_descs])

    pt, frame = opened(scene)
    with pt:
        fresh = pt.BlasSah(0, nd)
        assert fresh.tobytes() == np.array([i["sah"] for i in scene.build_info]).tobytes()
        assert fresh.tobytes() == host_sah(read_scene(pt, scene)).tobytes()
        cost = host.default_build_settings()
        cost.TriangleCost = 2.0
        assert pt.BlasSah(0, nd, settings=cost).tobytes() == host_sah(scene, 2.0).tobytes()
        assert pt.BlasSah(1, 0).size == 0
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(1, 1)
        refit = pt.BlasSah(1)
        assert refit.tobytes() == host_sah(read_scene(pt, scene))[1:2].tobytes()
        assert refit[0] > fresh[1]
        pt.RebuildBlases(1, 1)
        rebuilt = pt.BlasSah(0, nd)
        want = mirror(pt, scene, 1, 1)
        assert rebuilt.tobytes() == host_sah(want).tobytes()
        assert rebuilt[1] == want.build_info[1]["sah"] and rebuilt[1] < refit[0]
        with pytest.raises(IdkPtError, match=f"failed \\({ERR_INVALID_ARGUMENT}\\)"):
            pt.BlasSah(2, 2)


def test_large_refittable_atrium(monkeypatch):
    orig = host.Scene.add

    def add_refittable(self, *models, **kw):
        for m in models:
            m.refittable = True
        return orig(self, *models, **kw)

    monkeypatch.setattr(host.Scene, "add", add_refittable)
    scene, cam = scenes.atrium(262144, threads=ol.default_threads())
    monkeypatch.undo()
    assert scene.blas_descs[0]["IsRefittable"] == 1
    scene.build_tlas()
    u, jm, cmd = skinning_setup(scene, 0)
    with PathTracer(64, 48) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(0, 1)
        refit = pt.BlasSah(0)[0]
        pt.RebuildBlases(0, 1)
        pt.TlasBuild()
        want = mirror(pt, scene, 0, 1)
        assert_scene(pt, want)
        assert pt.BlasSah(0)[0] == want.build_info[0]["sah"] < refit
        rays = ol.primary_rays(scenes.camera_frame(cam, 64, 48), 64, 48)
        assert_traces(pt, want, rays)
