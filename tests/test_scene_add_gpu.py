"""idkpt_add_models (PathTracer.AddModels: ModelManager.Add on the device scene in place). The mirror of every case is
host.Scene.add of the same models onto a copy of the base scene, with the texture handles rebased onto the scene's table,
plus build_tlas() when the base uses a TLAS. Every comparison is exact."""
import copy
import ctypes

import numpy as np
import pytest

import oracle_lib as ol
from idkengine_b200 import capi, host, scenes, vxgi
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, deferred_setup, skinning_setup
from test_blas_rebuild_gpu import CAM, H, SKY, W, assert_image, assert_traces, opened, settings
from test_blas_rebuild_gpu import mirror as rebuild_mirror

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_NO_SCENE, ERR_UNSUPPORTED = -1, -4, -6
ARRAYS = ("blas_descs", "blas_nodes", "blas_triangles", "positions", "vertices", "tlas_nodes")


def with_handles(model, offset):
    """A copy of `model` whose texture handles k > 0 are moved behind `offset` textures."""
    m = copy.copy(model)
    m.materials = model.materials.copy()
    for f in host.TEXTURE_SLOTS:
        h = m.materials[f]
        m.materials[f] = np.where(h > 0, h + np.uint64(offset), np.uint64(0))
    return m


def placed(model, matrix):
    m = copy.copy(model)
    m.model_matrix = np.asarray(matrix, np.float64)
    return m


def mirror(base, models, textures=()):
    want = copy.deepcopy(base)
    want.add(*[with_handles(m, len(base.textures)) for m in models], threads=ol.default_threads())
    want.textures = want.textures + list(textures)
    if base.use_tlas:
        want.build_tlas()
    return want


def read(pt, like):
    """The device's arrays as a Scene shaped like `like`."""
    out = copy.deepcopy(like)
    out.blas_descs = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_DESCS, 0, len(like.blas_descs))
    out.blas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, len(like.blas_nodes))
    out.blas_triangles = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_TRIANGLES, 0, len(like.blas_triangles))
    out.positions = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(like.positions))
    out.vertices = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(like.vertices))
    if like.use_tlas:
        out.tlas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(like.tlas_nodes))
    return out


def assert_arrays(pt, want):
    got = read(pt, want)
    for f in ARRAYS:
        assert getattr(got, f).tobytes() == getattr(want, f).tobytes(), f
    last = want.blas_descs[-1]
    with pytest.raises(IdkPtError):    # and nothing more: the totals are the mirror's
        pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, int(last["NodeOffset"] + last["NodeCount"]) + 1)


def check(pt, frame, want, s, rays=None):
    assert_arrays(pt, want)
    assert_traces(pt, want, rays)
    assert_image(pt, want, frame, s)


def room_base(use_tlas):
    room, ball, crate = scenes.multi_blas_models()
    base = host.Scene().add(room, threads=1)
    base.add_light((-1.0, 2.5, 1.0), (30.0, 28.0, 20.0), 0.3)
    if use_tlas:
        base.build_tlas()
    return base, ball, crate


def captured(make, **kw):
    """(the Scene `make` returns, the models it added to it)."""
    got = []

    class Recording(host.Scene):
        def add(self, *models, **akw):
            got.extend(models)
            return super().add(*models, **akw)

    orig = scenes.Scene
    scenes.Scene = Recording
    try:
        out = make(**kw)
    finally:
        scenes.Scene = orig
    return out, got


# ---------------------------------------------------------------------------------------------------- the mirror
@pytest.mark.parametrize("use_tlas", [False, True], ids=["no_tlas", "tlas"])
def test_refittable_and_pre_split_models_in_one_call(use_tlas):
    base, ball, crate = room_base(use_tlas)
    s = settings()
    pt, frame = opened(base, s)
    with pt:
        pt.Compute()
        ms = pt.AddModels(ball, crate)
        assert ms > 0 and pt.AccumulatedSamples == 0
        want = mirror(base, [ball, crate])
        assert list(want.blas_descs["IsRefittable"]) == [0, 0, 1]
        assert want.use_tlas == use_tlas and len(want.tlas_nodes) == (5 if use_tlas else 0)
        check(pt, frame, want, s)


@pytest.mark.parametrize("use_tlas", [False, True], ids=["no_tlas", "tlas"])
def test_several_models_one_at_a_time_and_at_once(use_tlas):
    base, ball, crate = room_base(use_tlas)
    small = placed(crate, host.trs_matrix(0.5, 10.0, (-1.5, 1.0, -1.5)))
    want = mirror(base, [ball, crate, small])
    s = settings()
    results = []
    for calls in ([[ball], [crate, small]], [[ball, crate, small]], None):
        pt, frame = opened(want if calls is None else base, s)
        with pt:
            for c in calls or []:
                pt.AddModels(*c)
            check(pt, frame, want, s)
            results.append(pt.Result.copy())
    assert all(np.array_equal(r.view(np.uint32), results[0].view(np.uint32)) for r in results)


def test_textured_model_with_call_local_handles():
    (base, cam), models = captured(scenes.textured_room, threads=1)
    base.build_tlas()
    extra = placed(models[0], host.trs_matrix(0.25, 30.0, (0.6, 0.3, 0.2)))
    textures = base.textures[2:] + base.textures[:2]          # another order: handles are local to the call's table
    extra = copy.copy(extra)
    extra.materials = extra.materials.copy()
    for f in host.TEXTURE_SLOTS:
        h = extra.materials[f].astype(np.int64)
        extra.materials[f] = np.where(h > 0, (h - 3) % len(textures) + 1, 0).astype(np.uint64)
    s = settings()
    pt, frame = opened(base, s)
    with pt:
        pt.AddModels(extra, textures=textures)
        want = mirror(base, [extra], textures)
        assert want.materials["BaseColorTexture"][-8] == len(base.textures) + (1 - 3) % 8 + 1   # the floor's texture
        check(pt, frame, want, s)


def test_atrium_added_to_a_small_scene():
    base, ball, crate = room_base(True)
    (_, acam), (atrium,) = captured(scenes.atrium, target_tris=262144, threads=ol.default_threads())
    with PathTracer(W, H, settings()) as pt:
        pt.SetScene(base)
        pt.AddModels(atrium)
        want = mirror(base, [atrium])
        assert len(want.blas_triangles) > 262144
        assert_arrays(pt, want)
        frame = scenes.camera_frame(acam, 64, 48)
        assert_traces(pt, want, ol.primary_rays(frame, 64, 48))


# ---------------------------------------------------------------------------------------------------- what the call keeps
def raster_frame(pt, frame):
    g = pt.GBuffer(frame, W, H, jitter=JITTER)
    ao = pt.Ssao(frame, g[0], g[1])
    lit = pt.DeferredLighting(frame, *g[:5], settings=capi.default_deferred_settings(), jitter=JITTER)
    rates = pt.ShadingRate(frame, g[5], source=capi.LIT_SOURCE_DEFERRED)
    taa = pt.TaaResolve(g[0], g[5], W, H, source=capi.LIT_SOURCE_DEFERRED)
    return [np.ascontiguousarray(a) for a in list(g) + [ao, lit, rates, taa]]


def exported(pt, n_shadows):
    return ([pt.GBufferDevicePtrs()[0].Depth, pt.SsaoDevicePtr(), pt.DeferredDevicePtr(), pt.ShadingRateDevicePtr(), pt.TaaDevicePtr()] +
            [pt.PointShadowDevicePtr(k) for k in range(n_shadows)])


def test_twin_contexts_keep_their_state():
    scene, cam, shadows = deferred_setup("multi_blas_tlas")
    frame = scenes.camera_frame(cam, W, H)
    far = placed(scenes.multi_blas_models()[1], host.trs_matrix(2.0, 0.0, (4000.0, 0.0, 4000.0)))   # beyond every far plane
    twins = [PathTracer(W, H) for _ in range(2)]
    try:
        for pt in twins:
            pt.SetScene(scene)
            pt.SetPointShadows(shadows, [32] * len(shadows))
            pt.RenderPointShadows()
            for _ in range(2):
                raster_frame(pt, frame)
        before = exported(twins[0], len(shadows))
        twins[0].AddModels(far)
        assert exported(twins[0], len(shadows)) == before
        for k in range(len(shadows)):
            assert np.array_equal(twins[0].ReadPointShadow(k), twins[1].ReadPointShadow(k))
        got, ref = (raster_frame(pt, frame) for pt in twins)
        for a, b in zip(got, ref):
            assert a.tobytes() == b.tobytes()
        assert_arrays(twins[0], mirror(scene, [far]))
    finally:
        for pt in twins:
            pt.Dispose()


def test_prev_positions_restart_from_the_positions():
    base, ball, crate = room_base(False)
    u, jm, cmd = skinning_setup(base, 0)
    with PathTracer(W, H) as pt:
        pt.SetScene(base)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)                          # kept positions now differ from the positions
        old = pt.PrevPositionsDevicePtr()
        pt.AddModels(ball)
        want = mirror(base, [ball])
        p, n = pt.PrevPositionsDevicePtr()
        assert n == len(want.positions) * 12 and (p, n) != old
        frame = scenes.camera_frame(CAM, W, H)
        kept = pt.GBuffer(frame, W, H, jitter=JITTER, prev_positions="kept")
        now = pt.GBuffer(frame, W, H, jitter=JITTER)       # NULL: this frame's positions
        for a, b in zip(kept, now):
            assert np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def test_skinning_after_an_add():
    base, ball, crate = room_base(True)
    want = mirror(base, [ball, crate])
    u, jm, cmd = skinning_setup(want, 2)                 # the crate, appended behind no skinning data: input offset 0
    s = settings()
    pt, frame = opened(base, s)
    with pt:
        pt.AddModels(ball, crate, unskinned=u)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(2, 1)
        pt.TlasBuild()
        want.positions = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(want.positions))
        want.vertices = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(want.vertices))
        ol.blas_refit(want, 2)
        want.build_tlas()
        check(pt, frame, want, s)
        pt.RebuildBlases(2, 1)
        pt.TlasBuild()
        check(pt, frame, rebuild_mirror(pt, want, 2, 1), s)


@pytest.mark.parametrize("conservative", [False, True])
def test_bound_voxeliser_sees_the_added_models(conservative):
    base, ball, crate = room_base(True)
    lo, hi = (-3.2, -1.2, -3.2), (3.2, 4.2, 3.2)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(64, lo, hi) as bound, vxgi.Voxelizer(64, lo, hi) as owned:
        pt.SetScene(base)
        bound.SetSceneFrom(pt)
        bound.IsConservativeRasterization = owned.IsConservativeRasterization = conservative
        bound.Render()
        pt.AddModels(ball, crate)
        owned.SetScene(mirror(base, [ball, crate]))
        sb, so = bound.Render(), owned.Render()
        assert sb.Fragments == so.Fragments > 0
        for level in range(len(bound.sizes)):
            assert np.array_equal(bound.ReadLevel(level).view(np.uint16), owned.ReadLevel(level).view(np.uint16))


def test_queued_samples_finish_against_the_old_scene():
    base, ball, crate = room_base(True)
    s = settings()
    pt, frame = opened(base, s)
    with pt:
        pt.ComputeAsync()
        pt.ComputeAsync()
        pt.AddModels(ball)
        assert pt.AccumulatedSamples == 0
        res = np.zeros((H, W, 4), np.float32)
        o = ol.path_trace(base, frame, s, W, H, sky=SKY, result=res)
        ol.path_trace(base, frame, s, W, H, sky=SKY, accumulated=o.accumulated, result=res)
        assert np.array_equal(pt.Result.view(np.uint32), res.view(np.uint32))
        check(pt, frame, mirror(base, [ball]), s)


# ---------------------------------------------------------------------------------------------------- rejections
def raw_add(pt, rec, textures=(), settings=None, edit=None):
    d, keep = capi.add_models_desc(rec, textures)
    if edit:
        edit(d)
    st = PathTracer._blas_settings(settings)
    return pt._lib.idkpt_add_models(pt._ctx, ctypes.byref(d), ctypes.byref(st), None)


def test_rejections_leave_everything():
    base, ball, crate = room_base(True)
    with PathTracer(16, 16) as empty:
        assert raw_add(empty, host.model_records([ball])) == ERR_NO_SCENE
    pt, frame = opened(base)
    with pt:
        pt.Compute()
        image = pt.Result.copy()
        prev = pt.PrevPositionsDevicePtr()
        result = pt.ResultDevicePtr()
        rec = host.model_records([ball, crate])

        def changed(**edits):
            r = {k: v.copy() for k, v in rec.items()}
            for key, fn in edits.items():
                fn(r[key])
            return r

        def field(f, k, v):
            def fn(a):
                a[k][f] = v
            return fn

        def nullify(name):
            return lambda d: setattr(d, name, None)

        nan = host.default_build_settings()
        nan.TriangleCost = float("inf")
        stop = host.default_build_settings()
        stop.StopSplittingThreshold = 0
        n_tri, n_vtx = len(rec["triangles"]), len(rec["positions"])
        invalid = [
            dict(rec=rec, edit=nullify("Triangles")), dict(rec=rec, edit=nullify("Vertices")), dict(rec=rec, edit=nullify("BlasDescs")),
            dict(rec=changed(blas_instances=field("BlasId", 1, 2))),
            dict(rec=changed(blas_instances=field("MeshTransformId", 0, 2))),
            dict(rec=changed(triangles=field("Y", 5, n_vtx))),
            dict(rec=changed(triangles=field("MeshId", n_tri - 1, len(rec["meshes"])))),
            dict(rec=changed(triangles=field("MeshId", 0, -1))),
            dict(rec=changed(meshes=field("MaterialId", 0, len(rec["materials"])))),
            dict(rec=changed(materials=field("NormalTexture", 1, 1))),          # no textures in the call
            dict(rec=changed(blas_descs=field("TriangleCount", 1, 0))),
            dict(rec=changed(blas_descs=field("TriangleOffset", 1, n_tri - 2))),
            dict(rec=changed(blas_descs=field("TriangleOffset", 0, -1))),
            dict(rec=rec, settings=nan), dict(rec=rec, settings=stop),
        ]
        many = {k: v.copy() for k, v in rec.items()}
        many["blas_instances"] = np.zeros(16384, many["blas_instances"].dtype)   # 1 + 16384 instances under UseTlas
        unsupported = [dict(rec=rec, textures=[dict(format=99, width=4, height=4, data=np.zeros(64, np.uint8))]),
                       dict(rec=many)]
        cases = [(ERR_INVALID_ARGUMENT, c) for c in invalid] + [(ERR_UNSUPPORTED, c) for c in unsupported]
        for code, c in cases:
            assert raw_add(pt, c["rec"], c.get("textures", ()), c.get("settings"), c.get("edit")) == code, c
            assert_arrays(pt, base)
            assert pt.AccumulatedSamples == 1
            assert np.array_equal(pt.Result.view(np.uint32), image.view(np.uint32))
            assert pt.PrevPositionsDevicePtr() == prev and pt.ResultDevicePtr() == result
        assert raw_add(pt, host.model_records([])) == 0                      # an empty call does nothing
        assert pt.AccumulatedSamples == 1 and pt.PrevPositionsDevicePtr() == prev
        pt.AddModels(ball, crate)                                             # and the context still takes a valid one
        check(pt, frame, mirror(base, [ball, crate]), settings())
