"""The lifecycle of the device scene across the calls that replace or edit it: idkpt_set_scene, idkpt_blas_build(_batch),
idkpt_blas_rebuild, idkpt_add_models, idkpt_tlas_build, the TLAS step of idkpt_update_models and idkvx_set_scene.

- Every refusal returns its code with its full idkpt_last_error / idkvx_last_error text.
- A refusal that must change nothing leaves every array idkpt_read_range can read, the accumulation and a path-traced image
  byte for byte as they were.
- After a rebuild and after an add, a bound voxeliser and trace_rays see the same scene as a context freshly given the same
  arrays: the scene view the call left names the new arrays and nothing stale."""
import copy
import ctypes

import numpy as np
import pytest

from idkengine_b200 import capi, host, scenes, vxgi
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from test_blas_rebuild import random_rays, room_crate_ball
from test_blas_rebuild_gpu import read_scene
from test_scene_add_gpu import mirror, raw_add, read, room_base
from test_tlas_build_gpu import instanced, matrices

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_NO_SCENE, ERR_UNSUPPORTED = -1, -4, -6
N = 64
SKY = (0.6, 0.7, 0.9)
CAM = dict(position=(0.0, 1.6, 5.0), view_dir=(0.0, -0.1, -1.0), fov_y_deg=60.0)
READABLE = [(capi.IDKPT_ARRAY_BLAS_NODES, "blas_nodes"), (capi.IDKPT_ARRAY_VERTEX_POSITIONS, "positions"),
            (capi.IDKPT_ARRAY_VERTICES, "vertices"), (capi.IDKPT_ARRAY_TLAS_NODES, "tlas_nodes"),
            (capi.IDKPT_ARRAY_BLAS_TRIANGLES, "blas_triangles"), (capi.IDKPT_ARRAY_BLAS_DESCS, "blas_descs"),
            (capi.IDKPT_ARRAY_MESH_TRANSFORMS, "mesh_transforms")]
TLAS_STEP = "search radius out of range (TLAS.BuildSettings.SearchRadius, default 15)"
NOT_FINITE = "an instance's world box is not finite or its half area overflows (ModelMatrix or BLAS root)"


def last_error(pt):
    return pt._lib.idkpt_last_error(pt._ctx).decode()


def refused(pt, code, text, fn, *args, **kw):
    """fn raises IdkPtError with `code`, and the context's last error is `text`, whole."""
    with pytest.raises(IdkPtError, match=rf"failed \({code}\)"):
        fn(*args, **kw)
    assert last_error(pt) == text


def opened(scene):
    pt = PathTracer(N, N)
    pt.SetScene(scene)
    pt.SetSky(SKY)
    pt.SetFrame(scenes.camera_frame(CAM, N, N))
    return pt


def image(pt):
    pt.ResetAccumulation()
    pt.Compute()
    return pt.Result.view(np.uint32).copy()


class Unchanged:
    """What a context shows of its scene: every readable array at the scene's sizes, the accumulation and a 64x64 image."""

    def __init__(self, pt, scene):
        self.pt, self.scene = pt, scene
        self.arrays = self.read()
        self.image = image(pt)
        self.samples = pt.AccumulatedSamples

    def read(self):
        out = {}
        for which, name in READABLE:
            n = len(getattr(self.scene, name)) if (name != "tlas_nodes" or self.scene.use_tlas) else 0
            out[name] = self.pt.ReadRange(which, 0, n).tobytes()
            with pytest.raises(IdkPtError):               # and not one element more
                self.pt.ReadRange(which, 0, n + 1)
        return out

    def check(self):
        assert self.pt.AccumulatedSamples == self.samples
        assert self.read() == self.arrays
        assert np.array_equal(image(self.pt), self.image)


# ---------------------------------------------------------------------------------------------------- idkpt_set_scene
def test_set_scene_refusals():
    scene = room_crate_ball()
    scene.build_tlas()
    pt = opened(scene)
    with pt:
        kept = Unchanged(pt, scene)
        assert pt._lib.idkpt_set_scene(pt._ctx, None) == ERR_INVALID_ARGUMENT
        assert last_error(pt) == "idkpt_set_scene: null argument"
        kept.check()

        def edited(fn=None, desc=None):
            s = copy.deepcopy(scene)
            if fn:
                fn(s)
            d, keep = capi.scene_desc(s)
            if desc:
                desc(d)
            return pt._lib.idkpt_set_scene(pt._ctx, ctypes.byref(d))

        def field(name, f, k, v):
            def fn(s):
                getattr(s, name)[k][f] = v
            return fn

        def no_tlas(s):
            s.tlas_nodes = s.tlas_nodes[:-1]

        cases = [
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: a required array is null", None, lambda d: setattr(d, "BlasNodes", None)),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: a required array is null", None, lambda d: setattr(d, "Vertices", None)),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: BlasInstance references a missing BLAS or transform",
             field("blas_instances", "BlasId", 1, len(scene.blas_descs)), None),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: GpuBlasDesc triangle range outside the array",
             field("blas_descs", "TriangleCount", 2, len(scene.blas_triangles)), None),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: GpuBlasTriangle index out of range",
             field("blas_triangles", "Y", 5, len(scene.positions)), None),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: GpuBlasTriangle index out of range",
             field("blas_triangles", "MeshId", 7, len(scene.meshes)), None),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: GpuMesh.MaterialId out of range",
             field("meshes", "MaterialId", 0, len(scene.materials)), None),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: UseTlas needs 2*instances-1 TLAS nodes", no_tlas, None),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: GpuBlasDesc range outside the node array",
             field("blas_descs", "NodeOffset", 2, len(scene.blas_nodes)), None),
            (ERR_INVALID_ARGUMENT, "idkpt_set_scene: BlasStackSize smaller than a BLAS's RequiredStackSize",
             None, lambda d: setattr(d, "BlasStackSize", 0)),
            (ERR_UNSUPPORTED, "BlasStackSize too large for the shared-memory traversal stack",
             None, lambda d: setattr(d, "BlasStackSize", 1000)),
        ]
        for code, text, fn, desc in cases:
            assert edited(fn, desc) == code, text
            assert last_error(pt) == text
            kept.check()


# ---------------------------------------------------------------------------------------------------- BLAS builds
def test_blas_build_refusals():
    scene = room_crate_ball()
    pos, tris = scene.positions, scene.blas_triangles
    pt = opened(scene)
    with pt:
        kept = Unchanged(pt, scene)
        nan = capi.default_blas_build_settings()
        nan.SplitFactor = float("nan")
        stop = capi.default_blas_build_settings()
        stop.StopSplittingThreshold = 0
        bad = tris.copy()
        bad["Z"][11] = len(pos)
        refused(pt, ERR_INVALID_ARGUMENT, "idkpt_blas_build: no triangles", pt.BuildBlas, pos, tris[:0])
        refused(pt, ERR_INVALID_ARGUMENT, "idkpt_blas_build: vertex id out of range", pt.BuildBlas, pos, bad)
        refused(pt, ERR_INVALID_ARGUMENT, "idkpt_blas_build: non-finite setting", pt.BuildBlas, pos, tris, settings=nan)
        refused(pt, ERR_INVALID_ARGUMENT, "idkpt_blas_build: StopSplittingThreshold must be at least 1", pt.BuildBlas, pos, tris,
                settings=stop)
        h = ctypes.c_void_p()
        assert pt._lib.idkpt_blas_build(pt._ctx, None, len(pos), tris.ctypes.data, len(tris), None, ctypes.byref(h), None) == ERR_INVALID_ARGUMENT
        assert last_error(pt) == "idkpt_blas_build: null argument"
        kept.check()

        descs = scene.blas_descs
        who = "idkpt_blas_build_batch: "

        def desc(k, **kw):
            x = descs.copy()
            for f, v in kw.items():
                x[k][f] = v
            return x

        refused(pt, ERR_INVALID_ARGUMENT, who + "no BLASes", pt.BuildBlases, pos, tris, descs[:0])
        refused(pt, ERR_INVALID_ARGUMENT, who + "a BLAS without triangles", pt.BuildBlases, pos, tris, desc(1, TriangleCount=0))
        refused(pt, ERR_INVALID_ARGUMENT, who + "GpuBlasDesc triangle range outside the array", pt.BuildBlases, pos, tris,
                desc(2, TriangleOffset=-1))
        refused(pt, ERR_INVALID_ARGUMENT, who + "GpuBlasDesc triangle range outside the array", pt.BuildBlases, pos, tris[:-1], descs)
        refused(pt, ERR_INVALID_ARGUMENT, who + "vertex id out of range", pt.BuildBlases, pos, bad, descs)
        refused(pt, ERR_INVALID_ARGUMENT, who + "non-finite setting", pt.BuildBlases, pos, tris, descs, settings=nan)
        assert pt._lib.idkpt_blas_build_batch(pt._ctx, None, len(pos), tris.ctypes.data, len(tris), descs.ctypes.data, len(descs),
                                              None, ctypes.byref(h), None) == ERR_INVALID_ARGUMENT
        assert last_error(pt) == who + "null argument"
        kept.check()


# ---------------------------------------------------------------------------------------------------- idkpt_blas_rebuild
def test_blas_rebuild_refusals():
    scene = room_crate_ball()
    scene.build_tlas()
    with PathTracer(16, 16) as empty:
        refused(empty, ERR_NO_SCENE, "idkpt_blas_rebuild: no scene", empty.RebuildBlases, 0, 1)
    pt = opened(scene)
    with pt:
        kept = Unchanged(pt, scene)
        nan = host.default_build_settings()
        nan.TriangleCost = float("inf")
        stop = host.default_build_settings()
        stop.StopSplittingThreshold = 0
        who = "idkpt_blas_rebuild: "
        refused(pt, ERR_INVALID_ARGUMENT, who + "BLAS range outside BlasDescs", pt.RebuildBlases, 2, 2)
        refused(pt, ERR_INVALID_ARGUMENT, who + "non-finite setting", pt.RebuildBlases, 0, 1, settings=nan)
        refused(pt, ERR_INVALID_ARGUMENT, who + "StopSplittingThreshold must be at least 1", pt.RebuildBlases, 0, 1, settings=stop)
        kept.check()

        shifted = copy.deepcopy(scene)                    # a hole before the last BLAS
        o = int(shifted.blas_descs[2]["NodeOffset"])
        shifted.blas_nodes = np.concatenate([shifted.blas_nodes[:o], np.zeros(2, shifted.blas_nodes.dtype), shifted.blas_nodes[o:]])
        shifted.blas_descs["NodeOffset"][2] += 2
        pt.SetScene(shifted)
        kept = Unchanged(pt, shifted)
        refused(pt, ERR_INVALID_ARGUMENT, who + "the BLASes are not packed behind each other from the first one rebuilt", pt.RebuildBlases, 1, 1)
        kept.check()

        longer = copy.deepcopy(scene)                     # nodes behind the last BLAS
        longer.blas_nodes = np.concatenate([longer.blas_nodes, np.zeros(2, longer.blas_nodes.dtype)])
        pt.SetScene(longer)
        kept = Unchanged(pt, longer)
        refused(pt, ERR_INVALID_ARGUMENT, who + "the last BLAS does not end the node and triangle arrays", pt.RebuildBlases, 0, 1)
        kept.check()


# ---------------------------------------------------------------------------------------------------- idkpt_add_models
def test_add_models_refusals():
    base, ball, crate = room_base(True)
    with PathTracer(16, 16) as empty:
        assert raw_add(empty, host.model_records([ball])) == ERR_NO_SCENE
        assert last_error(empty) == "idkpt_add_models: no scene"
    pt = opened(base)
    with pt:
        kept = Unchanged(pt, base)
        prev = pt.PrevPositionsDevicePtr()
        rec = host.model_records([ball, crate])

        def changed(key, f, k, v):
            r = {name: a.copy() for name, a in rec.items()}
            r[key][k][f] = v
            return r

        def nullify(name):
            return lambda d: setattr(d, name, None)

        nan = host.default_build_settings()
        nan.TriangleCost = float("inf")
        stop = host.default_build_settings()
        stop.StopSplittingThreshold = 0
        n_tri, n_vtx = len(rec["triangles"]), len(rec["positions"])
        many = {name: a.copy() for name, a in rec.items()}
        many["blas_instances"] = np.zeros(16384, many["blas_instances"].dtype)   # 1 + 16384 instances: a chain under UseTlas
        infinite = {name: a.copy() for name, a in rec.items()}
        infinite["mesh_transforms"]["ModelMatrix"][1][1, 3] = np.inf
        who = "idkpt_add_models: "
        cases = [
            (ERR_INVALID_ARGUMENT, "a required array is null", dict(rec=rec, edit=nullify("Triangles"))),
            (ERR_INVALID_ARGUMENT, "a required array is null", dict(rec=rec, edit=nullify("Vertices"))),
            (ERR_INVALID_ARGUMENT, "BlasInstance references a BLAS or transform outside the call's arrays",
             dict(rec=changed("blas_instances", "BlasId", 1, 2))),
            (ERR_INVALID_ARGUMENT, "BlasInstance references a BLAS or transform outside the call's arrays",
             dict(rec=changed("blas_instances", "MeshTransformId", 0, 2))),
            (ERR_INVALID_ARGUMENT, "GpuBlasTriangle index outside the call's vertices or meshes", dict(rec=changed("triangles", "Y", 5, n_vtx))),
            (ERR_INVALID_ARGUMENT, "GpuBlasTriangle index outside the call's vertices or meshes", dict(rec=changed("triangles", "MeshId", 0, -1))),
            (ERR_INVALID_ARGUMENT, "GpuMesh.MaterialId outside the call's materials",
             dict(rec=changed("meshes", "MaterialId", 0, len(rec["materials"])))),
            (ERR_INVALID_ARGUMENT, "material texture handle outside the texture table (0 = white, k = Textures[k-1])",
             dict(rec=changed("materials", "NormalTexture", 1, 1))),
            (ERR_INVALID_ARGUMENT, "a BLAS without triangles", dict(rec=changed("blas_descs", "TriangleCount", 1, 0))),
            (ERR_INVALID_ARGUMENT, "GpuBlasDesc triangle range outside the call's triangles",
             dict(rec=changed("blas_descs", "TriangleOffset", 1, n_tri - 2))),
            (ERR_INVALID_ARGUMENT, "non-finite setting", dict(rec=rec, settings=nan)),
            (ERR_INVALID_ARGUMENT, "StopSplittingThreshold must be at least 1", dict(rec=rec, settings=stop)),
            (ERR_UNSUPPORTED, "texture format not supported (RGBA8 unorm / sRGB, BC7, BC5, BC4, R/RG/RGBA32F)",
             dict(rec=rec, textures=[dict(format=99, width=4, height=4, data=np.zeros(64, np.uint8))])),
            (ERR_UNSUPPORTED, "the TLAS is deeper than the 24-entry traversal stack of the TLAS walk (BVHIntersect.glsl:4)", dict(rec=many)),
            (ERR_INVALID_ARGUMENT, NOT_FINITE, dict(rec=infinite)),
        ]
        for code, text, c in cases:
            assert raw_add(pt, c["rec"], c.get("textures", ()), c.get("settings"), c.get("edit")) == code, text
            assert last_error(pt) == who + text
            kept.check()
            assert pt.PrevPositionsDevicePtr() == prev


# ---------------------------------------------------------------------------------------------------- TLAS builds
def test_tlas_build_refusals():
    with PathTracer(16, 16) as empty:
        refused(empty, ERR_NO_SCENE, "idkpt_tlas_build: no scene", empty.TlasBuild)
    flat = room_crate_ball()                              # no TLAS
    pt = opened(flat)
    with pt:
        kept = Unchanged(pt, flat)
        refused(pt, ERR_INVALID_ARGUMENT, "idkpt_tlas_build: the scene was set without UseTlas (no TLAS node array to fill)", pt.TlasBuild)
        kept.check()
        scene = copy.deepcopy(flat)
        scene.build_tlas()
        pt.SetScene(scene)
        kept = Unchanged(pt, scene)
        for radius in (0, 1025):
            refused(pt, ERR_INVALID_ARGUMENT, "idkpt_tlas_build: " + TLAS_STEP, pt.TlasBuild, radius)
            kept.check()

        sc = instanced(matrices(1000, "uniform"))         # a NaN model matrix: the build merges nothing and invalidates the scene
        pt.SetScene(sc)
        moved = sc.mesh_transforms.copy()
        moved["ModelMatrix"][500][0, 0] = np.nan
        pt.UpdateRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, 0, moved)
        refused(pt, ERR_INVALID_ARGUMENT, "idkpt_tlas_build: " + NOT_FINITE + "; scene invalidated; set it again", pt.TlasBuild)
        refused(pt, ERR_NO_SCENE, "idkpt_read_range: no scene", pt.ReadRange, capi.IDKPT_ARRAY_TLAS_NODES, 0, 1)

        m = np.zeros((16385, 3, 4))                       # a chain of 16384: deeper than the walk's stack
        m[:, 0, 0] = m[:, 1, 1] = m[:, 2, 2] = 1.0
        m[0, :, 3] = (5.0, 0.0, 0.0)
        pt.SetScene(instanced(m, blas_ids=np.full(16385, 2)))
        refused(pt, ERR_UNSUPPORTED, "idkpt_tlas_build: the built TLAS is deeper than the 24-entry traversal stack of the TLAS walk "
                "(scene invalidated; set it again)", pt.TlasBuild)
        refused(pt, ERR_NO_SCENE, "idkpt_read_range: no scene", pt.ReadRange, capi.IDKPT_ARRAY_TLAS_NODES, 0, 1)


def test_update_models_tlas_step_refusals():
    sc, anim, u = scenes.animated_skinned_rig()
    variants = [(copy.deepcopy(sc), True), (copy.deepcopy(sc), False)]
    variants[0][0].build_tlas()
    variants[1][0].use_tlas = 0
    variants[1][0].tlas_nodes = variants[1][0].tlas_nodes[:0]
    for scene, tlas in variants:
        with PathTracer(16, 16) as pt:
            pt.SetScene(scene)
            pt.SetSkinningData(u)
            pt.SetAnimations(anim)
            if tlas:
                for t, radius in ((0.2, 0), (0.4, 1025)):     # each time moves the rig, so the TLAS step runs
                    refused(pt, ERR_INVALID_ARGUMENT, "idkpt_update_models: " + TLAS_STEP, pt.UpdateModels, t, radius)
                assert pt.UpdateModels(0.6)[0] == 3
            else:
                refused(pt, ERR_INVALID_ARGUMENT, "idkpt_update_models: the scene was set without UseTlas (no TLAS node array to fill)",
                        pt.UpdateModels, 0.3)


# ---------------------------------------------------------------------------------------------------- idkvx_set_scene
def test_voxeliser_set_scene_refusals():
    scene = room_crate_ball()
    lo, hi = (-3.2, -1.2, -3.2), (3.2, 4.2, 3.2)
    with vxgi.Voxelizer(32, lo, hi) as vx:
        vx.SetScene(scene)
        before = vx.Render().Fragments
        levels = [vx.ReadLevel(k).tobytes() for k in range(len(vx.sizes))]

        def last():
            return vx._lib.idkvx_last_error(vx._ctx).decode()

        assert vx._lib.idkvx_set_scene(vx._ctx, None) == ERR_INVALID_ARGUMENT
        assert last() == "idkvx_set_scene: null argument"

        def edited(name, f, k, v):
            s = copy.deepcopy(scene)
            getattr(s, name)[k][f] = v
            return s

        lights = copy.deepcopy(scene)
        lights.lights = np.concatenate([lights.lights] * 257)
        cases = [
            ("idkvx_set_scene: BlasInstance references a missing BLAS or transform", edited("blas_instances", "MeshTransformId", 0, 99)),
            ("idkvx_set_scene: GpuBlasDesc triangle range outside the array", edited("blas_descs", "TriangleOffset", 1, -1)),
            ("idkvx_set_scene: GpuBlasTriangle index out of range", edited("blas_triangles", "X", 3, len(scene.vertices))),
            ("idkvx_set_scene: GpuMesh.MaterialId out of range", edited("meshes", "MaterialId", 1, -1)),
            ("idkvx_set_scene: more than 256 lights", lights),
        ]
        for text, s in cases:
            d, keep = capi.scene_desc(s)
            assert vx._lib.idkvx_set_scene(vx._ctx, ctypes.byref(d)) == ERR_INVALID_ARGUMENT, text
            assert last() == text
        d, keep = capi.scene_desc(scene)
        d.Meshes = None
        assert vx._lib.idkvx_set_scene(vx._ctx, ctypes.byref(d)) == ERR_INVALID_ARGUMENT
        assert last() == "idkvx_set_scene: a required array is null"
        assert vx.Render().Fragments == before                # the copy it holds is the old scene's
        assert [vx.ReadLevel(k).tobytes() for k in range(len(vx.sizes))] == levels


# ---------------------------------------------------------------------------------------------------- a commit leaves a usable context
LO, HI = (-3.2, -1.2, -3.2), (3.2, 4.2, 3.2)


def assert_as_fresh(pt, bound, want):
    """`bound` (bound to `pt` before the commit), trace_rays and a 64x64 image of `pt` equal a voxeliser and a path tracer
    freshly given `want`'s arrays."""
    with PathTracer(N, N) as fresh, vxgi.Voxelizer(64, LO, HI) as owned:
        fresh.SetScene(want)
        fresh.SetSky(SKY)
        fresh.SetFrame(scenes.camera_frame(CAM, N, N))
        owned.SetScene(want)
        sb, so = bound.Render(), owned.Render()
        assert sb.Fragments == so.Fragments > 0
        for level in range(len(bound.sizes)):
            assert bound.ReadLevel(level).tobytes() == owned.ReadLevel(level).tobytes(), level
        rays = random_rays()
        for trace, ref in ((pt.TraceRays, fresh.TraceRays), (pt.TraceRaysAny, fresh.TraceRaysAny)):
            got, _ = trace(rays, trace_lights=True)
            assert got.tobytes() == ref(rays, trace_lights=True)[0].tobytes()
            assert (got["T"] < 1e30).sum() > len(rays) // 10
        assert np.array_equal(image(pt), image(fresh))


def test_rebuild_leaves_a_usable_context():
    scene = room_crate_ball()
    scene.build_tlas()
    pt = opened(scene)
    with pt, vxgi.Voxelizer(64, LO, HI) as bound:
        bound.SetSceneFrom(pt)
        bound.Render()
        pt.RebuildBlases(1, 2)
        pt.TlasBuild()
        assert_as_fresh(pt, bound, read_scene(pt, scene))


def test_add_leaves_a_usable_context():
    base, ball, crate = room_base(True)
    pt = opened(base)
    with pt, vxgi.Voxelizer(64, LO, HI) as bound:
        bound.SetSceneFrom(pt)
        bound.Render()
        pt.AddModels(ball, crate)
        assert_as_fresh(pt, bound, read(pt, mirror(base, [ball, crate])))
