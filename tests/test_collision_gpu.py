"""idkpt_collide_spheres and idkpt_collide_spheres_tlas (PathTracer.CollideSpheres, use_tlas=False / True): the engine's
scene-versus-moving-sphere collision on the device scene, over every instance in index order or, as with BVH.CpuUseTlas,
walking the device TLAS. Every case requires the device's Position, Velocity and Hits to equal oracle_collide_spheres under
the same walk byte for byte, over the scene as set or, after a call that changes the scene on the device, over the arrays
read back from it, the TLAS nodes included in TLAS mode."""
import copy

import numpy as np
import pytest

import collision_oracle as co
import oracle_lib as ol
from collision_oracle import random_spheres, spheres, visit_order_case, with_tlas
from idkengine_b200 import capi, gpu_types as gt, host, scenes
from idkengine_b200.pathtracer import CAMERA_COLLISION, LIGHT_COLLISION, IdkPtError, PathTracer
from raster_lib import skinning_setup

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_NO_SCENE = -1, -4
PRESETS = pytest.mark.parametrize("settings", [LIGHT_COLLISION, CAMERA_COLLISION], ids=["lights", "camera"])
WALKS = pytest.mark.parametrize("use_tlas", [False, True], ids=["linear", "tlas"])


def assert_collide(pt, scene, s, settings, use_tlas=False):
    got, _ = pt.CollideSpheres(s, settings, use_tlas=use_tlas)
    want, _, _ = co.collide_spheres(scene, s, settings, use_tlas=use_tlas)
    for f in ("Position", "Velocity", "Hits"):
        assert got[f].tobytes() == want[f].tobytes(), (f, use_tlas, np.flatnonzero((got[f] != want[f]).reshape(len(s), -1).any(1))[:8])
    return got


def collide_on(scene, s, settings):
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        return assert_collide(pt, scene, s, settings)


def device_tlas(pt, like):
    """`like` with the device's TLAS nodes."""
    out = copy.deepcopy(like)
    out.tlas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * len(like.blas_instances) - 1)
    return out


def device_scene(pt, like, tlas=False):
    """The device's arrays, with tlas=True its TLAS nodes too, as a Scene shaped like `like`; the instance list is `like`'s
    (the library does not export it)."""
    out = device_tlas(pt, like) if tlas else copy.deepcopy(like)
    out.blas_descs = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_DESCS, 0, len(like.blas_descs))
    last = out.blas_descs[-1]
    out.blas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, int(last["NodeOffset"] + last["NodeCount"]))
    out.blas_triangles = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_TRIANGLES, 0, int(last["TriangleOffset"] + last["TriangleCount"]))
    out.positions = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(like.positions))
    out.mesh_transforms = pt.ReadRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, 0, len(like.mesh_transforms))
    out.blas_stack_size = max(1, int(out.blas_descs["RequiredStackSize"].max()))
    return out


def _atrium(instances):
    sc, _ = scenes.atrium(instances=instances, threads=ol.default_threads())
    if instances:
        sc.build_tlas()
    return sc


# Each walk's scenes (TLAS mode needs a scene set with UseTlas). name: (scene, whether the device builds the TLAS after the
# scene is set)
SCENES = {
    "linear": {
        "closed_box": (lambda: scenes.closed_box(subdiv=4, threads=1)[0], False),
        "open_floor": (lambda: scenes.open_floor(threads=1)[0], False),
        "instance_grid": (lambda: scenes.instance_grid(3, threads=1)[0], False),
        "atrium": (lambda: _atrium(False), False),
        "atrium_instances_tlas": (lambda: _atrium(True), False),
    },
    "tlas": {
        "instance_grid": (lambda: scenes.instance_grid(3, threads=1)[0], False),
        "atrium_tlas": (lambda: with_tlas(scenes.atrium(threads=ol.default_threads())[0]), False),
        "grid_4096_device_tlas": (lambda: scenes._instanced(scenes._grid_matrices(4096)), True),
        "closed_box_tlas": (lambda: with_tlas(scenes.closed_box(subdiv=4, threads=1)[0]), False),
    },
}


@PRESETS
@pytest.mark.parametrize("walk,name", [(walk, name) for walk in SCENES for name in SCENES[walk]])
def test_scene_matches_the_oracle(walk, name, settings):
    make, build = SCENES[walk][name]
    sc = make()
    s = random_spheres(sc, 2048, seed=len(name))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        if build:
            pt.TlasBuild()
            sc = device_tlas(pt, sc)
        got = assert_collide(pt, sc, s, settings, use_tlas=walk == "tlas")
    assert (got["Hits"] > 0).sum() >= 16, (got["Hits"] > 0).sum()


def _two_quads(gap):
    """A floor quad and, `gap` above it, a second model's quad: two instances."""
    meshes, mats = scenes._materials([dict(color=(0.6, 0.6, 0.6))])
    models = []
    for y in (0.0, gap):
        a = scenes._Assembler()
        a.add(scenes.quad([-2, y, -2], [-2, y, 2], [2, y, 2], [2, y, -2]), 0)
        models.append(a.model(meshes, mats, name=f"quad{y}"))
    return host.Scene().add(*models, threads=1)


@PRESETS
def test_ties_edge_cases_and_special_spheres(settings):
    floor, _ = scenes.open_floor(threads=1)
    # the floor quad's two triangles share the diagonal through (-4, 0, -4) .. (4, 0, 4): centres above it tie on that edge
    tie_edge = spheres([[0.5, 0.3, 0.5], [-1.0, 0.1, -1.0], [2.0, 0.2, 2.0]], [[0.5, 0.1, 0.5], [-1.0, 0.1, -1.0], [2.0, 0.0, 2.0]], 0.25)
    on_plane = spheres([[0.3, 0.0, 0.7], [0.3, 0.5, 0.7]], [[0.3, 0.0, 0.7], [0.3, 0.0, 0.7]], 0.25)   # a centre exactly on a triangle
    zero_r = spheres([[0.3, 0.1, 0.7], [0.3, 0.5, 0.7]], [[0.3, -0.1, 0.7], [0.3, 0.0, 0.7]], 0.0)
    still = spheres([[0.1, 0.2, 0.1], [1.0, 0.05, -1.0]], [[0.1, 0.2, 0.1], [1.0, 0.05, -1.0]], 0.25, [[0.0, -1.0, 0.0], [1.0, 0.0, 0.0]])
    for s in (tie_edge, on_plane, zero_r, still):
        collide_on(floor, s, settings)
    # two instances at equal distance from the centre
    quads = _two_quads(1.0)
    collide_on(quads, spheres([[0.2, 0.5, 0.3], [0.2, 0.6, 0.3]], [[0.2, 0.5, 0.3], [0.2, 0.5, 0.3]], 0.6), settings)
    # starting inside geometry: inside instance_grid's models and outside the closed box
    grid, _ = scenes.instance_grid(3, threads=1)
    inside = grid.mesh_transforms["ModelMatrix"][1:, :, 3].astype(np.float32)
    collide_on(grid, spheres(inside, inside + np.float32(0.05), 0.3), settings)
    box, _ = scenes.closed_box(threads=1)
    collide_on(box, spheres([[1.1, 1.0, 0.0], [0.0, -0.1, 0.0]], [[0.9, 1.0, 0.0], [0.0, 0.2, 0.3]], 0.3), settings)


@PRESETS
def test_ties_go_to_the_depth_first_instance(settings):
    """Spheres half-way between two stacked quads whose depth-first TLAS order is not their index order: the TLAS walk
    settles the tie on the other quad than the linear walk does, and so moves the sphere the other way."""
    sc, s, want = visit_order_case()
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        tl = assert_collide(pt, sc, s, settings, use_tlas=True)
        lin = assert_collide(pt, sc, s, settings)
    assert len(want) >= 2 and (tl["Hits"] > 0).all()
    assert (tl["Position"] != lin["Position"]).any(1).all()


@pytest.mark.parametrize("count", [0, 1, 257, 65536])
@WALKS
def test_counts(count, use_tlas):
    sc, _ = scenes.instance_grid(3, threads=1)
    s = random_spheres(sc, count, seed=count)
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        got = assert_collide(pt, sc, s, LIGHT_COLLISION, use_tlas)
        assert len(got) == count
        again, _ = pt.CollideSpheres(s, LIGHT_COLLISION, use_tlas=use_tlas)      # repeat calls give identical results
        assert again.tobytes() == got.tobytes()


@PRESETS
def test_full_size_grid(settings):
    """The 262 144-instance grid with its TLAS built on the device, 65 536 spheres."""
    sc = scenes._instanced(scenes._grid_matrices(262144))
    s = random_spheres(sc, 65536, seed=5)
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.TlasBuild()
        got = assert_collide(pt, device_tlas(pt, sc), s, settings, use_tlas=True)
    assert (got["Hits"] > 0).sum() >= 16


@PRESETS
@pytest.mark.parametrize("use_tlas,rig", [(False, "animated_crowd"), (False, "animated_skinned_rig"), (True, "animated_crowd")],
                         ids=["linear-animated_crowd", "linear-animated_skinned_rig", "tlas-animated_crowd"])
def test_after_update_models(use_tlas, rig, settings):
    if rig == "animated_crowd":
        sc, anim = scenes.animated_crowd(64)
        unskinned = None
    else:
        sc, anim, unskinned = scenes.animated_skinned_rig()
    s = random_spheres(sc, 1024, seed=7, step=0.3, radius=(0.05, 0.4))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        if unskinned is not None:
            pt.SetSkinningData(unskinned)
        pt.SetAnimations(anim)
        for t in (0.3, 0.8):
            pt.UpdateModels(t)
            got = assert_collide(pt, device_scene(pt, sc, use_tlas), s, settings, use_tlas)
        assert (got["Hits"] > 0).any()


@PRESETS
@WALKS
def test_after_skinning_refit_and_rebuild(use_tlas, settings):
    sc, _ = scenes.multi_blas(threads=1)
    if use_tlas:
        sc.build_tlas()
    u, jm, cmd = skinning_setup(sc, 2)
    s = random_spheres(sc, 1024, seed=11, step=0.3, radius=(0.05, 0.4))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(2, 1)
        if use_tlas:
            pt.TlasBuild()
        assert_collide(pt, device_scene(pt, sc, use_tlas), s, settings, use_tlas)
        pt.RebuildBlases(0, len(sc.blas_descs))
        if use_tlas:
            pt.TlasBuild()
        got = assert_collide(pt, device_scene(pt, sc, use_tlas), s, settings, use_tlas)
    assert (got["Hits"] > 0).any()


@PRESETS
@WALKS
def test_after_add_models(use_tlas, settings):
    room, ball, crate = scenes.multi_blas_models()
    base = host.Scene().add(room, threads=1)
    base.build_tlas()
    s = random_spheres(base, 1024, seed=13, step=0.3, radius=(0.05, 0.4))
    added = copy.deepcopy(base)
    added.add(ball, crate, threads=1)
    with PathTracer(16, 16) as pt:
        pt.SetScene(base)
        assert_collide(pt, base, s, settings, use_tlas)
        pt.AddModels(ball, crate)
        got = assert_collide(pt, device_scene(pt, added, use_tlas), s, settings, use_tlas)
    assert (got["Hits"] > 0).any()


@PRESETS
def test_stale_tlas_is_walked_as_it_is(settings):
    """An instance moved by a transform upload without a TLAS rebuild: the walk still reads its old leaf box, so spheres
    dropped onto the instance's new place miss it in TLAS mode and hit it in linear mode; the call rebuilds nothing."""
    sc, _ = scenes.instance_grid(3, threads=1)
    k = 5
    mt = int(sc.blas_instances["MeshTransformId"][k])
    xf = sc.mesh_transforms[mt:mt + 1].copy()
    full = np.eye(4)
    full[:3, :] = xf["ModelMatrix"][0]
    full[:3, 3] += (40.0, 0.0, 0.0)
    xf["ModelMatrix"] = xf["PrevModelMatrix"] = full[:3, :].astype(np.float32)
    xf["InvModelMatrix"] = np.linalg.inv(full)[:3, :].astype(np.float32)
    centre = full[:3, 3].astype(np.float32)
    drop = spheres(np.repeat(centre[None] + np.float32([0.0, 1.5, 0.0]), 64, 0),
                   np.repeat(centre[None], 64, 0) + np.random.default_rng(3).uniform(-0.2, 0.2, (64, 3)).astype(np.float32), 0.5)
    s = np.concatenate([drop, random_spheres(sc, 1024, seed=19)])
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        before = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(sc.tlas_nodes))
        pt.UpdateRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, mt, xf)
        dev = device_scene(pt, sc, tlas=True)
        assert dev.tlas_nodes.tobytes() == before.tobytes() == sc.tlas_nodes.tobytes()
        tl = assert_collide(pt, dev, s, settings, use_tlas=True)
        lin = assert_collide(pt, dev, s, settings)
        assert pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(sc.tlas_nodes)).tobytes() == before.tobytes()
    assert (tl["Hits"][:64] == 0).all() and (lin["Hits"][:64] > 0).all()


def test_leaves_the_image_and_the_accumulation_alone():
    sc, cam = scenes.cornell_1k(threads=1)
    s = random_spheres(sc, 257, seed=3)
    with PathTracer(64, 48) as pt:
        pt.SetScene(sc)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(scenes.camera_frame(cam, 64, 48))
        pt.Compute()
        img, n = pt.Result, pt.AccumulatedSamples
        for st in (LIGHT_COLLISION, CAMERA_COLLISION):
            pt.CollideSpheres(s, st)
        assert pt.AccumulatedSamples == n and pt.Result.tobytes() == img.tobytes()


def test_interleaved_modes_leave_the_image_and_the_accumulation_alone():
    """TLAS-mode calls, interleaved with linear ones, leave the image and the accumulation count alone too."""
    sc, cam = scenes.cornell_1k(threads=1)
    sc.build_tlas()
    s = random_spheres(sc, 257, seed=3)
    with PathTracer(64, 48) as pt:
        pt.SetScene(sc)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(scenes.camera_frame(cam, 64, 48))
        pt.Compute()
        img, n = pt.Result, pt.AccumulatedSamples
        for st in (LIGHT_COLLISION, CAMERA_COLLISION):
            for use_tlas in (True, False, True):
                assert_collide(pt, sc, s, st, use_tlas)
        assert pt.AccumulatedSamples == n and pt.Result.tobytes() == img.tobytes()


def check_refusals(use_tlas):
    """Every refusal of idkpt_collide_spheres (use_tlas=False) or idkpt_collide_spheres_tlas returns its status and text,
    prefixed with the entry point's name, with `out` untouched, and leaves the context usable."""
    entry = "idkpt_collide_spheres_tlas" if use_tlas else "idkpt_collide_spheres"
    plain, _ = scenes.open_floor(threads=1)
    sc = with_tlas(scenes.open_floor(threads=1)[0]) if use_tlas else plain
    good = spheres([[0.0, 0.5, 0.0]], [[0.0, 0.1, 0.0]], 0.25)
    with PathTracer(16, 16) as pt:
        L, ctx = pt._lib, pt._ctx

        def call(s, st, n=None, null_spheres=False, null_out=False):
            out = np.full(32 * len(s), 0x5A, np.uint8)
            stp = None if st is None else np.array(tuple(st), gt.IdkPtCollisionSettings)
            rc = getattr(L, entry)(ctx, None if null_spheres else s.ctypes.data, len(s) if n is None else n,
                                   None if stp is None else stp.ctypes.data, None if null_out else out.ctypes.data, None)
            return rc, L.idkpt_last_error(ctx).decode(), bool((out == 0x5A).all())

        assert call(good, LIGHT_COLLISION) == (ERR_NO_SCENE, entry + ": no scene", True)
        if use_tlas:
            pt.SetScene(plain)
            assert call(good, LIGHT_COLLISION) == (ERR_INVALID_ARGUMENT, entry + ": the scene was set without UseTlas (no TLAS to walk)", True)
            with pytest.raises(IdkPtError, match="without UseTlas"):
                pt.CollideSpheres(good, LIGHT_COLLISION, use_tlas=True)
            assert_collide(pt, plain, good, LIGHT_COLLISION)       # the linear call takes the same scene
        pt.SetScene(sc)
        cases = [
            (dict(s=good, st=LIGHT_COLLISION, null_spheres=True), "null argument"),
            (dict(s=good, st=LIGHT_COLLISION, null_out=True), "null argument"),
            (dict(s=good, st=None), "null argument"),
            (dict(s=good, st=LIGHT_COLLISION, n=1 << 31), "too many spheres"),
            (dict(s=good, st=(0, 8, 0.001, 1)), "TestSteps must be at least 1"),
            (dict(s=good, st=(1, -1, 0.001, 1)), "RecursiveSteps outside 0..IDKPT_MAX_COLLISION_RECURSIVE_STEPS"),
            (dict(s=good, st=(1, 65, 0.001, 1)), "RecursiveSteps outside 0..IDKPT_MAX_COLLISION_RECURSIVE_STEPS"),
            (dict(s=good, st=(1, 8, 0.001, 2)), "unknown Response"),
            (dict(s=good, st=(1, 8, 0.001, -1)), "unknown Response"),
        ]
        for bad_r in (-0.5, np.inf, np.nan):
            b = good.copy()
            b["Radius"] = bad_r
            cases.append((dict(s=b, st=LIGHT_COLLISION), "a Radius is negative or not finite"))
        for kw, text in cases:
            assert call(**kw) == (ERR_INVALID_ARGUMENT, entry + ": " + text, True), (kw, text)
        with pytest.raises(IdkPtError, match="unknown Response"):
            pt.CollideSpheres(good, (1, 8, 0.001, 7), use_tlas=use_tlas)
        assert call(good[:0], LIGHT_COLLISION, null_spheres=True, null_out=True)[0] == 0   # count 0 takes null arrays
        got = assert_collide(pt, sc, good, CAMERA_COLLISION, use_tlas)      # a refusal leaves the context usable
        assert got["Hits"][0] > 0


def test_refusals_leave_out_untouched():
    check_refusals(use_tlas=False)


def test_refusals_leave_out_untouched_tlas():
    check_refusals(use_tlas=True)
