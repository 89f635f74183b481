"""idkpt_collide_spheres (PathTracer.CollideSpheres): the engine's scene-versus-moving-sphere collision on the device scene.
Every case requires the device's Position, Velocity and Hits to equal oracle_collide_spheres byte for byte, over the scene
as set or, after a call that changes the scene on the device, over the arrays read back from it."""
import copy

import numpy as np
import pytest

import collision_oracle as co
import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt, host, scenes
from idkengine_b200.pathtracer import CAMERA_COLLISION, LIGHT_COLLISION, IdkPtError, PathTracer
from raster_lib import skinning_setup

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_NO_SCENE = -1, -4
PRESETS = pytest.mark.parametrize("settings", [LIGHT_COLLISION, CAMERA_COLLISION], ids=["lights", "camera"])


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


def assert_collide(pt, scene, s, settings):
    got, _ = pt.CollideSpheres(s, settings)
    want, _, _ = co.collide_spheres(scene, s, settings)
    for f in ("Position", "Velocity", "Hits"):
        assert got[f].tobytes() == want[f].tobytes(), (f, np.flatnonzero((got[f] != want[f]).reshape(len(s), -1).any(1))[:8])
    return got


def collide_on(scene, s, settings):
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        return assert_collide(pt, scene, s, settings)


def _atrium(instances):
    sc, _ = scenes.atrium(instances=instances, threads=ol.default_threads())
    if instances:
        sc.build_tlas()
    return sc


SCENES = {
    "closed_box": lambda: scenes.closed_box(subdiv=4, threads=1)[0],
    "open_floor": lambda: scenes.open_floor(threads=1)[0],
    "instance_grid": lambda: scenes.instance_grid(3, threads=1)[0],
    "atrium": lambda: _atrium(False),
    "atrium_instances_tlas": lambda: _atrium(True),
}


@PRESETS
@pytest.mark.parametrize("name", list(SCENES))
def test_scene_matches_the_oracle(name, settings):
    sc = SCENES[name]()
    s = random_spheres(sc, 2048, seed=len(name))
    got = collide_on(sc, s, settings)
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


@pytest.mark.parametrize("count", [0, 1, 257, 65536])
def test_counts(count):
    sc, _ = scenes.instance_grid(3, threads=1)
    s = random_spheres(sc, count, seed=count)
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        got = assert_collide(pt, sc, s, LIGHT_COLLISION)
        assert len(got) == count
        again, _ = pt.CollideSpheres(s, LIGHT_COLLISION)      # repeat calls give identical results
        assert again.tobytes() == got.tobytes()


def device_scene(pt, like):
    """The device's arrays as a Scene shaped like `like`; the instance list is `like`'s (the library does not export it)."""
    out = copy.deepcopy(like)
    out.blas_descs = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_DESCS, 0, len(like.blas_descs))
    last = out.blas_descs[-1]
    out.blas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, int(last["NodeOffset"] + last["NodeCount"]))
    out.blas_triangles = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_TRIANGLES, 0, int(last["TriangleOffset"] + last["TriangleCount"]))
    out.positions = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(like.positions))
    out.mesh_transforms = pt.ReadRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, 0, len(like.mesh_transforms))
    out.blas_stack_size = max(1, int(out.blas_descs["RequiredStackSize"].max()))
    return out


@PRESETS
@pytest.mark.parametrize("rig", ["animated_crowd", "animated_skinned_rig"])
def test_after_update_models(rig, settings):
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
            got = assert_collide(pt, device_scene(pt, sc), s, settings)
        assert (got["Hits"] > 0).any()


@PRESETS
def test_after_skinning_refit_and_rebuild(settings):
    sc, _ = scenes.multi_blas(threads=1)
    u, jm, cmd = skinning_setup(sc, 2)
    s = random_spheres(sc, 1024, seed=11, step=0.3, radius=(0.05, 0.4))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(2, 1)
        assert_collide(pt, device_scene(pt, sc), s, settings)
        pt.RebuildBlases(0, len(sc.blas_descs))
        got = assert_collide(pt, device_scene(pt, sc), s, settings)
    assert (got["Hits"] > 0).any()


@PRESETS
def test_after_add_models(settings):
    room, ball, crate = scenes.multi_blas_models()
    base = host.Scene().add(room, threads=1)
    base.build_tlas()
    s = random_spheres(base, 1024, seed=13, step=0.3, radius=(0.05, 0.4))
    added = copy.deepcopy(base)
    added.add(ball, crate, threads=1)
    with PathTracer(16, 16) as pt:
        pt.SetScene(base)
        assert_collide(pt, base, s, settings)
        pt.AddModels(ball, crate)
        got = assert_collide(pt, device_scene(pt, added), s, settings)
    assert (got["Hits"] > 0).any()


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


def test_refusals_leave_out_untouched():
    sc, _ = scenes.open_floor(threads=1)
    good = spheres([[0.0, 0.5, 0.0]], [[0.0, 0.1, 0.0]], 0.25)
    with PathTracer(16, 16) as pt:
        L, ctx = pt._lib, pt._ctx

        def call(s, st, n=None, null_spheres=False, null_out=False):
            out = np.full(32 * len(s), 0x5A, np.uint8)
            stp = None if st is None else np.array(tuple(st), gt.IdkPtCollisionSettings)
            rc = L.idkpt_collide_spheres(ctx, None if null_spheres else s.ctypes.data, len(s) if n is None else n,
                                         None if stp is None else stp.ctypes.data, None if null_out else out.ctypes.data, None)
            return rc, L.idkpt_last_error(ctx).decode(), bool((out == 0x5A).all())

        assert call(good, LIGHT_COLLISION) == (ERR_NO_SCENE, "idkpt_collide_spheres: no scene", True)
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
            assert call(**kw) == (ERR_INVALID_ARGUMENT, "idkpt_collide_spheres: " + text, True), (kw, text)
        with pytest.raises(IdkPtError, match="unknown Response"):
            pt.CollideSpheres(good, (1, 8, 0.001, 7))
        assert call(good[:0], LIGHT_COLLISION, null_spheres=True, null_out=True)[0] == 0   # count 0 takes null arrays
        assert_collide(pt, sc, good, CAMERA_COLLISION)  # a refusal leaves the context usable
