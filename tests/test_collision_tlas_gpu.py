"""idkpt_collide_spheres_tlas (PathTracer.CollideSpheres(use_tlas=True)): the engine's scene-versus-moving-sphere collision
with BVH.CpuUseTlas, walking the device TLAS. Every case requires the device's Position, Velocity and Hits to equal
oracle_collide_spheres_tlas byte for byte, over the scene as set or, after a call that changes the scene on the device, over
the arrays read back from it, the TLAS nodes included."""
import copy

import numpy as np
import pytest

import collision_oracle as co
import collision_tlas_oracle as cto
import oracle_lib as ol
from idkengine_b200 import capi, gpu_types as gt, host, scenes
from idkengine_b200.pathtracer import CAMERA_COLLISION, LIGHT_COLLISION, IdkPtError, PathTracer
from raster_lib import skinning_setup
from test_collision_gpu import ERR_INVALID_ARGUMENT, ERR_NO_SCENE, PRESETS, device_scene, random_spheres, spheres
from test_collision_tlas import visit_order_case, with_tlas

pytestmark = pytest.mark.gpu


def check(pt, scene, s, settings, use_tlas=True):
    got, _ = pt.CollideSpheres(s, settings, use_tlas=use_tlas)
    want, _, _ = cto.collide_spheres(scene, s, settings) if use_tlas else co.collide_spheres(scene, s, settings)
    for f in ("Position", "Velocity", "Hits"):
        assert got[f].tobytes() == want[f].tobytes(), (f, use_tlas, np.flatnonzero((got[f] != want[f]).reshape(len(s), -1).any(1))[:8])
    return got


def device_tlas(pt, like):
    """`like` with the device's TLAS nodes."""
    out = copy.deepcopy(like)
    out.tlas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * len(like.blas_instances) - 1)
    return out


def device_scene_tlas(pt, like):
    """The device's arrays, its TLAS nodes included, as a Scene shaped like `like`."""
    out = device_scene(pt, like)
    out.tlas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * len(like.blas_instances) - 1)
    return out


def _atrium_tlas():
    sc, _ = scenes.atrium(threads=ol.default_threads())
    return with_tlas(sc)


# name: (scene, whether the device builds the TLAS after the scene is set)
SCENES = {
    "instance_grid": (lambda: scenes.instance_grid(3, threads=1)[0], False),
    "atrium_tlas": (_atrium_tlas, False),
    "grid_4096_device_tlas": (lambda: scenes._instanced(scenes._grid_matrices(4096)), True),
    "closed_box_tlas": (lambda: with_tlas(scenes.closed_box(subdiv=4, threads=1)[0]), False),
}


@PRESETS
@pytest.mark.parametrize("name", list(SCENES))
def test_scene_matches_the_oracle(name, settings):
    make, build = SCENES[name]
    sc = make()
    s = random_spheres(sc, 2048, seed=len(name))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        if build:
            pt.TlasBuild()
            sc = device_tlas(pt, sc)
        got = check(pt, sc, s, settings)
    assert (got["Hits"] > 0).sum() >= 16, (got["Hits"] > 0).sum()


@PRESETS
def test_ties_go_to_the_depth_first_instance(settings):
    """Spheres half-way between two stacked quads whose depth-first TLAS order is not their index order: the TLAS walk
    settles the tie on the other quad than the linear walk does, and so moves the sphere the other way."""
    sc, s, want = visit_order_case()
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        tl = check(pt, sc, s, settings)
        lin = check(pt, sc, s, settings, use_tlas=False)
    assert len(want) >= 2 and (tl["Hits"] > 0).all()
    assert (tl["Position"] != lin["Position"]).any(1).all()


@pytest.mark.parametrize("count", [0, 1, 257, 65536])
def test_counts(count):
    sc, _ = scenes.instance_grid(3, threads=1)
    s = random_spheres(sc, count, seed=count)
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        got = check(pt, sc, s, LIGHT_COLLISION)
        assert len(got) == count
        again, _ = pt.CollideSpheres(s, LIGHT_COLLISION, use_tlas=True)      # repeat calls give identical results
        assert again.tobytes() == got.tobytes()


@PRESETS
def test_full_size_grid(settings):
    """The 262 144-instance grid with its TLAS built on the device, 65 536 spheres."""
    sc = scenes._instanced(scenes._grid_matrices(262144))
    s = random_spheres(sc, 65536, seed=5)
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.TlasBuild()
        got = check(pt, device_tlas(pt, sc), s, settings)
    assert (got["Hits"] > 0).sum() >= 16


@PRESETS
def test_after_update_models(settings):
    sc, anim = scenes.animated_crowd(64)
    s = random_spheres(sc, 1024, seed=7, step=0.3, radius=(0.05, 0.4))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.SetAnimations(anim)
        for t in (0.3, 0.8):
            pt.UpdateModels(t)
            got = check(pt, device_scene_tlas(pt, sc), s, settings)
    assert (got["Hits"] > 0).any()


@PRESETS
def test_after_skinning_refit_and_rebuild(settings):
    sc, _ = scenes.multi_blas(threads=1)
    sc.build_tlas()
    u, jm, cmd = skinning_setup(sc, 2)
    s = random_spheres(sc, 1024, seed=11, step=0.3, radius=(0.05, 0.4))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(2, 1)
        pt.TlasBuild()
        check(pt, device_scene_tlas(pt, sc), s, settings)
        pt.RebuildBlases(0, len(sc.blas_descs))
        pt.TlasBuild()
        got = check(pt, device_scene_tlas(pt, sc), s, settings)
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
        check(pt, base, s, settings)
        pt.AddModels(ball, crate)
        got = check(pt, device_scene_tlas(pt, added), s, settings)
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
        dev = device_scene_tlas(pt, sc)
        assert dev.tlas_nodes.tobytes() == before.tobytes() == sc.tlas_nodes.tobytes()
        tl = check(pt, dev, s, settings)
        lin = check(pt, dev, s, settings, use_tlas=False)
        assert pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(sc.tlas_nodes)).tobytes() == before.tobytes()
    assert (tl["Hits"][:64] == 0).all() and (lin["Hits"][:64] > 0).all()


def test_interleaved_modes_leave_the_image_and_the_accumulation_alone():
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
                check(pt, sc, s, st, use_tlas=use_tlas)
        assert pt.AccumulatedSamples == n and pt.Result.tobytes() == img.tobytes()


def test_refusals_leave_out_untouched():
    plain, _ = scenes.open_floor(threads=1)
    sc = with_tlas(scenes.open_floor(threads=1)[0])
    good = spheres([[0.0, 0.5, 0.0]], [[0.0, 0.1, 0.0]], 0.25)
    with PathTracer(16, 16) as pt:
        L, ctx = pt._lib, pt._ctx

        def call(s, st, n=None, null_spheres=False, null_out=False):
            out = np.full(32 * len(s), 0x5A, np.uint8)
            stp = None if st is None else np.array(tuple(st), gt.IdkPtCollisionSettings)
            rc = L.idkpt_collide_spheres_tlas(ctx, None if null_spheres else s.ctypes.data, len(s) if n is None else n,
                                              None if stp is None else stp.ctypes.data, None if null_out else out.ctypes.data, None)
            return rc, L.idkpt_last_error(ctx).decode(), bool((out == 0x5A).all())

        assert call(good, LIGHT_COLLISION) == (ERR_NO_SCENE, "idkpt_collide_spheres_tlas: no scene", True)
        pt.SetScene(plain)
        assert call(good, LIGHT_COLLISION) == (ERR_INVALID_ARGUMENT,
                                               "idkpt_collide_spheres_tlas: the scene was set without UseTlas (no TLAS to walk)", True)
        with pytest.raises(IdkPtError, match="without UseTlas"):
            pt.CollideSpheres(good, LIGHT_COLLISION, use_tlas=True)
        check(pt, plain, good, LIGHT_COLLISION, use_tlas=False)       # the linear call takes the same scene
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
            assert call(**kw) == (ERR_INVALID_ARGUMENT, "idkpt_collide_spheres_tlas: " + text, True), (kw, text)
        with pytest.raises(IdkPtError, match="unknown Response"):
            pt.CollideSpheres(good, (1, 8, 0.001, 7), use_tlas=True)
        assert call(good[:0], LIGHT_COLLISION, null_spheres=True, null_out=True)[0] == 0   # count 0 takes null arrays
        got = check(pt, sc, good, CAMERA_COLLISION)      # a refusal leaves the context usable
        assert got["Hits"][0] > 0
