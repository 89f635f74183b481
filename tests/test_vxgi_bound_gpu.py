"""A voxeliser bound to a path tracer's device scene (idkvx_set_scene_from): the same grid as a voxeliser holding its own copy
of the same arrays, every level byte for byte; skinning, dirty-range updates and a new scene reach the next voxelisation with
no copy; the binding's lifetime and its ordering against queued path-tracer samples."""
import copy
import itertools

import numpy as np
import pytest

import oracle_lib as ol
import vxgi_conservative_oracle as vco
from idkengine_b200 import capi, scenes, vxgi
from idkengine_b200.host import mesh_transform, trs_matrix
from idkengine_b200.pathtracer import PathTracer
from raster_lib import GRID_MAX, GRID_MIN, TEX_GRID_MAX, TEX_GRID_MIN, lit_cornell, lit_cornell_shadowed, skinning_setup

pytestmark = pytest.mark.gpu

ERR_NO_SCENE = -4   # IdkPtStatus
MB_MIN, MB_MAX = (-3.2, -1.2, -3.2), (3.2, 4.2, 3.2)          # multi_blas
IG_MIN, IG_MAX = (-6.2, -1.0, -6.2), (6.2, 4.6, 6.2)          # instance_grid

SCENES = {
    # name: (scene, grid min, grid max)
    "cornell_1k": (lambda: lit_cornell(2)[0], GRID_MIN, GRID_MAX),
    "multi_blas": (lambda: scenes.multi_blas(threads=1)[0], MB_MIN, MB_MAX),
    "instance_grid": (lambda: scenes.instance_grid(threads=1)[0], IG_MIN, IG_MAX),
    "textured_room": (lambda: scenes.textured_room(threads=1)[0], TEX_GRID_MIN, TEX_GRID_MAX),
}
ORACLE_SCENES = ("multi_blas", "textured_room")
SIZES = [64, (40, 56, 30)]


def chain(vx):
    return [vx.ReadLevel(l).view(np.uint16) for l in range(len(vx.sizes))]


def assert_chain(got, want, what=""):
    assert len(got) == len(want)
    for l, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(np.asarray(a).view(np.uint16), np.asarray(b).view(np.uint16)), f"{what} level {l}"


def oracle(scene, ci, conservative=False):
    return (vco if conservative else ol).vx_voxelize(scene, ci)[0]


def raises_no_scene(vx, match=None):
    with pytest.raises(vxgi.IdkVxError, match=match) as e:
        vx.Render()
    assert f"failed ({ERR_NO_SCENE})" in str(e.value)


# ------------------------------------------------------------------------------------------------ static scenes
@pytest.mark.parametrize("conservative", [False, True])
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("name", sorted(SCENES))
def test_bound_equals_owned_copy(name, size, conservative):
    make, gmin, gmax = SCENES[name]
    scene = make()
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(size, gmin, gmax) as bound, vxgi.Voxelizer(size, gmin, gmax) as owned:
        pt.SetScene(scene)
        bound.SetSceneFrom(pt)
        owned.SetScene(scene)
        bound.IsConservativeRasterization = owned.IsConservativeRasterization = conservative
        sb, so = bound.Render(), owned.Render()
        assert sb.Fragments == so.Fragments > 0 and sb.KernelLaunches == so.KernelLaunches
        got = chain(bound)
        assert_chain(got, chain(owned))
    if name in ORACLE_SCENES:
        assert_chain(got, oracle(scene, vxgi.create_info(size, gmin, gmax), conservative), "oracle")


@pytest.mark.parametrize("conservative", [False, True])
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("mode", ["shadow_maps", "shadow_tracer"])
def test_bound_point_shadows_equal_owned_copy(mode, size, conservative):
    scene, shadows = lit_cornell_shadowed()
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as bound, vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as owned:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [96, 128])
        pt.RenderPointShadows()
        bound.SetSceneFrom(pt)
        owned.SetScene(scene)
        for vx in (bound, owned):
            vx.IsConservativeRasterization = conservative
            (vx.SetShadowMaps if mode == "shadow_maps" else vx.SetShadowTracer)(pt)
        sb, so = bound.Render(), owned.Render()
        assert sb.Fragments == so.Fragments > 0
        assert_chain(chain(bound), chain(owned))


# ------------------------------------------------------------------------------------------------ animated scenes
def test_skinned_scene_reaches_the_next_voxelisation():
    """Two skins with different joints: after each, the bound grid equals the oracle's grid of the skinned scene and that of
    a voxeliser given ReadRange's arrays; a BLAS refit and a TLAS build in between change nothing in it."""
    scene, _ = scenes.multi_blas(threads=1)
    scene.build_tlas()
    expect = copy.deepcopy(scene)
    u, jm, cmd = skinning_setup(scene, 2)
    jm2 = skinning_setup(scene, 2, seed=9)[1]
    ci = vxgi.create_info(64, MB_MIN, MB_MAX)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(64, MB_MIN, MB_MAX) as bound, vxgi.Voxelizer(64, MB_MIN, MB_MAX) as owned:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        bound.SetSceneFrom(pt)
        bound.Render()
        previous = chain(bound)
        for joints in (jm, jm2):
            pt.SkinVertices(joints, cmd)
            ol.skin_vertices(u, joints, expect.positions, expect.vertices, cmd[0])
            bound.Render()
            got = chain(bound)
            assert any(not np.array_equal(a, b) for a, b in zip(got, previous))
            assert_chain(got, oracle(expect, ci), "oracle")
            read = copy.deepcopy(scene)
            read.positions[:] = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(scene.positions))
            read.vertices[:] = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(scene.vertices))
            owned.SetScene(read)
            owned.Render()
            assert_chain(got, chain(owned), "read back")
            pt.BlasRefit(2, 1)
            pt.TlasBuild()
            bound.Render()
            assert_chain(chain(bound), got, "after refit and TLAS build")
            previous = got


# ------------------------------------------------------------------------------------------------ updates
def test_updates_reach_the_next_voxelisation():
    scene, _ = scenes.multi_blas(threads=1)
    expect = copy.deepcopy(scene)
    ci = vxgi.create_info(64, MB_MIN, MB_MAX)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(64, MB_MIN, MB_MAX) as bound:
        pt.SetScene(scene)
        bound.SetSceneFrom(pt)
        bound.Render()
        previous = [chain(bound)]

        def check(what):
            bound.Render()
            got = chain(bound)
            assert any(not np.array_equal(a, b) for a, b in zip(got, previous[0])), f"{what}: the grid did not change"
            assert_chain(got, oracle(expect, ci), what)
            previous[0] = got

        expect.mesh_transforms[1] = mesh_transform(trs_matrix(0.9, 30.0, (-1.0, 0.9, 0.2)))[0]
        pt.UpdateRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, 1, expect.mesh_transforms[1:2])
        check("instance moved")
        expect.lights["Position"][0] = (0.8, 2.2, -0.6)
        expect.lights["Color"][0] = (12.0, 30.0, 9.0)
        pt.UpdateRange(capi.IDKPT_ARRAY_LIGHTS, 0, expect.lights[0:1])
        check("light moved and recoloured")
        m = int(expect.meshes["MaterialId"][0])
        expect.materials["BaseColorFactor"][m] = 0xFF2040F0
        expect.materials["EmissiveFactor"][m] = (0.6, 0.1, 0.9)
        pt.UpdateRange(capi.IDKPT_ARRAY_MATERIALS, m, expect.materials[m:m + 1])
        check("material")
        expect.meshes["MaterialId"][0] = (m + 1) % len(expect.materials)
        pt.UpdateRange(capi.IDKPT_ARRAY_MESHES, 0, expect.meshes[0:1])
        check("mesh with another material")


def test_light_past_the_shadow_count_fails_and_keeps_the_grid():
    scene, shadows = lit_cornell_shadowed()
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(48, GRID_MIN, GRID_MAX) as bound:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [64, 64])
        pt.RenderPointShadows()
        bound.SetSceneFrom(pt)
        bound.SetShadowMaps(pt)
        bound.Render()
        before = chain(bound)
        lights = scene.lights.copy()
        lights["PointShadowIndex"][0] = 2
        pt.UpdateRange(capi.IDKPT_ARRAY_LIGHTS, 0, lights[0:1])
        with pytest.raises(vxgi.IdkVxError, match="not below the shadow-map context's shadow count"):
            bound.Render()
        assert_chain(chain(bound), before)


# ------------------------------------------------------------------------------------------------ lifetime and ordering
def test_new_scene_reaches_the_next_voxelisation():
    a, b = lit_cornell(2)[0], scenes.multi_blas(threads=1)[0]
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(48, MB_MIN, MB_MAX) as bound, vxgi.Voxelizer(48, MB_MIN, MB_MAX) as owned:
        pt.SetScene(a)
        bound.SetSceneFrom(pt)
        bound.Render()
        assert_chain(chain(bound), oracle(a, vxgi.create_info(48, MB_MIN, MB_MAX)), "first scene")
        pt.SetScene(b)
        bound.Render()
        owned.SetScene(b)
        owned.Render()
        assert_chain(chain(bound), chain(owned), "second scene")


def test_unbind_and_a_path_tracer_without_a_scene_give_no_scene():
    scene = lit_cornell(2)[0]
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(32, GRID_MIN, GRID_MAX) as vx:
        vx.SetSceneFrom(pt)
        raises_no_scene(vx, "path-tracer context bound with idkvx_set_scene_from has no scene")
        pt.SetScene(scene)
        vx.Render()
        vx.SetSceneFrom(None)
        raises_no_scene(vx)
        vx.SetSceneFrom(pt)
        vx.Render()
        vx.SetScene(scene)                  # back to an owned copy: a new path-tracer scene no longer reaches the grid
        grid = chain(vx)
        pt.SetScene(scenes.multi_blas(threads=1)[0])
        vx.Render()
        assert_chain(chain(vx), grid)


def test_disposing_the_path_tracer_gives_no_scene():
    scene = lit_cornell(2)[0]
    with vxgi.Voxelizer(32, GRID_MIN, GRID_MAX) as vx:
        pt = PathTracer(16, 16)
        pt.SetScene(scene)
        vx.SetSceneFrom(pt)
        vx.Render()
        grid = chain(vx)
        pt.Dispose()
        raises_no_scene(vx)
        vx.SetScene(scene)
        vx.Render()
        assert_chain(chain(vx), grid)
        with PathTracer(16, 16) as pt2:
            pt2.SetScene(scene)
            vx.SetSceneFrom(pt2)
            vx.Render()
            assert_chain(chain(vx), grid)


@pytest.mark.parametrize("order", list(itertools.permutations(["pt", "a", "b"])))
def test_two_voxelisers_on_one_path_tracer(order):
    """Dispose the path tracer and two voxelisers bound to it in every order: a voxeliser whose path tracer is gone reports
    no scene, one whose path tracer lives goes on voxelising."""
    scene = lit_cornell(2)[0]
    objs = {"pt": PathTracer(16, 16), "a": vxgi.Voxelizer(32, GRID_MIN, GRID_MAX), "b": vxgi.Voxelizer(32, GRID_MIN, GRID_MAX)}
    objs["pt"].SetScene(scene)
    objs["a"].SetSceneFrom(objs["pt"])
    objs["b"].SetSceneFrom(objs["pt"])
    objs["a"].Render()
    objs["b"].Render()
    grid = chain(objs["a"])
    assert_chain(chain(objs["b"]), grid)
    alive = set(objs)
    for name in order:
        objs[name].Dispose()
        alive.discard(name)
        for v in sorted(alive - {"pt"}):
            if "pt" in alive:
                objs[v].Render()
                assert_chain(chain(objs[v]), grid, v)
            else:
                raises_no_scene(objs[v])


def test_voxelise_between_queued_samples():
    """Three queued samples, then a bound voxelisation, then Sync: the grid and the accumulated image both equal the oracle."""
    scene, cam = lit_cornell(2)
    w, h = 96, 64
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    with PathTracer(w, h, s, lanes=3) as pt, vxgi.Voxelizer(48, GRID_MIN, GRID_MAX) as vx:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(frame)
        vx.SetSceneFrom(pt)
        for _ in range(3):
            pt.ComputeAsync()
        vx.Render()
        pt.Sync()
        img = pt.Result.copy()
        assert pt.AccumulatedSamples == 3
        got = chain(vx)
    assert_chain(got, oracle(scene, vxgi.create_info(48, GRID_MIN, GRID_MAX)))
    res = np.zeros((h, w, 4), np.float32)
    acc = 0
    for _ in range(3):
        acc = ol.path_trace(scene, frame, s, w, h, accumulated=acc, result=res).accumulated
    assert np.array_equal(img.view(np.uint32), res.view(np.uint32))


def test_bound_slab_equals_owned_slab():
    scene = lit_cornell(2)[0]
    size = (40, 56, 30)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as bound, vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as owned:
        pt.SetScene(scene)
        bound.SetSceneFrom(pt)
        owned.SetScene(scene)
        for vx in (bound, owned):
            vx.SetSlab(11, 23)
        sb, so = bound.Render(), owned.Render()
        assert sb.Fragments == so.Fragments > 0
        assert_chain(chain(bound), chain(owned), "slab")
        bound.Mipmap()
        owned.Mipmap()
        assert_chain(chain(bound), chain(owned), "mip chain")
