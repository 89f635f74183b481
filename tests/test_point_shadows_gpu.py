"""Point-shadow cube maps (k_point_shadow_faces) and the voxeliser's shadow-map mode on the GPU, bit for bit against the oracle."""
import copy

import numpy as np
import pytest

import oracle_lib as ol
import point_shadow_oracle as pso
from idkengine_b200 import multigpu, scenes, vxgi
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import GRID_MAX, GRID_MIN, lit_cornell_shadowed, skinning_setup


def scene_and_light(which):
    if which == "cornell":
        return scenes.cornell_1k(threads=1)[0], ((0.3, 1.1, 0.2), 0.35, 1.25)
    if which in ("multi_blas", "multi_blas_tlas"):
        scene = scenes.multi_blas(threads=1)[0]
        if which == "multi_blas_tlas":
            scene.build_tlas()
        return scene, ((0.2, 1.9, 0.8), 0.3, 60.0)
    scene = scenes.atrium(20000, threads=1)[0]
    return scene, ((0.0, 3.0, 0.5), 0.3, 60.0)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 7, 64, 512])
@pytest.mark.parametrize("which", ["cornell", "multi_blas", "multi_blas_tlas", "atrium"])
def test_gpu_cube_maps_match_oracle(which, size):
    scene, light = scene_and_light(which)
    sh = scenes.point_shadows([(*light, 0)])
    want = pso.point_shadow_render(scene, sh[0], size)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(sh, [size])
        assert np.all(pt.ReadPointShadow(0) == 65535)                    # allocation clears to ShadowMap.Fill(1.0)
        ms = pt.RenderPointShadows()
        got = pt.ReadPointShadow(0)
    assert np.array_equal(got, want)
    assert ms > 0
    if size >= 64:
        assert (got != 65535).mean() > 0.3 and len(np.unique(got)) > 100


@pytest.mark.gpu
def test_gpu_several_shadows_face_mask_and_device_ptr():
    scene, cam = scenes.cornell_1k(threads=1)
    sh = scenes.point_shadows([((0.3, 1.1, 0.2), 0.35, 1.25, 0), ((-0.5, 0.6, 0.5), 0.1, 60.0, 0), ((0.0, 1.9, 0.0), 0.05, 3.0, 0)])
    sizes = [33, 64, 8]
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(sh, sizes)
        pt.RenderPointShadows()                                           # all three in one call
        first = [pt.ReadPointShadow(i) for i in range(3)]
        for i in range(3):
            assert np.array_equal(first[i], pso.point_shadow_render(scene, sh[i], sizes[i])), i
            p, nbytes = pt.PointShadowDevicePtr(i)
            assert nbytes == first[i].nbytes
            import torch
            dev = torch.as_tensor(multigpu.DeviceArray(p, (nbytes // 2,), "<i2"), device="cuda").cpu().numpy().view(np.uint16)
            assert np.array_equal(dev.reshape(first[i].shape), first[i])
        # move the second light, keep the sizes (the maps stay), re-render only faces -X, -Y, -Z of it
        moved = sh.copy()
        moved[1]["Position"] = (-0.4, 0.9, 0.3)
        pt.SetPointShadows(moved, sizes)
        assert np.array_equal(pt.ReadPointShadow(1), first[1])
        pt.RenderPointShadows(1, 1, [0b101010])
        got = pt.ReadPointShadow(1)
        assert np.array_equal(got[[0, 2, 4]], first[1][[0, 2, 4]])       # untouched faces keep their previous bytes
        assert np.array_equal(got, pso.point_shadow_render(scene, moved[1], 64, 0b101010, inout=first[1]))
        assert not np.array_equal(got[[1, 3, 5]], first[1][[1, 3, 5]])
        assert np.array_equal(pt.ReadPointShadow(0), first[0]) and np.array_equal(pt.ReadPointShadow(2), first[2])
        pt.RenderPointShadows(0, 3, [0, 0, 0])                           # empty masks write nothing
        assert np.array_equal(pt.ReadPointShadow(1), got)
        pt.SetPointShadows(moved, [33, 65, 8])                           # other sizes: reallocated and cleared
        assert np.all(pt.ReadPointShadow(1) == 65535) and np.all(pt.ReadPointShadow(0) == 65535)


@pytest.mark.gpu
def test_gpu_point_shadow_errors():
    scene, cam = scenes.cornell_1k(threads=1)
    sh = scenes.point_shadows([((0.0, 1.0, 0.0), 0.1, 60.0, 0)])
    with PathTracer(16, 16) as pt:
        with pytest.raises(IdkPtError, match="idkpt_set_point_shadows: no scene"):
            pt.SetPointShadows(sh, [16])
        with pytest.raises(IdkPtError, match="idkpt_render_point_shadows: no scene"):
            pt.RenderPointShadows(0, 0)
        pt.SetScene(scene)
        for bad in (0, 16385, -3):
            with pytest.raises(IdkPtError, match="size outside 1..16384"):
                pt.SetPointShadows(sh, [bad])
        for near in (0.0, -1.0, np.nan):
            b = sh.copy(); b["NearPlane"] = near
            with pytest.raises(IdkPtError, match="NearPlane must be > 0"):
                pt.SetPointShadows(b, [16])
        for far in (0.1, 0.05, np.inf):
            b = sh.copy(); b["FarPlane"] = far
            with pytest.raises(IdkPtError, match="FarPlane must be > NearPlane"):
                pt.SetPointShadows(b, [16])
        with pytest.raises(IdkPtError, match="more than IDKPT_MAX_POINT_SHADOWS"):
            pt.SetPointShadows(np.repeat(sh, 129), [1] * 129)
        pt.SetPointShadows(np.repeat(sh, 128), [1] * 128)                  # the engine's limit itself is fine
        pt.SetPointShadows(sh, [16])
        with pytest.raises(IdkPtError, match="shadow range outside the set shadows"):
            pt.RenderPointShadows(0, 2)
        with pytest.raises(IdkPtError, match="shadow range outside the set shadows"):
            pt.RenderPointShadows(2, 0)
        with pytest.raises(IdkPtError, match="face mask has bits above the six faces"):
            pt.RenderPointShadows(0, 1, [0x40])
        with pytest.raises(IdkPtError, match="shadow index out of range"):
            pt.ReadPointShadow(1)
        with pytest.raises(IdkPtError, match="shadow index out of range"):
            pt.PointShadowDevicePtr(-1)
        with pytest.raises(IdkPtError, match="buffer too small"):
            pt._check(pt._lib.idkpt_read_point_shadow(pt._ctx, 0, np.zeros(4, np.uint16).ctypes.data, 8), "idkpt_read_point_shadow")
        pt.SetScene(scene)                                                # a new scene drops the shadows
        with pytest.raises(IdkPtError, match="shadow index out of range"):
            pt.ReadPointShadow(0)
        # voxelising with a light whose PointShadowIndex is not below the context's shadow count
        lit = copy.deepcopy(scene)
        lit.add_light((0.0, 1.6, 0.3), (6.0, 5.5, 5.0), 0.2)
        lit.add_light((-0.6, 0.5, 0.6), (0.5, 0.8, 3.0), 0.1)
        lit.lights["PointShadowIndex"][:] = [0, 1]
        pt.SetScene(lit)
        pt.SetPointShadows(sh, [16])
        with vxgi.Voxelizer(16, GRID_MIN, GRID_MAX) as vx:
            vx.SetScene(lit)
            vx.SetShadowMaps(pt)
            with pytest.raises(vxgi.IdkVxError, match="PointShadowIndex is not below the shadow-map context's shadow count"):
                vx.Render()
            assert vx._lib.idkvx_voxelize(vx._ctx, None) == -1                 # IDKPT_ERR_INVALID_ARGUMENT


@pytest.mark.gpu
def test_gpu_voxelize_with_shadow_maps_matches_oracle():
    scene, shadows = lit_cornell_shadowed()
    sizes = [96, 128]
    dims = (48, 40, 44)
    ci = vxgi.create_info(dims, GRID_MIN, GRID_MAX)
    maps = [pso.point_shadow_render(scene, shadows[i], sizes[i]) for i in range(2)]
    levels, raw, frags = pso.vx_voxelize_shadow_maps(scene, ci, shadows, maps)
    ray_levels, _, ray_frags = ol.vx_voxelize(scene, ci)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(dims, GRID_MIN, GRID_MAX) as vx:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, sizes)
        pt.RenderPointShadows()
        for i in range(2):
            assert np.array_equal(pt.ReadPointShadow(i), maps[i])
        vx.SetScene(scene)
        vx.SetShadowTracer(pt)
        vx.SetShadowMaps(pt)                                               # maps take precedence over the tracer
        s = vx.Render()
        assert s.Fragments == frags
        for l, lv in enumerate(levels):
            assert np.array_equal(vx.ReadLevel(l).view(np.uint16), lv.view(np.uint16)), f"level {l}"
        assert not np.array_equal(levels[0].view(np.uint16), ray_levels[0].view(np.uint16))
        vx.SetShadowMaps(None)                                             # detached: back to today's shadow rays
        s = vx.Render()
        assert s.Fragments == ray_frags
        for l, lv in enumerate(ray_levels):
            assert np.array_equal(vx.ReadLevel(l).view(np.uint16), lv.view(np.uint16)), f"shadow rays, level {l}"
        vx.SetShadowTracer(None)
        with pytest.raises(vxgi.IdkVxError, match="point-shadowed"):
            vx.Render()
        # z-slab voxelisation with maps: every slab equals that range of the single pass
        vx.SetShadowMaps(pt)
        d = dims[2]
        got = np.zeros_like(levels[0].view(np.uint16))
        for z0, z1 in ((0, 17), (17, 30), (30, d)):
            vx.SetSlab(z0, z1)
            vx.Render()
            l0 = vx.ReadLevel(0).view(np.uint16)
            assert not l0[:z0].any() and not l0[z1:].any()
            got[z0:z1] = l0[z0:z1]
        assert np.array_equal(got, levels[0].view(np.uint16))


@pytest.mark.gpu
def test_gpu_maps_after_skin_refit_tlas_build():
    scene, cam = scenes.multi_blas(threads=1)
    scene.build_tlas()
    expect = copy.deepcopy(scene)
    u, jm, cmd = skinning_setup(scene, 2)
    ol.skin_vertices(u, jm, expect.positions, expect.vertices, cmd[0])
    ol.blas_refit(expect, 2)
    expect.build_tlas()
    sh = scenes.point_shadows([((0.2, 1.9, 0.8), 0.3, 60.0, 0), ((1.8, 0.6, 1.5), 0.1, 20.0, 0)])
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(sh, [64, 48])
        pt.RenderPointShadows()
        still = [pt.ReadPointShadow(i) for i in range(2)]
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(2, 1)
        pt.TlasBuild()
        pt.RenderPointShadows()
        for i, n in enumerate((64, 48)):
            got = pt.ReadPointShadow(i)
            assert np.array_equal(got, pso.point_shadow_render(expect, sh[i], n)), i
        assert any(not np.array_equal(pt.ReadPointShadow(i), still[i]) for i in range(2))


@pytest.mark.gpu
def test_gpu_render_between_async_computes_leaves_image_unchanged():
    scene, cam = scenes.cornell_1k(threads=1)
    w, h = 160, 120
    frame = scenes.camera_frame(cam, w, h)
    sh = scenes.point_shadows([((0.0, 1.6, 0.3), 0.2, 60.0, 0)])

    def run(with_render):
        with PathTracer(w, h, lanes=4) as pt:
            pt.SetScene(scene)
            pt.SetSky((0.6, 0.7, 0.9))
            pt.SetFrame(frame)
            pt.SetPointShadows(sh, [256])
            for k in range(6):
                pt.ComputeAsync()
                if with_render and k in (1, 3):
                    pt.RenderPointShadows()
            pt.Sync()
            return pt.Result.copy(), pt.ReadPointShadow(0)

    img0, map0 = run(False)
    img1, map1 = run(True)
    assert np.array_equal(img0.view(np.uint32), img1.view(np.uint32))
    assert np.all(map0 == 65535) and np.array_equal(map1, pso.point_shadow_render(scene, sh[0], 256))
