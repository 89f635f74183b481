"""Transparency (k_transparency) on the GPU, bit for bit against the oracle, in the device chain, and its errors and lifetime.

float32 images are compared as bytes with every NaN canonicalised (the device and x86 produce different NaN payloads)."""
import copy
import ctypes
import functools

import numpy as np
import pytest

import gbuffer_oracle as go
import transparency_oracle as to
from idkengine_b200 import capi, scenes, vxgi
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, canon, rule_scene

pytestmark = pytest.mark.gpu

GRID_MIN, GRID_MAX = (-2.0, -1.2, -3.2), (2.0, 3.2, 3.2)
ERR_INVALID_ARGUMENT, ERR_NO_SCENE = -1, -4


@functools.lru_cache(maxsize=None)
def setup(which):
    """(scene, camera, shadows) with a shadowed light, a light without a shadow, and blended surfaces in view."""
    if which == "rule":
        scene, cam = rule_scene()
    elif which == "cornell":
        scene, cam = scenes.cornell_1k(threads=1)
    elif which in ("multi_blas", "multi_blas_tlas"):
        scene, cam = scenes.multi_blas(threads=1)
        if which == "multi_blas_tlas":
            scene.build_tlas()
    elif which == "atrium":
        scene, cam = scenes.atrium(20000, threads=1)
    else:
        scene, cam = scenes.textured_room(threads=1)
    if which != "rule":   # every scene gets blended surfaces: a third of its materials
        scene.materials["AlphaCutoff"][::3] = 2.0
        scene.materials["BaseColorFactor"][::3] = (scene.materials["BaseColorFactor"][::3] & 0x00FFFFFF) | (0x80 << 24)
    scene.add_light((0.2, 1.5, 0.8), (5.0, 4.5, 4.0), 0.2)
    scene.add_light((-0.5, 1.0, 1.0), (1.0, 0.5, 0.3), 0.1)
    n = len(scene.lights)
    scene.lights["PointShadowIndex"][:] = -1
    scene.lights["PointShadowIndex"][n - 2] = 0
    return scene, cam, scenes.point_shadows([(scene.lights[n - 2]["Position"], 0.1, 60.0, n - 2)])


def lit_image(h, w, seed=4):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.random((h, w, 3), dtype=np.float32) * 2.0, np.ones((h, w, 1), np.float32)], -1)


def voxels_of(scene):
    """A voxelised grid of the scene (lights unshadowed) and the oracle's inputs: (Voxelizer, (create info, levels, cone))."""
    unshadowed = copy.deepcopy(scene)
    unshadowed.lights["PointShadowIndex"][:] = -1
    vx = vxgi.Voxelizer(32, GRID_MIN, GRID_MAX)
    vx.SetScene(unshadowed)
    vx.Render()
    levels = np.concatenate([vx.ReadLevel(l).view(np.uint16).ravel() for l in range(len(vx.sizes))])
    cone = vxgi.IdkVxConeSettings(4, 0.16, 1.3, 1.0 / 1.3, 1.0, 5)
    return vx, (vx.ci, levels, cone)


def run(which, w, h, mode, vxgi_on, jitter, source, on_device, sky=(0.6, 0.7, 0.9)):
    scene, cam, shadows = setup(which)
    frame = scenes.camera_frame(cam, w, h)
    vx, vox = voxels_of(scene) if vxgi_on else (None, None)
    try:
        with PathTracer(16, 16) as pt:
            pt.SetScene(scene)
            pt.SetSky(sky)
            pt.SetPointShadows(shadows, [32])
            pt.RenderPointShadows()
            maps = [pt.ReadPointShadow(0)]
            g = pt.GBuffer(frame, w, h, jitter=jitter)
            depth = g[0]
            color = lit_image(h, w)
            st = capi.IdkPtTransparencySettings(mode, int(vxgi_on))
            cone = vox[2] if vox else None
            if source == capi.LIT_SOURCE_DEFERRED:
                color = pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0), jitter=jitter)
                got = pt.Transparency(frame, depth, settings=st, jitter=jitter, source=capi.LIT_SOURCE_DEFERRED, voxelizer=vx, cone=cone)
            elif on_device:
                import torch
                dd = torch.from_numpy(depth).cuda()
                cd = torch.from_numpy(color.copy()).cuda()
                out = pt.Transparency(frame, dd, settings=st, jitter=jitter, color=cd, voxelizer=vx, cone=cone)
                got = cd.cpu().numpy()
                assert np.array_equal(canon(out), canon(got))
            else:
                arr = color.copy()
                out = pt.Transparency(frame, depth, settings=st, jitter=jitter, color=arr, voxelizer=vx, cone=cone)
                got = arr
                assert np.array_equal(canon(out), canon(got))
            assert pt.last_transparency_ms > 0
    finally:
        if vx is not None:
            vx.__exit__(None, None, None)
    want, layers, counts = to.transparency(scene, frame, depth, color, shadow_mode=mode, shadows=shadows, maps=maps, jitter=jitter,
                                           sky=capi.sky_desc(sky), voxels=vox)
    bad = canon(got) != canon(want)
    assert not bad.any(), f"{int(bad.sum())} values differ"
    return got, color, counts


@pytest.mark.parametrize("which", ["rule", "cornell", "multi_blas", "multi_blas_tlas", "atrium", "textured_room"])
@pytest.mark.parametrize("size", [(96, 64), (37, 23), (8, 8), (1, 1)])
def test_transparency_matches_oracle(which, size):
    w, h = size
    got, color, counts = run(which, w, h, 1, False, JITTER, capi.LIT_SOURCE_ARRAY, False)
    if size == (96, 64):
        assert counts.any()
    keep = counts == 0
    assert np.array_equal(got[keep].view(np.uint32), color[keep].view(np.uint32))


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("vxgi_on", [False, True])
@pytest.mark.parametrize("jitter", [None, JITTER])
def test_every_mode_matches_oracle(mode, vxgi_on, jitter):
    run("rule", 48, 32, mode, vxgi_on, jitter, capi.LIT_SOURCE_ARRAY, False)


@pytest.mark.parametrize("which", ["rule", "cornell"])
@pytest.mark.parametrize("source, on_device", [(capi.LIT_SOURCE_ARRAY, True), (capi.LIT_SOURCE_DEFERRED, False)])
def test_sources_match_oracle(which, source, on_device):
    run(which, 40, 24, 1, False, JITTER, source, on_device)


def test_device_chain_equals_array_chain():
    """G-buffer -> deferred lighting -> transparency (DEFERRED) -> SSR -> TAA on the device gives the bytes of the same chain fed
    with downloaded arrays (ARRAY)."""
    scene, cam, shadows = setup("rule")
    w, h = 48, 32
    frame = scenes.camera_frame(cam, w, h)
    st = capi.IdkPtTransparencySettings(1, 0)
    ds = capi.IdkPtDeferredSettings(1, 0, 0, 0)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [32])
        pt.RenderPointShadows()
        g = pt.GBuffer(frame, w, h, jitter=JITTER)
        lit = pt.DeferredLighting(frame, *g[:5], settings=ds, jitter=JITTER)
        arr = lit.copy()
        pt.Transparency(frame, g[0], settings=st, jitter=JITTER, color=arr)
        m_arr = pt.Ssr(frame, g[0], g[1], g[2], g[3], color=arr)[0]
        t_arr = pt.TaaResolve(g[0], g[5], w, h, color=m_arr)

    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [32])
        pt.RenderPointShadows()
        pt.GBuffer(frame, w, h, jitter=JITTER, download=False)
        gt_ = pt.GBufferDevicePtrs(tensors=True)
        pt.DeferredLighting(frame, *gt_[:5], settings=ds, jitter=JITTER, download=False)
        dev = pt.Transparency(frame, gt_[0], settings=st, jitter=JITTER, source=capi.LIT_SOURCE_DEFERRED)
        m_dev = pt.Ssr(frame, *gt_[:4], source=capi.LIT_SOURCE_DEFERRED)[0]
        t_dev = pt.TaaResolve(gt_[0], gt_[5], w, h, source=capi.LIT_SOURCE_MERGED)
    assert np.array_equal(canon(dev), canon(arr))
    assert np.array_equal(canon(m_dev), canon(m_arr))
    assert np.array_equal(np.asarray(t_dev).view(np.uint16), np.asarray(t_arr).view(np.uint16))


def test_scene_without_blended_meshes_leaves_the_image():
    scene, cam = scenes.cornell_1k(threads=1)
    scene.materials["AlphaCutoff"][scene.materials["AlphaCutoff"] == 2.0] = 0.0                 # the card becomes opaque
    w, h = 40, 24
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        g = pt.GBuffer(frame, w, h)
        lit = pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0))
        out = pt.Transparency(frame, g[0], settings=capi.IdkPtTransparencySettings(0, 0), source=capi.LIT_SOURCE_DEFERRED)
    assert np.array_equal(out.view(np.uint32), lit.view(np.uint32))


def test_errors_leave_the_target_unchanged():
    scene, cam, shadows = setup("rule")
    w, h = 24, 16
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(16, 16) as pt:
        with pytest.raises(IdkPtError):                                                     # no scene
            pt.Transparency(frame, np.ones((h, w), np.float32), color=lit_image(h, w))
        pt.SetScene(scene)
        g = pt.GBuffer(frame, w, h)
        lit = pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0))
        arr = lit_image(h, w)
        before = arr.copy()
        bad = [dict(settings=capi.IdkPtTransparencySettings(3, 0)), dict(settings=capi.IdkPtTransparencySettings(-1, 0)),
               dict(settings=capi.IdkPtTransparencySettings(0, 2)), dict(settings=capi.IdkPtTransparencySettings(0, 1)),
               dict(settings=capi.IdkPtTransparencySettings(1, 0)),                        # Pcf: shadow index 0 without shadows
               dict(jitter=(np.nan, 0.0)), dict(jitter=(0.0, np.inf))]
        for kw in bad:
            with pytest.raises(IdkPtError):
                pt.Transparency(frame, g[0], color=arr, **kw)
            assert np.array_equal(arr.view(np.uint32), before.view(np.uint32))
        for kw in bad[:4] + bad[5:]:
            with pytest.raises(IdkPtError):
                pt.Transparency(frame, g[0], source=capi.LIT_SOURCE_DEFERRED, **kw)
        with pytest.raises(IdkPtError):                                                     # MERGED is rejected
            pt.Transparency(frame, g[0], source=capi.LIT_SOURCE_MERGED)
        with pytest.raises(IdkPtError):                                                     # DEFERRED of another size
            pt.Transparency(frame, np.ones((h + 1, w), np.float32), source=capi.LIT_SOURCE_DEFERRED)
        assert np.array_equal(pt.Transparency(frame, np.zeros((h, w), np.float32), settings=capi.IdkPtTransparencySettings(0, 0),
                                              source=capi.LIT_SOURCE_DEFERRED).view(np.uint32), lit.view(np.uint32))
        with vxgi.Voxelizer(16, GRID_MIN, GRID_MAX) as vx:                                  # never voxelised
            with pytest.raises(IdkPtError):
                pt.Transparency(frame, g[0], color=arr, settings=capi.IdkPtTransparencySettings(0, 1), voxelizer=vx)
            unshadowed = copy.deepcopy(scene)
            unshadowed.lights["PointShadowIndex"][:] = -1
            vx.SetScene(unshadowed)
            vx.Render()
            with pytest.raises(IdkPtError):                                                 # cone MaxSamples out of range
                pt.Transparency(frame, g[0], color=arr, settings=capi.IdkPtTransparencySettings(0, 1), voxelizer=vx,
                                cone=vxgi.IdkVxConeSettings(0, 0.16, 1.3, 1.0, 1.0, 0))
        assert np.array_equal(arr.view(np.uint32), before.view(np.uint32))


def test_lifetime_set_scene_sizes_and_async_compute():
    scene, cam, shadows = setup("rule")
    with PathTracer(32, 24) as pt:
        pt.SetScene(scene)
        for w, h in [(32, 24), (17, 9), (32, 24)]:
            frame = scenes.camera_frame(cam, w, h)
            g = pt.GBuffer(frame, w, h)
            color = lit_image(h, w)
            pt.SetFrame(scenes.camera_frame(cam, 32, 24))
            pt.ComputeAsync()                                                               # queued, not waited for
            arr = color.copy()
            pt.Transparency(frame, g[0], settings=capi.IdkPtTransparencySettings(0, 0), color=arr)
            want = to.transparency(scene, frame, g[0], color)[0]
            assert np.array_equal(canon(arr), canon(want))
        pt.SetScene(scene)
        with pytest.raises(IdkPtError):                                                     # set_scene dropped the deferred image
            pt.Transparency(frame, g[0], source=capi.LIT_SOURCE_DEFERRED)


def test_null_and_pointer_errors_leave_the_target_unchanged():
    """Null arguments through the C entry point, device-array pointer checks (a host pointer with OnDevice = 1, a misaligned
    colour or depth), each against the DEFERRED image and the caller's array, compared byte for byte after every call."""
    import torch
    scene, cam, shadows = setup("rule")
    w, h = 24, 16
    frame = np.ascontiguousarray(scenes.camera_frame(cam, w, h))
    st = capi.IdkPtTransparencySettings(0, 0)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        g = pt.GBuffer(frame, w, h)
        pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0))
        p, nbytes = pt.DeferredDevicePtr()
        from idkengine_b200.multigpu import DeviceArray
        deferred = torch.as_tensor(DeviceArray(p, (h, w, 4)), device=torch.device("cuda", 0))

        def snapshot():
            torch.cuda.synchronize()
            return deferred.cpu().numpy().view(np.uint32).copy()
        ref = snapshot()
        depth = np.ascontiguousarray(g[0])
        arr = lit_image(h, w)
        arr_before = arr.copy()
        L, ctx = pt._lib, pt._ctx
        gh = capi.IdkPtGBuffer(w, h, 0, depth.ctypes.data, None, None, None, None)
        gh_nodepth = capi.IdkPtGBuffer(w, h, 0, None, None, None, None, None)
        fr = frame.ctypes.data
        calls = [(None, fr, st, gh, capi.LIT_SOURCE_DEFERRED, None), (ctx, None, st, gh, capi.LIT_SOURCE_DEFERRED, None),
                 (ctx, fr, None, gh, capi.LIT_SOURCE_DEFERRED, None), (ctx, fr, st, None, capi.LIT_SOURCE_DEFERRED, None),
                 (ctx, fr, st, gh_nodepth, capi.LIT_SOURCE_DEFERRED, None), (ctx, fr, st, gh, capi.LIT_SOURCE_ARRAY, None),
                 (ctx, fr, st, capi.IdkPtGBuffer(w, h, 2, depth.ctypes.data, None, None, None, None), capi.LIT_SOURCE_DEFERRED, None),
                 (ctx, fr, st, capi.IdkPtGBuffer(0, h, 0, depth.ctypes.data, None, None, None, None), capi.LIT_SOURCE_DEFERRED, None),
                 (ctx, fr, st, capi.IdkPtGBuffer(w, 16385, 0, depth.ctypes.data, None, None, None, None), capi.LIT_SOURCE_DEFERRED, None)]
        dd = torch.from_numpy(depth).cuda()
        cd = torch.from_numpy(arr.copy()).cuda()
        big = torch.zeros(h * w * 4 + 4, dtype=torch.float32, device="cuda")
        calls += [(ctx, fr, st, capi.IdkPtGBuffer(w, h, 1, depth.ctypes.data, None, None, None, None), capi.LIT_SOURCE_DEFERRED, None),
                  (ctx, fr, st, capi.IdkPtGBuffer(w, h, 1, dd.data_ptr() + 2, None, None, None, None), capi.LIT_SOURCE_DEFERRED, None),
                  (ctx, fr, st, capi.IdkPtGBuffer(w, h, 1, dd.data_ptr(), None, None, None, None), capi.LIT_SOURCE_ARRAY, arr.ctypes.data),
                  (ctx, fr, st, capi.IdkPtGBuffer(w, h, 1, dd.data_ptr(), None, None, None, None), capi.LIT_SOURCE_ARRAY, big.data_ptr() + 4)]
        for c, f_, s_, g_, src, col in calls:
            rc = L.idkpt_transparency(c, f_, ctypes.byref(s_) if s_ is not None else None, ctypes.byref(g_) if g_ is not None else None,
                                      None, None, None, src, col, None, None)
            assert rc == ERR_INVALID_ARGUMENT, rc
            assert np.array_equal(snapshot(), ref)
            assert np.array_equal(arr.view(np.uint32), arr_before.view(np.uint32))
        torch.cuda.synchronize()
        assert not big.any()
        assert np.array_equal(cd.cpu().numpy().view(np.uint32), arr_before.view(np.uint32))


def test_voxels_must_hold_a_whole_current_voxelisation():
    """IsVXGI needs a grid voxelised whole: a slab voxelisation is refused until idkvx_mipmap completes it, and a new grid, scene
    or slab refuses it again."""
    scene, cam, shadows = setup("rule")
    w, h = 16, 12
    frame = scenes.camera_frame(cam, w, h)
    unshadowed = copy.deepcopy(scene)
    unshadowed.lights["PointShadowIndex"][:] = -1
    st = capi.IdkPtTransparencySettings(0, 1)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(16, GRID_MIN, GRID_MAX) as vx:
        pt.SetScene(scene)
        g = pt.GBuffer(frame, w, h)
        arr = lit_image(h, w)

        def call():
            pt.Transparency(frame, g[0], settings=st, color=arr.copy(), voxelizer=vx)
        vx.SetScene(unshadowed)
        vx.SetSlab(0, 8)
        vx.Render()
        with pytest.raises(IdkPtError):
            call()
        vx.Mipmap()
        call()
        vx.SetSlab(0, 16)
        with pytest.raises(IdkPtError):
            call()
        vx.Render()
        call()
        vx.SetScene(unshadowed)
        with pytest.raises(IdkPtError):
            call()
        vx.Render()
        call()
        f3 = ctypes.c_float * 3
        vx._check(vx._lib.idkvx_set_grid(vx._ctx, f3(*GRID_MIN), f3(*GRID_MAX)), "idkvx_set_grid")
        with pytest.raises(IdkPtError):
            call()
