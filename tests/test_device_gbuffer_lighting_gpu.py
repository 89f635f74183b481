"""The ray-traced shadows, the cone trace and the volumetric light on an IdkPtGBuffer: the device G-buffer of idkpt_gbuffer read
in place, the same G-buffer downloaded and passed as host arrays, the host-array entry points and the oracle all give the same
bits (NaN as NaN); a whole raster frame kept on the device equals the same frame through the host; rejected calls leave the
device images as they were."""
import copy
import functools

import numpy as np
import pytest

import oracle_lib as ol
import volumetric_oracle as vo
from idkengine_b200 import capi, multigpu, scenes, vxgi
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import CORNELL_LIGHTS, GRID_MAX, GRID_MIN, JITTER, assert_bits, deferred_setup

INVALID = r"failed \(-1\)"                  # IDKPT_ERR_INVALID_ARGUMENT
SIZES = [(1, 1), (7, 5), (37, 19), (256, 144)]
RUNS = [("cornell", s) for s in SIZES] + [(w, s) for w in ("multi_blas_tlas", "atrium") for s in ((37, 19), (256, 144))]
NOISE = (0, 7)
SAMPLES = 2


def tensor(ptr, shape, typestr="<f4"):
    """A zero-copy CUDA tensor over a library image."""
    import torch
    return torch.as_tensor(multigpu.DeviceArray(ptr, shape, typestr), device="cuda")


def volumetric_settings(scale=0.6):
    st = capi.default_volumetric_settings()
    st.Absorbance[:] = [0.025, 0.04, 0.06]
    st.ResolutionScale = scale
    return st


def grid_bounds(scene):
    """A VXGI grid around the scene: the Cornell box's, or the positions' bounds with a margin."""
    p = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1)
    return tuple(p.min(0) - 0.1), tuple(p.max(0) + 0.1)


@functools.lru_cache(maxsize=None)
def voxel_scene(which):
    """(scene with every light unshadowed, grid min, grid max): what the voxeliser lights."""
    scene, _, _ = deferred_setup(which)
    unshadowed = copy.deepcopy(scene)
    unshadowed.lights["PointShadowIndex"][:] = -1
    lo, hi = (GRID_MIN, GRID_MAX) if which == "cornell" else grid_bounds(scene)
    return unshadowed, lo, hi


def gpu_chain(vx):
    """The voxeliser's grid as the raw uint16 mip chain the oracle's cone trace reads."""
    return np.concatenate([vx.ReadLevel(l).reshape(-1).view(np.uint16) for l in range(len(vx.sizes))])


@pytest.mark.gpu
@pytest.mark.parametrize("which, size", RUNS)
def test_gpu_shadows_device_host_and_oracle_agree(which, size):
    scene, cam, _ = deferred_setup(which)
    W, H = size
    frame = scenes.camera_frame(cam, W, H)
    lights = [int(i) for i in np.nonzero(scene.lights["PointShadowIndex"] >= 0)[0]]
    prev = np.zeros((H, W), np.float32)         # what slots 0..2 hold: a new image is 0, then sky pixels keep their values
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        for jitter in (None, JITTER):          # the jittered G-buffer has other sky pixels: they keep the first one's values
            host = pt.GBuffer(frame, W, H, jitter)
            dev = pt.GBufferDevicePtrs()
            for li in lights:
                for noise in NOISE:
                    kw = dict(samples=SAMPLES, noise_index=noise, jitter=jitter)
                    got = pt.ShadowsRayTracedGBuffer(frame, dev, li, 0, **kw)
                    assert_bits(got, pt.ShadowsRayTracedGBuffer(frame, host[:2], li, 1, **kw))
                    assert_bits(got, pt.ShadowsRayTraced(frame, host[0], host[1], li, visibility=prev.copy(), **kw)[0])
                    assert_bits(got, ol.shadows_ray_traced(scene, frame, host[0], host[1], li, SAMPLES, noise, jitter or (0.0, 0.0), prev))
                    prev = got
                    assert pt.ShadowsRayTracedGBuffer(frame, dev, li, 2, download=False, **kw) is None
                    p, nbytes = pt.ShadowsDevicePtr(2)
                    assert nbytes == W * H * 4
                    assert_bits(tensor(p, (H, W)).cpu().numpy(), got)
    if W * H > 1 and which == "cornell":
        assert (got > 0).any() and (host[0] == 1.0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("which, size", RUNS)
def test_gpu_cone_trace_device_host_and_oracle_agree(which, size):
    scene, cam, _ = deferred_setup(which)
    voxels, lo, hi = voxel_scene(which)
    W, H = size
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(32, lo, hi) as vx:
        pt.SetScene(scene)
        vx.SetScene(voxels)
        vx.Render()
        raw = gpu_chain(vx)
        for jitter in (None, JITTER):
            host = pt.GBuffer(frame, W, H, jitter)
            dev = pt.GBufferDevicePtrs()
            for noise in NOISE:
                st = vxgi.default_cone_settings()
                st.NoiseIndex = noise
                got, stats = vx.ConeTraceGBuffer(frame, dev, st)
                host_gb, host_stats = vx.ConeTraceGBuffer(frame, (host[0], host[1], None, host[3]), st)
                assert_bits(got, host_gb)
                old, old_stats = vx.ConeTrace(frame, host[0], host[1], host[3], st)
                assert_bits(got, old)
                want, steps = ol.vx_cone_trace(vx.ci, raw, frame, st, host[0], host[1], host[3])
                assert_bits(got, want)
                assert stats.ConeSteps == host_stats.ConeSteps == old_stats.ConeSteps == steps
                assert vx.ConeTraceGBuffer(frame, dev, st, download=False)[0] is None
                p, nbytes = vx.ConeTraceDevicePtr()
                assert nbytes == W * H * 16 and p % 16 == 0
                assert_bits(tensor(p, (H, W, 4)).cpu().numpy(), got)


@pytest.mark.gpu
@pytest.mark.parametrize("which, size", RUNS)
def test_gpu_volumetric_device_host_and_oracle_agree(which, size):
    scene, cam, shadows = deferred_setup(which)
    W, H = size
    frame = scenes.camera_frame(cam, W, H)
    st = volumetric_settings(0.6 if min(W, H) > 1 else 1.0)          # a 1x1 output at scale 0.6 renders nothing
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [40, 24])
        pt.RenderPointShadows()
        maps = [pt.ReadPointShadow(i) for i in range(len(shadows))]
        for jitter in (None, JITTER):
            host = pt.GBuffer(frame, W, H, jitter)
            dev = pt.GBufferDevicePtrs()
            for ow, oh in ((W, H), (2 * W + 1, H + 3)):             # the output at the depth's size and at another one
                got = pt.VolumetricLightingGBuffer(frame, dev, ow, oh, st, jitter)
                assert got.shape == (oh, ow, 4)
                assert_bits(got, pt.VolumetricLightingGBuffer(frame, (host[0],), ow, oh, st, jitter))
                assert_bits(got, pt.VolumetricLighting(frame, host[0], ow, oh, st, jitter))
                assert_bits(got, vo.volumetric_lighting(scene.lights, frame, st, shadows, maps, host[0], ow, oh, jitter)[0])
                assert pt.VolumetricLightingGBuffer(frame, dev, ow, oh, st, jitter, download=False) is None
                p, nbytes = pt.VolumetricDevicePtr()
                assert nbytes == ow * oh * 8
                assert_bits(tensor(p, (oh, ow, 4), "<f2").cpu().numpy(), got)


# ------------------------------------------------------------------------------------------------ the whole frame
def three_shadowed():
    """The Cornell box with its three lights, each with a point shadow (shadow k belongs to light k)."""
    scene, cam = scenes.cornell_1k(threads=1)
    for light in CORNELL_LIGHTS:
        scene.add_light(*light)
    scene.lights["PointShadowIndex"][:] = [0, 1, 2]
    return scene, cam, scenes.point_shadows([(scene.lights[k]["Position"], 0.1, 60.0, k) for k in range(3)])


def open_tracer(scene, shadows):
    pt = PathTracer(16, 16)
    pt.SetScene(scene)
    pt.SetPointShadows(shadows, [48, 32, 40])
    pt.RenderPointShadows()
    return pt


RT_VXGI = capi.IdkPtDeferredSettings(capi.SHADOW_MODE_RAY_TRACED, 1, 1, 0)


def device_frame(pt, vx, frame, W, H, cone):
    """The frame with every image on the device: G-buffer, visibility and indirect light through the new entry points."""
    pt.GBuffer(frame, W, H, JITTER, download=False)
    g = pt.GBufferDevicePtrs()
    for k in range(3):
        assert pt.ShadowsRayTracedGBuffer(frame, g, k, k, samples=SAMPLES, noise_index=4, jitter=JITTER, download=False) is None
    assert vx.ConeTraceGBuffer(frame, g, cone, download=False)[0] is None
    t = pt.GBufferDevicePtrs(tensors=True)
    indirect = tensor(vx.ConeTraceDevicePtr()[0], (H, W, 4))
    rt = [tensor(pt.ShadowsDevicePtr(k)[0], (H, W)) for k in range(3)]
    pt.Ssao(frame, t[0], t[1], download=False)
    pt.DeferredLighting(frame, *t[:5], settings=RT_VXGI, jitter=JITTER, indirect=indirect, rt_visibility=rt, download=False)
    pt.LightsAndSkybox(frame, JITTER, download=False)
    t = pt.GBufferDevicePtrs(tensors=True)
    pt.Transparency(frame, t[0], jitter=JITTER, source=capi.LIT_SOURCE_DEFERRED, voxelizer=vx, download=False)
    pt.Ssr(frame, t[0], t[1], t[2], t[3], source=capi.LIT_SOURCE_DEFERRED, download=False)
    taa = pt.TaaResolve(t[0], t[5], W, H, source=capi.LIT_SOURCE_MERGED)
    return taa, pt.VolumetricLightingGBuffer(frame, g, W, H, volumetric_settings(), JITTER)


def host_frame(pt, vx, frame, W, H, cone):
    """The same frame through host arrays and the host-array entry points."""
    g = pt.GBuffer(frame, W, H, JITTER)
    rt = [pt.ShadowsRayTraced(frame, g[0], g[1], k, samples=SAMPLES, noise_index=4, jitter=JITTER)[0] for k in range(3)]
    indirect = vx.ConeTrace(frame, g[0], g[1], g[3], cone)[0]
    pt.Ssao(frame, g[0], g[1], download=False)
    pt.DeferredLighting(frame, *g[:5], settings=RT_VXGI, jitter=JITTER, indirect=indirect, rt_visibility=rt, download=False)
    pt.LightsAndSkybox(frame, JITTER, download=False)
    g = [t.cpu().numpy() for t in pt.GBufferDevicePtrs(tensors=True)]
    pt.Transparency(frame, g[0], jitter=JITTER, source=capi.LIT_SOURCE_DEFERRED, voxelizer=vx, download=False)
    pt.Ssr(frame, g[0], g[1], g[2], g[3], source=capi.LIT_SOURCE_DEFERRED, download=False)
    taa = pt.TaaResolve(g[0], g[5], W, H, source=capi.LIT_SOURCE_MERGED)
    return taa, pt.VolumetricLighting(frame, g[0], W, H, volumetric_settings(), JITTER)


@pytest.mark.gpu
def test_gpu_whole_frame_on_the_device_equals_the_host_frame():
    scene, cam, shadows = three_shadowed()
    W, H = 96, 64
    frame = scenes.camera_frame(cam, W, H)
    cone = vxgi.default_cone_settings()
    cone.NoiseIndex = 3
    dev_pt, host_pt = open_tracer(scene, shadows), open_tracer(scene, shadows)
    try:
        with vxgi.Voxelizer(32, GRID_MIN, GRID_MAX) as vx:
            vx.SetScene(scene)
            vx.SetShadowMaps(dev_pt)
            vx.Render()
            got = [device_frame(dev_pt, vx, frame, W, H, cone) for _ in range(2)]      # two frames: the TAA history too
            want = [host_frame(host_pt, vx, frame, W, H, cone) for _ in range(2)]
    finally:
        dev_pt.Dispose()
        host_pt.Dispose()
    for (taa, vol), (taa_h, vol_h) in zip(got, want):
        assert_bits(taa, taa_h)
        assert_bits(vol, vol_h)
    assert np.isfinite(got[1][0]).all() and (got[1][0][..., :3] > 0).any() and (got[1][1][..., :3] > 0).any()


# ------------------------------------------------------------------------------------------------ rejections and the shims
def images(pt, vx, W, H):
    """The bytes of the shadow image of slot 0, the cone-trace image and the volumetric image, with their pointers."""
    out = []
    for p, n in (pt.ShadowsDevicePtr(0), vx.ConeTraceDevicePtr(), pt.VolumetricDevicePtr()):
        out.append((p, n, tensor(p, (n // 4,)).cpu().numpy().view(np.uint32).copy()))
    return out


@pytest.mark.gpu
def test_gpu_rejected_calls_leave_the_device_images_as_they_were():
    scene, cam, shadows = deferred_setup("cornell")
    voxels, lo, hi = voxel_scene("cornell")
    W, H = 40, 24
    frame = scenes.camera_frame(cam, W, H)
    st = volumetric_settings()
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(32, lo, hi) as vx:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [40, 24])
        pt.RenderPointShadows()
        vx.SetScene(voxels)
        vx.Render()
        host = pt.GBuffer(frame, W, H, JITTER)
        g, _ = pt.GBufferDevicePtrs()
        with pytest.raises(IdkPtError, match="call idkpt_shadows_ray_traced_gbuffer for the slot first"):
            pt.ShadowsDevicePtr(0)
        with pytest.raises(vxgi.IdkVxError, match="call idkvx_cone_trace_gbuffer first"):
            vx.ConeTraceDevicePtr()
        pt.ShadowsRayTracedGBuffer(frame, g, 0, 0, samples=SAMPLES, jitter=JITTER, download=False)
        vx.ConeTraceGBuffer(frame, g, download=False)
        pt.VolumetricLightingGBuffer(frame, g, W, H, st, JITTER, download=False)
        before = images(pt, vx, W, H)

        def variant(**kw):
            v = capi.IdkPtGBuffer.from_buffer_copy(g)
            for k, val in kw.items():
                setattr(v, k, val)
            return v
        hostp = host[0].ctypes.data
        bad = [variant(Depth=hostp),                                         # a host pointer with OnDevice = 1
               variant(Depth=g.Depth + 2), variant(NormalRG=g.NormalRG + 4),     # misaligned
               variant(OnDevice=2),
               variant(Width=0), variant(Height=16385), variant(Width=-3)]
        for v in bad:                                                        # download=False: no host image of a bad size
            with pytest.raises(IdkPtError, match=INVALID):
                pt.ShadowsRayTracedGBuffer(frame, v, 0, 0, samples=SAMPLES, download=False)
            with pytest.raises(vxgi.IdkVxError, match=INVALID):
                vx.ConeTraceGBuffer(frame, v, download=False)
            if v.NormalRG == g.NormalRG:                                     # the volumetric pass reads Depth only
                with pytest.raises(IdkPtError, match=INVALID):
                    pt.VolumetricLightingGBuffer(frame, v, W, H, st)
        with pytest.raises(vxgi.IdkVxError, match=INVALID):
            vx.ConeTraceGBuffer(frame, variant(MetallicRoughness=g.MetallicRoughness + 4))
        with pytest.raises(vxgi.IdkVxError, match=INVALID):
            vx.ConeTraceGBuffer(frame, variant(MetallicRoughness=None))
        for slot in (-1, capi.IDKPT_MAX_POINT_SHADOWS):
            with pytest.raises(IdkPtError, match=INVALID):
                pt.ShadowsRayTracedGBuffer(frame, g, 0, slot)
            with pytest.raises(IdkPtError, match=INVALID):
                pt.ShadowsDevicePtr(slot)
        for kw in (dict(light_index=len(scene.lights)), dict(samples=0), dict(samples=1025)):
            args = dict(light_index=0, samples=SAMPLES) | kw
            with pytest.raises(IdkPtError, match=INVALID):
                pt.ShadowsRayTracedGBuffer(frame, g, args["light_index"], 0, samples=args["samples"])
        for ow, oh, s in ((0, H, st), (W, 16385, st), (W, H, volumetric_settings(0.01))):
            with pytest.raises(IdkPtError, match=INVALID):
                pt.VolumetricLightingGBuffer(frame, g, ow, oh, s)
        cone = vxgi.default_cone_settings()
        cone.MaxSamples = 65
        with pytest.raises(vxgi.IdkVxError, match=INVALID):
            vx.ConeTraceGBuffer(frame, g, cone)
        after = images(pt, vx, W, H)
        for (p0, n0, b0), (p1, n1, b1) in zip(before, after):
            assert p0 == p1 and n0 == n1 and np.array_equal(b0, b1)
        # and the context still works
        assert_bits(pt.ShadowsRayTracedGBuffer(frame, g, 0, 0, samples=SAMPLES, jitter=JITTER),
                    ol.shadows_ray_traced(scene, frame, host[0], host[1], 0, SAMPLES, 0, JITTER))


@pytest.mark.gpu
def test_gpu_host_array_shims_keep_their_behaviour():
    """idkpt_shadows_ray_traced leaves the caller's depth == 1 pixels as they were and touches no slot image;
    idkvx_cone_trace_rows equals the full-frame trace on its rows."""
    scene, cam, _ = deferred_setup("cornell")
    voxels, lo, hi = voxel_scene("cornell")
    W, H = 37, 19
    frame = scenes.camera_frame(cam, W, H)
    rng = np.random.default_rng(5)
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(32, lo, hi) as vx:
        pt.SetScene(scene)
        host = pt.GBuffer(frame, W, H, JITTER)
        g, _ = pt.GBufferDevicePtrs()
        sky = host[0] == 1.0
        assert sky.any() and (~sky).any()
        slot0 = pt.ShadowsRayTracedGBuffer(frame, g, 0, 0, samples=SAMPLES, jitter=JITTER)
        seed = (rng.random((H, W)) * 3.0 - 1.0).astype(np.float32)
        seed[0, :4] = np.nan
        vis, _ = pt.ShadowsRayTraced(frame, host[0], host[1], 0, samples=SAMPLES, jitter=JITTER, visibility=seed)
        assert_bits(vis[sky], seed[sky])
        assert_bits(vis, ol.shadows_ray_traced(scene, frame, host[0], host[1], 0, SAMPLES, 0, JITTER, visibility=seed))
        assert_bits(tensor(pt.ShadowsDevicePtr(0)[0], (H, W)).cpu().numpy(), slot0)
        vx.SetScene(voxels)
        vx.Render()
        full, _ = vx.ConeTraceGBuffer(frame, g)
        for r0, r1 in ((0, 1), (3, 11), (11, H)):
            rows, _ = vx.ConeTraceRows(frame, host[0][r0:r1], host[1][r0:r1], host[3][r0:r1], H, r0)
            assert_bits(rows, full[r0:r1])
            p, nbytes = vx.ConeTraceDevicePtr()                              # the rows variant's image is the device image now
            assert nbytes == W * (r1 - r0) * 16
            assert_bits(tensor(p, (r1 - r0, W, 4)).cpu().numpy(), rows)
