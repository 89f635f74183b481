"""SSAO (k_ssao) and deferred lighting (k_deferred_lighting) on the GPU, bit for bit against the oracle.

float32 images are compared as bytes with every NaN canonicalised (the device and x86 produce different NaN payloads)."""
import ctypes

import numpy as np
import pytest

import deferred_oracle as do
from idkengine_b200 import capi, multigpu, scenes
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, canon, cone_trace_gi, deferred_settings, deferred_setup, gbuffer, rt_images


def ssao_settings(samples=10, radius=0.2, noise=0, strength=1.3):
    return capi.IdkPtSsaoSettings(samples, radius, strength, noise)


SSAO_CASES = {   # name: (W, H, SampleCount, Radius, NoiseIndex)
    "37x23_s10": (37, 23, 10, 0.2, 0),
    "37x23_s1_noise": (37, 23, 1, 0.2, 37),
    "37x23_s64_r05": (37, 23, 64, 0.5, 90),
    "8x8_s10_r05_noise": (8, 8, 10, 0.5, 3),
    "1x1_s64": (1, 1, 64, 0.2, 0),
}
SSAO_RUNS = [("cornell", c) for c in SSAO_CASES] + [(w, c) for w in ("multi_blas_tlas", "atrium") for c in ("37x23_s10", "37x23_s64_r05")]


@pytest.mark.gpu
@pytest.mark.parametrize("which, case", SSAO_RUNS)
def test_gpu_ssao_matches_oracle(which, case):
    scene, cam, _ = deferred_setup(which)
    W, H, samples, radius, noise = SSAO_CASES[case]
    st = ssao_settings(samples, radius, noise)
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        g = gbuffer(pt, scene, frame, W, H)
        got = pt.Ssao(frame, g[0], g[1], st)
    want = do.ssao(frame, st, g[0], g[1])
    assert got.dtype == np.uint8 and got.shape == (H, W)
    assert np.array_equal(got, want)
    if W * H > 1:
        assert got.any()


def run_deferred(pt, scene, frame, shadows, maps, g, st, jitter=JITTER, ssao=None, indirect=None, rt=None):
    got = pt.DeferredLighting(frame, *g, settings=st, jitter=jitter, indirect=indirect if st.IsVXGI else None,
                              rt_visibility=rt if st.ShadowMode == 2 else None)
    want = do.deferred_lighting(scene.lights, frame, st.ShadowMode, shadows, maps, g, jitter, ssao if st.IsSSAO else None,
                                indirect if st.IsVXGI else None, rt if st.ShadowMode == 2 else None)
    assert got.shape == want.shape
    assert np.array_equal(canon(got), canon(want))
    return got


@pytest.mark.gpu
def test_gpu_deferred_every_mode_matches_oracle():
    """Every ShadowMode x IsSSAO x IsVXGI on the Cornell box: RT visibility from idkpt_shadows_ray_traced, GI from the cone trace."""
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 37, 23
    frame = scenes.camera_frame(cam, W, H)
    gi = cone_trace_gi(W, H)
    results = {}
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [64, 33])
        pt.RenderPointShadows()
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        g = gbuffer(pt, scene, frame, W, H)
        ao = pt.Ssao(frame, g[0], g[1])
        rt = rt_images(pt, scene, frame, g, shadows)
        for mode in (0, 1, 2):
            for is_ssao in (0, 1):
                for is_vxgi in (0, 1):
                    st = deferred_settings(mode, is_ssao, is_vxgi)
                    results[(mode, is_ssao, is_vxgi)] = run_deferred(pt, scene, frame, shadows, maps, g, st, ssao=ao, indirect=gi, rt=rt)
    assert ao.any() and not np.array_equal(results[(1, 0, 0)], results[(0, 0, 0)])
    assert not np.array_equal(results[(2, 0, 0)], results[(0, 0, 0)])
    assert not np.array_equal(results[(0, 1, 0)], results[(0, 0, 0)]) and not np.array_equal(results[(0, 0, 1)], results[(0, 0, 0)])
    r = results[(0, 0, 0)]
    assert np.all(r[0, 0] == [0, 0, 0, 1]) and np.all(r[..., 3] == 1)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cornell", "multi_blas_tlas", "atrium"])
def test_gpu_deferred_maps_cleared_masked_rendered_and_seeded_inputs(which):
    """PCF on maps cleared, partly rendered through face masks and fully rendered; jitter NULL and non-zero; RayTraced from a
    seeded float image (values outside [0, 1] and NaN included); GI from a seeded image."""
    scene, cam, shadows = deferred_setup(which)
    W, H = 40, 24
    frame = scenes.camera_frame(cam, W, H)
    rng = np.random.default_rng(7)
    gi = (rng.random((H, W, 4)) * 2.0).astype(np.float32)
    rt = [(rng.random((H, W)) * 1.4 - 0.2).astype(np.float32) for _ in range(2)]
    rt[1][0, :3] = np.nan
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        g = gbuffer(pt, scene, frame, W, H, seed=3)
        ao = pt.Ssao(frame, g[0], g[1], ssao_settings(16, 0.3, 5))
        pt.SetPointShadows(shadows, [48, 32])
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        assert all(np.all(m == 65535) for m in maps)
        pcf = deferred_settings(1, 1, 1)
        res = [run_deferred(pt, scene, frame, shadows, maps, g, pcf, ssao=ao, indirect=gi)]
        pt.RenderPointShadows(0, 2, [0b010101, 0b101010])
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        res.append(run_deferred(pt, scene, frame, shadows, maps, g, pcf, ssao=ao, indirect=gi))
        pt.RenderPointShadows()
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        res.append(run_deferred(pt, scene, frame, shadows, maps, g, pcf, ssao=ao, indirect=gi))
        res.append(run_deferred(pt, scene, frame, shadows, maps, g, pcf, jitter=None, ssao=ao, indirect=gi))
        run_deferred(pt, scene, frame, shadows, maps, g, deferred_settings(2, 0, 1), jitter=None, indirect=gi, rt=rt)
        run_deferred(pt, scene, frame, shadows, maps, g, deferred_settings(0, 1, 0), ssao=ao)
    assert not np.array_equal(res[0], res[2])


@pytest.mark.gpu
def test_gpu_device_tensor_gbuffer_gives_identical_bytes():
    import torch
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 37, 23
    frame = scenes.camera_frame(cam, W, H)
    gi = cone_trace_gi(W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [40, 24])
        pt.RenderPointShadows()
        g = gbuffer(pt, scene, frame, W, H)
        rt = rt_images(pt, scene, frame, g, shadows)
        dg = [torch.from_numpy(a).cuda() for a in g]
        for st in (ssao_settings(), ssao_settings(64, 0.5, 11)):
            assert np.array_equal(pt.Ssao(frame, g[0], g[1], st), pt.Ssao(frame, dg[0], dg[1], st))
        for mode in (0, 1, 2):
            st = deferred_settings(mode, 1, 1)
            pt.Ssao(frame, g[0], g[1])
            host = pt.DeferredLighting(frame, *g, settings=st, jitter=JITTER, indirect=gi, rt_visibility=rt)
            dev = pt.DeferredLighting(frame, *dg, settings=st, jitter=JITTER, indirect=torch.from_numpy(gi).cuda(),
                                      rt_visibility=[torch.from_numpy(x).cuda() for x in rt])
            assert np.array_equal(canon(host), canon(dev))
        with pytest.raises(TypeError):
            pt.Ssao(frame, dg[0], g[1])


@pytest.mark.gpu
def test_gpu_device_ptrs_match_download():
    import torch
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 53, 31
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [40, 24])
        pt.RenderPointShadows()
        g = gbuffer(pt, scene, frame, W, H)
        with pytest.raises(IdkPtError, match="call idkpt_ssao first"):
            pt.SsaoDevicePtr()
        with pytest.raises(IdkPtError, match="call idkpt_deferred_lighting first"):
            pt.DeferredDevicePtr()
        ao = pt.Ssao(frame, g[0], g[1])
        assert pt.Ssao(frame, g[0], g[1], download=False) is None
        p, nbytes = pt.SsaoDevicePtr()
        assert nbytes == W * H
        dev = torch.as_tensor(multigpu.DeviceArray(p, (nbytes,), "|u1"), device="cuda").cpu().numpy()
        assert np.array_equal(dev.reshape(H, W), ao)
        lit = pt.DeferredLighting(frame, *g, jitter=JITTER)                    # the engine's defaults: PCF, IsSSAO
        assert pt.DeferredLighting(frame, *g, jitter=JITTER, download=False) is None
        p, nbytes = pt.DeferredDevicePtr()
        assert nbytes == W * H * 16
        dev = torch.as_tensor(multigpu.DeviceArray(p, (nbytes // 4,), "<f4"), device="cuda").cpu().numpy()
        assert np.array_equal(canon(dev.reshape(H, W, 4)), canon(lit))
        assert pt.last_ssao_ms > 0 and pt.last_deferred_ms > 0


@pytest.mark.gpu
def test_gpu_deferred_errors_leave_the_context_working():
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 24, 16
    frame = scenes.camera_frame(cam, W, H)
    fr = np.ascontiguousarray(frame)
    lib = capi.load()
    with PathTracer(16, 16) as pt:
        z = np.zeros((H, W), np.float32)
        with pytest.raises(IdkPtError, match="idkpt_ssao: no scene"):
            pt.Ssao(frame, z, np.zeros((H, W, 2), np.float32))
        with pytest.raises(IdkPtError, match="idkpt_deferred_lighting: no scene"):
            pt.DeferredLighting(frame, z, np.zeros((H, W, 2), np.float32), np.zeros((H, W, 3), np.float32), np.zeros((H, W, 2), np.float32),
                                np.zeros((H, W, 3), np.float32))
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [16, 16])
        pt.RenderPointShadows()
        g = gbuffer(pt, scene, frame, W, H)
        pt.Ssao(frame, g[0], g[1])
        good = pt.DeferredLighting(frame, *g, jitter=JITTER)
        gb, _, keep = PathTracer._gbuffer(list(g), [1, 2, 3, 2, 3])
        sst, dst = ssao_settings(), deferred_settings(1, 1, 0)

        def ssao_rc(f=fr, s=sst, gg=None):
            return lib.idkpt_ssao(pt._ctx, f.ctypes.data if f is not None else None, s, gg if gg is not None else gb, None, None)

        def deferred_rc(f=fr, s=dst, gg=None, indirect=None, rt=None, n=0):
            return lib.idkpt_deferred_lighting(pt._ctx, f.ctypes.data if f is not None else None, s, gg if gg is not None else gb,
                                               None, indirect, rt, n, None, None)

        assert ssao_rc(f=None) == -1 and deferred_rc(f=None) == -1                 # IDKPT_ERR_INVALID_ARGUMENT
        assert lib.idkpt_ssao(pt._ctx, fr.ctypes.data, None, gb, None, None) == -1
        assert lib.idkpt_deferred_lighting(pt._ctx, fr.ctypes.data, dst, None, None, None, None, 0, None, None) == -1

        def expect(rc, msg):
            with pytest.raises(IdkPtError, match=msg):
                pt._check(rc, "call")

        for field in ("Depth", "NormalRG"):
            bad = capi.IdkPtGBuffer.from_buffer_copy(gb)
            setattr(bad, field, None)
            expect(ssao_rc(gg=bad), "idkpt_ssao: null argument")
        for field in ("Depth", "NormalRG", "AlbedoRGB", "MetallicRoughness", "EmissiveRGB"):
            bad = capi.IdkPtGBuffer.from_buffer_copy(gb)
            setattr(bad, field, None)
            expect(deferred_rc(gg=bad), "idkpt_deferred_lighting: null argument")
        for w, h in ((0, H), (W, 0), (-3, H), (16385, H), (W, 16385)):
            bad = capi.IdkPtGBuffer.from_buffer_copy(gb)
            bad.Width, bad.Height = w, h
            expect(ssao_rc(gg=bad), "size outside 1..16384")
            expect(deferred_rc(gg=bad), "size outside 1..16384")
        bad = capi.IdkPtGBuffer.from_buffer_copy(gb)
        bad.OnDevice = 2
        expect(ssao_rc(gg=bad), "OnDevice is neither 0 nor 1")
        bad.OnDevice = 1                                                             # host pointers passed as device memory
        expect(ssao_rc(gg=bad), "not device memory on the context's device")
        expect(deferred_rc(gg=bad), "not device memory on the context's device")
        for n in (0, 1025, -5):
            expect(ssao_rc(s=ssao_settings(samples=n)), "SampleCount outside 1..1024")
        for mode in (-1, 3):
            expect(deferred_rc(s=deferred_settings(mode, 0, 0)), "ShadowMode outside 0..2")
        expect(deferred_rc(s=deferred_settings(0, 0, 1)), "IsVXGI without an indirect-light image")
        with PathTracer(16, 16) as other:                                            # IsSSAO needs an SSAO image of this size
            other.SetScene(scene)
            with pytest.raises(IdkPtError, match="IsSSAO needs an idkpt_ssao image"):
                other.DeferredLighting(frame, *g)
            other.Ssao(frame, g[0][:8, :8], g[1][:8, :8])
            with pytest.raises(IdkPtError, match="IsSSAO needs an idkpt_ssao image"):
                other.DeferredLighting(frame, *g)
            other.DeferredLighting(frame, *g, settings=deferred_settings(0, 0, 0))
        # PointShadowIndex: -1 or below the shadow count in Pcf / RayTraced, also after idkpt_update_range(LIGHTS)
        lights = scene.lights.copy()
        for idx in (2, -2, 100):
            lights["PointShadowIndex"][2] = idx
            pt.UpdateRange(capi.IDKPT_ARRAY_LIGHTS, 0, lights)
            for mode in (1, 2):
                with pytest.raises(IdkPtError, match="PointShadowIndex is neither -1 nor below the point-shadow count"):
                    pt.DeferredLighting(frame, *g, settings=deferred_settings(mode, 0, 0), rt_visibility=[g[0], g[0]])
            pt.DeferredLighting(frame, *g, settings=deferred_settings(0, 0, 0))      # None mode ignores the index
        pt.UpdateRange(capi.IDKPT_ARRAY_LIGHTS, 0, scene.lights)
        with_null = (ctypes.c_void_p * 2)(g[0].ctypes.data, None)
        expect(deferred_rc(s=deferred_settings(2, 0, 0), rt=with_null, n=2), "a visibility image is null")
        expect(deferred_rc(s=deferred_settings(2, 0, 0), rt=with_null, n=1), "RayTraced needs a visibility image per point shadow")
        expect(deferred_rc(s=deferred_settings(2, 0, 0)), "RayTraced needs a visibility image per point shadow")
        pt.SetPointShadows(shadows[:1], [16])                                        # one shadow: index 1 is now out of range
        with pytest.raises(IdkPtError, match="PointShadowIndex is neither -1"):
            pt.DeferredLighting(frame, *g, jitter=JITTER)
        pt.SetPointShadows(shadows, [16, 16])
        pt.RenderPointShadows()
        pt.Ssao(frame, g[0], g[1])
        assert np.array_equal(canon(pt.DeferredLighting(frame, *g, jitter=JITTER)), canon(good))
        pt.SetScene(scene)                                                           # a new scene drops both images
        with pytest.raises(IdkPtError, match="call idkpt_ssao first"):
            pt.SsaoDevicePtr()
        with pytest.raises(IdkPtError, match="call idkpt_deferred_lighting first"):
            pt.DeferredDevicePtr()


@pytest.mark.gpu
def test_gpu_deferred_between_async_computes():
    scene, cam, shadows = deferred_setup("cornell")
    w, h = 160, 120
    frame = scenes.camera_frame(cam, w, h)

    def go(with_lighting):
        with PathTracer(w, h, lanes=4) as pt:
            pt.SetScene(scene)
            pt.SetSky((0.6, 0.7, 0.9))
            pt.SetFrame(frame)
            pt.SetPointShadows(shadows, [64, 64])
            pt.RenderPointShadows()
            g = gbuffer(pt, scene, frame, w, h)
            want_ao = pt.Ssao(frame, g[0], g[1])
            want = pt.DeferredLighting(frame, *g, jitter=JITTER)
            got = []
            for k in range(6):
                pt.ComputeAsync()
                if with_lighting and k in (1, 3):
                    got.append((pt.Ssao(frame, g[0], g[1]), pt.DeferredLighting(frame, *g, jitter=JITTER)))
            pt.Sync()
            return pt.Result.copy(), (want_ao, want), got

    img0, _, _ = go(False)
    img1, (want_ao, want), got = go(True)
    assert np.array_equal(img0.view(np.uint32), img1.view(np.uint32))
    for ao, lit in got:
        assert np.array_equal(ao, want_ao) and np.array_equal(canon(lit), canon(want))


@pytest.mark.gpu
def test_gpu_misaligned_device_pointers_are_rejected_before_anything_runs():
    """OnDevice arrays must be aligned to the kernels' loads (8 B for NormalRG / MetallicRoughness, 16 B for the indirect image,
    4 B otherwise). Only the rejection is checked: no misaligned pointer is ever launched. A rejected call leaves the previous
    images valid."""
    import torch
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 24, 16
    frame = scenes.camera_frame(cam, W, H)
    fr = np.ascontiguousarray(frame)
    lib = capi.load()
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [16, 16])
        pt.RenderPointShadows()
        g = gbuffer(pt, scene, frame, W, H)
        dg = [torch.from_numpy(a).cuda() for a in g]
        small = pt.Ssao(frame, g[0][:8, :8], g[1][:8, :8])
        lit = pt.DeferredLighting(frame, *[a[:8, :8] for a in g], jitter=JITTER)

        def shifted(a, floats):   # the same values starting `floats` floats into a larger buffer
            buf = torch.zeros(a.numel() + 8, dtype=torch.float32, device="cuda")
            v = buf[floats:floats + a.numel()].view(a.shape)
            v.copy_(a)
            return v
        with pytest.raises(IdkPtError, match="NormalRG / MetallicRoughness pointer not 8-byte aligned"):
            pt.Ssao(frame, dg[0], shifted(dg[1], 1))
        with pytest.raises(IdkPtError, match="NormalRG / MetallicRoughness pointer not 8-byte aligned"):
            pt.DeferredLighting(frame, dg[0], dg[1], dg[2], shifted(dg[3], 3), dg[4], settings=deferred_settings(0, 0, 0))
        gi = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
        with pytest.raises(IdkPtError, match="indirect-light pointer not 16-byte aligned"):
            pt.DeferredLighting(frame, *dg, settings=deferred_settings(0, 0, 1), indirect=shifted(gi, 2))
        gb, _, keep = PathTracer._gbuffer(dg, [1, 2, 3, 2, 3])
        bad = capi.IdkPtGBuffer.from_buffer_copy(gb)
        bad.Depth = gb.Depth + 2                                                     # not even float-aligned
        with pytest.raises(IdkPtError, match="OnDevice pointer not 4-byte aligned"):
            pt._check(lib.idkpt_ssao(pt._ctx, fr.ctypes.data, ssao_settings(), bad, None, None), "idkpt_ssao")
        rt = [torch.from_numpy(x).cuda() for x in (g[0], g[0])]
        with pytest.raises(IdkPtError, match="OnDevice pointer not 4-byte aligned"):
            rt_ptrs = (ctypes.c_void_p * 2)(rt[0].data_ptr(), rt[1].data_ptr() + 2)
            pt._check(lib.idkpt_deferred_lighting(pt._ctx, fr.ctypes.data, deferred_settings(2, 0, 0), gb, None, None, rt_ptrs, 2, None, None),
                      "idkpt_deferred_lighting")
        # the rejected calls (at another size) left the last images in place and valid
        p, nbytes = pt.SsaoDevicePtr()
        assert nbytes == 64
        assert np.array_equal(torch.as_tensor(multigpu.DeviceArray(p, (nbytes,), "|u1"), device="cuda").cpu().numpy().reshape(8, 8), small)
        p, nbytes = pt.DeferredDevicePtr()
        assert nbytes == 64 * 16
        dev = torch.as_tensor(multigpu.DeviceArray(p, (nbytes // 4,), "<f4"), device="cuda").cpu().numpy()
        assert np.array_equal(canon(dev.reshape(8, 8, 4)), canon(lit))
        assert np.array_equal(pt.Ssao(frame, dg[0], dg[1]), pt.Ssao(frame, g[0], g[1]))   # aligned device arrays still work


@pytest.mark.gpu
@pytest.mark.parametrize("wrapper", ["ShadowsRayTraced", "VolumetricLighting", "DeferredLighting", "GBuffer", "Transparency", "LightsAndSkybox"])
def test_gpu_wrappers_reject_a_jitter_without_two_components(wrapper):
    """The library reads taaJitter[0] and [1]: a one-element jitter is a ValueError before it reaches the library, and the
    context renders the same image afterwards."""
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 24, 16
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [16, 16])
        pt.RenderPointShadows()
        gb = pt.GBuffer(frame, W, H)
        lit = pt.DeferredLighting(frame, *gb[:5], settings=deferred_settings(1, 0, 0))

        def lights_and_skybox(jitter):   # draws into the G-buffer pass's images and the lit image: render both again first
            pt.GBuffer(frame, W, H, download=False)
            pt.DeferredLighting(frame, *gb[:5], settings=deferred_settings(1, 0, 0), download=False)
            return pt.LightsAndSkybox(frame, jitter=jitter)
        call = {
            "ShadowsRayTraced": lambda j: pt.ShadowsRayTraced(frame, gb[0], gb[1], 0, samples=2, jitter=j)[0],
            "VolumetricLighting": lambda j: pt.VolumetricLighting(frame, gb[0], W, H, jitter=j),
            "DeferredLighting": lambda j: pt.DeferredLighting(frame, *gb[:5], settings=deferred_settings(1, 0, 0), jitter=j),
            "GBuffer": lambda j: np.concatenate([a.reshape(H, W, -1) for a in pt.GBuffer(frame, W, H, jitter=j)], -1),
            "Transparency": lambda j: pt.Transparency(frame, gb[0], jitter=j, color=lit.copy()),
            "LightsAndSkybox": lights_and_skybox,
        }[wrapper]
        want = call(JITTER)
        with pytest.raises(ValueError, match="jitter has two components"):
            call((0.01,))
        assert np.array_equal(canon(call(JITTER)), canon(want))
